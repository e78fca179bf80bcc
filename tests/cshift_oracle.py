"""Float64 restatement of the reference's ``RandomTransform`` (``attacks/auxiliaries/augmentations.py:141-205``) with its draw ``randgen``
given, and a view trial oracle whose entries may contain it.

``continuous_shift(x, shift, randgen, mode, padding, fliplr, flipud)``: the S x S grid of ``linspace(-1, 1, S)`` (S = x.shape[2]) shifted
per image by ``(randgen[:, 0 / 1] - 0.5) * 2 * shift / (S - 1)``, the x (y) coordinate negated for images with ``randgen[:, 2 (3)] > 0.5``
when ``fliplr`` (``flipud``), ``padding="circular"`` mapped to ``(g + 1) % 1 - 1`` with zeros padding, then ``F.grid_sample`` with
``align_corners=True`` (the module forces it).  ``randgen_from_draws`` builds ``randgen`` from the engine's read-back draws.
"""
import torch
import torch.nn.functional as F

from oracle import augment_views as AV


def continuous_shift(x, shift, randgen, mode="bilinear", padding="reflection", fliplr=False, flipud=False):
    N, S = x.shape[0], x.shape[2]
    lin = torch.linspace(-1, 1, S, dtype=x.dtype)
    randgen = torch.as_tensor(randgen, dtype=x.dtype)
    delta = shift / (S - 1)
    gx = lin[None, None, :].expand(N, S, S) + ((randgen[:, 0] - 0.5) * 2 * delta)[:, None, None]
    gy = lin[None, :, None].expand(N, S, S) + ((randgen[:, 1] - 0.5) * 2 * delta)[:, None, None]
    if fliplr:
        gx = torch.where((randgen[:, 2] > 0.5)[:, None, None], -gx, gx)
    if flipud:
        gy = torch.where((randgen[:, 3] > 0.5)[:, None, None], -gy, gy)
    grid = torch.stack([gx, gy], dim=-1)
    if padding == "circular":
        grid, padding = (grid + 1) % 1 - 1, "zeros"
    return F.grid_sample(x, grid, mode=mode, padding_mode=padding, align_corners=True)


def source_coordinates(S, shift, randgen, padding, fliplr=False, flipud=False):
    """Float64 source coordinates [N, S] of every output column (x) and row (y) after the padding rule of bilinear / nearest sampling:
    what nearest rounds.  Used to keep the fixture's nearest cases away from rounding boundaries."""
    randgen = torch.as_tensor(randgen, dtype=torch.float64)
    lin = torch.linspace(-1, 1, S, dtype=torch.float64)
    out = []
    for axis, flip in ((0, fliplr), (1, flipud)):
        g = lin[None, :] + ((randgen[:, axis] - 0.5) * 2 * (shift / (S - 1)))[:, None]
        if flip:
            g = torch.where((randgen[:, 2 + axis] > 0.5)[:, None], -g, g)
        if padding == "circular":
            g = (g + 1) % 1 - 1
        p = (g + 1) / 2 * (S - 1)
        if padding == "border":
            p = p.clamp(0, S - 1)
        elif padding == "reflection":
            p = p.abs()
            extra, flips = torch.fmod(p, S - 1), torch.floor(p / (S - 1))
            p = torch.where(flips % 2 == 0, extra, (S - 1) - extra).clamp(0, S - 1)
        out.append(p)
    return out


def randgen_from_draws(sx, sy, fliplr=None, flipud=None):
    n = len(sx)
    lr = fliplr if fliplr is not None else [0] * n
    ud = flipud if flipud is not None else [0] * n
    return torch.tensor([[float(a), float(b), float(c), float(d)] for a, b, c, d in zip(sx, sy, lr, ud)], dtype=torch.float64)


def apply(x, entries):
    """``oracle.augment_views.apply`` with one more key: ("continuous_shift", opts, draw) applies ``continuous_shift(x, **draw)``."""
    for entry in entries:
        x = continuous_shift(x, **entry[2]) if entry[0] == "continuous_shift" else AV.apply(x, [entry])
    return x


class ShiftTrialOracle(AV.ViewTrialOracle):
    def objective_terms(self, x):
        return super(AV.ViewTrialOracle, self).objective_terms(apply(x, self.entries))
