"""Restatements of the shape-changing augmentations of the reference (``attacks/auxiliaries/augmentations.py``) with explicit draws,
composable in config order with ``restate.augment_candidate``, and a trial oracle whose closure sees the view
(``optimization_based_attack.py:149-162`` with ``differentiable_augmentations: True``).

- ``zoom(x, out)``: ``Zoom`` (:34-40), ``Upsample(size=(out, out), bilinear, align_corners=False)``.
- ``centerzoom(x, fov, out)``: ``CenterZoom`` (:43-55), the centred ``fov x fov`` crop resized to ``out x out``.
- ``focus(x, size, std, pert)``: ``Focus`` (:20-31) with its draw ``pert`` = ``(rand(2) * 2 - 1) * std`` given; ``corner`` instead of
  ``pert`` takes the window corner directly (what the engine reads back).
- ``antialias(x, width, stride, channels)``: ``AntiAlias`` (:198-226), depthwise binomial filter, zero padding ``width // 2``.
"""
import torch
import torch.nn.functional as F

from . import restate

FILTER_BANK = {1: [1.0], 2: [1.0, 1.0], 3: [1.0, 2.0, 1.0], 4: [1.0, 3.0, 3.0, 1.0], 5: [1.0, 4.0, 6.0, 4.0, 1.0],
               6: [1.0, 5.0, 10.0, 10.0, 5.0, 1.0], 7: [1.0, 6.0, 15.0, 20.0, 15.0, 6.0, 1.0]}   # binomial rows


def zoom(x, out_size):
    return F.interpolate(x, size=(out_size, out_size), mode="bilinear", align_corners=False)


def centerzoom(x, initial_fov, out_size):
    H, W = x.shape[-2:]
    y0, x0 = (H - initial_fov) // 2, (W - initial_fov) // 2
    return F.interpolate(x[:, :, y0:y0 + initial_fov, x0:x0 + initial_fov], size=out_size, mode="bilinear", align_corners=False)


def focus_corner(H, W, size, pert):
    """The window corner of ``Focus`` for the draw ``pert`` (two values in [-std, std)): ``.long()`` truncates toward zero."""
    pert = torch.as_tensor(pert, dtype=torch.float32)
    y0 = int((pert[0] + H // 2 - size // 2).long().clamp(min=0, max=H - size))
    x0 = int((pert[1] + W // 2 - size // 2).long().clamp(min=0, max=W - size))
    return y0, x0


def focus(x, size, pert=None, corner=None):
    H, W = x.shape[-2:]
    y0, x0 = corner if corner is not None else focus_corner(H, W, size, pert)
    return x[:, :, y0:y0 + size, x0:x0 + size]


def antialias(x, width=5, stride=1, channels=3):
    base = torch.as_tensor(FILTER_BANK[int(width)], dtype=x.dtype)
    k = base[:, None] * base[None, :]
    k = k / k.sum()
    weight = k[None, None].repeat(channels, 1, 1, 1)
    return F.conv2d(x, weight, padding=int(width) // 2, stride=stride, groups=x.shape[1])


def apply(x, entries):
    """Compose in config order.  ``entries``: list of (key, opts, draw) with key one of zoom / centerzoom / focus / antialias /
    pixel (``draw`` = the keyword arguments of ``restate.augment_candidate``); a focus ``draw`` is {"corner": (y0, x0)} or
    {"pert": (p0, p1)}."""
    for key, opts, draw in entries:
        if key == "zoom":
            x = zoom(x, int(opts.get("out_size", 224)))
        elif key == "centerzoom":
            x = centerzoom(x, int(opts.get("initial_fov", 32)), int(opts.get("out_size", 224)))
        elif key == "focus":
            x = focus(x, int(opts.get("size", 224)), **draw)
        elif key == "antialias":
            x = antialias(x, int(opts.get("width", 5)), int(opts.get("stride", 1)), int(opts.get("channels", 3)))
        elif key == "pixel":
            x = restate.augment_candidate(x, **draw)
        else:
            raise KeyError(key)
    return x


class ViewTrialOracle(restate.TrialOracle):
    """``TrialOracle`` whose objective and regularisers see ``view(x)`` (deterministic entries, see ``apply``); the candidate gradient
    comes through autograd of the composed view, as in the reference's differentiable mode.  Scores stay on the candidate."""

    def __init__(self, *args, entries=(), **kwargs):
        super().__init__(*args, **kwargs)
        self.entries = list(entries)

    def objective_terms(self, x):
        return super().objective_terms(apply(x, self.entries))
