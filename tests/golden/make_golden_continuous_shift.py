"""Regenerate tests/golden/continuous_shift.pt: the *unmodified* reference ``RandomTransform`` (loaded through oracle/refshim.py, run in
float64 with its draw ``randgen`` passed in) on fixed inputs, for every ``mode`` x ``padding`` x (``fliplr``, ``flipud``) combination:
views and vector-Jacobian products against fixed probes.

Each (mode, padding) pair meets all four size / shift variants, one per flip combination: S = 17 with shifts 3 and 17 (two images, one of
them flipped by each enabled flag), S = 32 with shifts 3 and 64 (one image; a shift of 64 moves the grid by up to 32 pixels, so
reflection folds more than once).  The uniforms are fp32 numbers, so the device receives them exactly, and the nearest cases are drawn
again until no source coordinate lies within 1e-5 of a rounding boundary.

    python tests/golden/make_golden_continuous_shift.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from cshift_oracle import source_coordinates  # noqa: E402
from oracle import refshim  # noqa: E402

MODES = ("bilinear", "nearest", "bicubic")
PADDINGS = ("zeros", "border", "reflection", "circular")
FLIPS = ((False, False), (True, False), (False, True), (True, True))
VARIANTS = ((17, 2, 3), (17, 2, 17), (32, 1, 3), (32, 1, 64))     # (S, images, shift), one per flip combination


def _randgen(gen, N, S, shift, mode, padding, flips):
    while True:
        u = torch.rand(N, 2, generator=gen).float().double()       # fp32-exact uniforms
        bits = torch.tensor([[0.75, 0.75], [0.25, 0.25]], dtype=torch.float64)[:N]
        r = torch.cat([u, bits], dim=1)
        if mode != "nearest":
            return r
        dist = min((p - p.floor() - 0.5).abs().min().item() for p in source_coordinates(S, shift, r, padding, *flips))
        if dist > 1e-5:
            return r


def main():
    torch.set_default_dtype(torch.float64)          # the module builds its grid in the default dtype
    ref = refshim.import_reference()
    from breaching.attacks.auxiliaries.augmentations import RandomTransform

    assert ref is not None
    gen = torch.Generator().manual_seed(20261017)
    inputs = {}
    for S, N, _ in VARIANTS:
        if S not in inputs:
            inputs[S] = dict(x=torch.randn(N, 1, S, S, generator=gen), probe=torch.randn(N, 1, S, S, generator=gen))
    cases = []
    for mode in MODES:
        for padding in PADDINGS:
            for flips, (S, N, shift) in zip(FLIPS, VARIANTS):
                randgen = _randgen(gen, N, S, shift, mode, padding, flips)
                module = RandomTransform(shift=shift, fliplr=flips[0], flipud=flips[1], mode=mode, padding=padding)
                x = inputs[S]["x"].clone().requires_grad_(True)
                view = module(x, randgen=randgen)
                (vjp,) = torch.autograd.grad((view * inputs[S]["probe"]).sum(), x)
                cases.append(dict(S=S, shift=shift, mode=mode, padding=padding, fliplr=flips[0], flipud=flips[1], randgen=randgen,
                                  view=view.detach(), vjp=vjp))
    out = os.path.join(ROOT, "tests", "golden", "continuous_shift.pt")
    torch.save(dict(inputs=inputs, cases=cases), out)
    print(out, os.path.getsize(out), "bytes,", len(cases), "cases")


if __name__ == "__main__":
    main()
