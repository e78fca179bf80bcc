"""128 x 32 tiles for the under-filled data / weight gradients of the tensor-core GEMM (csrc/igemm_tc.cu, tc_plan): at batch 1
ResNet-18's layer-3 / layer-4 dgrad and the stem's column wgrad have so few 128 x 64 tiles that even the 8-CTA split leaves half the
H100 idle, and they run on twice as many 128 x 32 tiles instead.  Every output element keeps its k-ranges, MMA chain and cluster
reduction order, so the results must be bitwise those of 128 x 64 tiles (BRE_TC_NARROW=0, read once per process, hence a
subprocess), and within the sweep checker's GEMM bound of float64."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "scripts")):
    if p not in sys.path:
        sys.path.insert(0, p)

from breaching_b200 import engine as E  # noqa: E402
from oracle.sweep_check import rna  # noqa: E402
from profile_gemms import split_plan  # noqa: E402

DEV = "cuda:0"
U = 2.0 ** -23

# (label, mode, (N, H, W, Ci, Co, R, stride, pad), nsrc): mode 0 fprop, 1 dgrad, 2 wgrad -- config-2 shapes
CASES = [
    ("layer4 dgrad", 1, (1, 7, 7, 512, 512, 3, 1, 1), 1),
    ("layer4 tangent dgrad", 1, (1, 7, 7, 512, 512, 3, 1, 1), 2),
    ("layer3 dgrad", 1, (1, 14, 14, 256, 256, 3, 1, 1), 1),
    ("layer3 tangent dgrad", 1, (1, 14, 14, 256, 256, 3, 1, 1), 2),
    ("layer4.0 conv1 tangent dgrad (stride-2, per class)", 1, (1, 14, 14, 256, 512, 3, 2, 1), 2),
    ("stem column wgrad", 2, (1, 112, 112, 192, 64, 1, 1, 0), 1),
    ("stem column wgrad, dual source", 2, (1, 112, 112, 192, 64, 1, 1, 0), 2),
    ("layer1 wgrad", 2, (1, 56, 56, 64, 64, 3, 1, 1), 1),
    ("layer4 fprop", 0, (1, 7, 7, 512, 512, 3, 1, 1), 1),
    ("layer4 tangent fprop", 0, (1, 7, 7, 512, 512, 3, 1, 1), 2),
    ("stem column tangent dgrad", 1, (1, 112, 112, 192, 64, 1, 1, 0), 2),
]
NARROW = {"layer4 dgrad", "layer4 tangent dgrad", "layer3 dgrad", "layer3 tangent dgrad", "stem column wgrad", "stem column wgrad, dual source"}


def _rand(*shape, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return rna(torch.randn(*shape, generator=g, dtype=torch.float64)).float().to(DEV)   # on the TF32 grid: the products are exact


def operands(mode, geom, nsrc):
    N, H, W, Ci, Co, R, st, pd = geom
    Ho, Wo = (H + 2 * pd - R) // st + 1, (W + 2 * pd - R) // st + 1
    x = [_rand(N, H, W, Ci, seed=1 + s) for s in range(nsrc)]
    w = [_rand(Co, R, R, Ci, seed=3 + s) for s in range(nsrc)]
    dy = [_rand(N, Ho, Wo, Co, seed=5 + s) for s in range(nsrc)]
    out = torch.full({0: (N, Ho, Wo, Co), 1: (N, H, W, Ci), 2: (Co, R, R, Ci)}[mode], float("nan"), device=DEV)
    return x, w, dy, out


def launch(mode, geom, nsrc, ops):
    N, H, W, Ci, Co, R, st, pd = geom
    x, w, dy, out = ops
    a, b = {0: (x, w), 1: (dy, w), 2: (x, dy)}[mode]
    E.conv_gemm(mode, a[0], b[0], out, N, H, W, Ci, Co, R, R, st, pd, a2=a[1] if nsrc == 2 else None, w2=b[1] if nsrc == 2 else None,
                backend=1)
    return out


def reference(mode, geom, nsrc, ops, absolute=False):
    """float64 result (NHWC / OHWI like the kernel's output) and, with absolute=True, the same contraction over |operands|."""
    import torch.nn.functional as F
    from torch.nn.grad import conv2d_input, conv2d_weight

    N, H, W, Ci, Co, R, st, pd = geom
    x, w, dy, _ = ops
    f = (lambda t: t.double().abs()) if absolute else (lambda t: t.double())
    nchw = lambda t: f(t).permute(0, 3, 1, 2)  # noqa: E731
    total = 0
    for s in range(nsrc):
        if mode == 0:
            total = total + F.conv2d(nchw(x[s]), nchw(w[s]), stride=st, padding=pd)
        elif mode == 1:
            total = total + conv2d_input((N, Ci, H, W), nchw(w[s]), nchw(dy[s]), stride=st, padding=pd)
        else:
            total = total + conv2d_weight(nchw(x[s]), (Co, Ci, R, R), nchw(dy[s]), stride=st, padding=pd)
    return total.permute(0, 2, 3, 1)


def results():
    return {label: launch(mode, geom, nsrc, operands(mode, geom, nsrc)).cpu() for label, mode, geom, nsrc in CASES}


@pytest.mark.parametrize("label,mode,geom,nsrc", CASES, ids=[c[0] for c in CASES])
def test_matches_float64_within_the_gemm_bound(label, mode, geom, nsrc):
    _, bn, splits, kb = split_plan(mode, geom, nsrc)
    assert (bn == 32) == (label in NARROW) and (label not in NARROW or splits == 8), (bn, splits)
    ops = operands(mode, geom, nsrc)
    out = launch(mode, geom, nsrc, ops).double()
    ref, mag = reference(mode, geom, nsrc, ops), reference(mode, geom, nsrc, ops, absolute=True)
    N, H, W, Ci, Co, R, st, pd = geom
    K = {0: R * R * Ci, 1: R * R * Co, 2: N * ((H + 2 * pd - R) // st + 1) * ((W + 2 * pd - R) // st + 1)}[mode] * nsrc
    ratio = ((out - ref).abs() / ((K + 2) * U * mag).clamp_min(1e-300)).max().item()
    print(f"{label}: 128 x {bn} tiles, split {splits}, max |err| / bound = {ratio:.3g}")
    assert torch.isfinite(out).all() and ratio <= 1.0, ratio
    again = launch(mode, geom, nsrc, ops).double()
    assert torch.equal(again, out)   # run to run


def test_narrow_tiles_are_bitwise_the_wide_result(tmp_path):
    """The same launches with 128 x 64 tiles everywhere (BRE_TC_NARROW=0) give exactly the same bits."""
    path = str(tmp_path / "wide.pt")
    code = (f"import sys, torch; sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]; import test_tc_narrow_tiles_gpu as t; "
            f"torch.save(t.results(), {path!r})")
    res = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, BRE_TC_NARROW="0"), capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
    wide, narrow = torch.load(path), results()
    for label in wide:
        assert torch.equal(wide[label], narrow[label]), label
