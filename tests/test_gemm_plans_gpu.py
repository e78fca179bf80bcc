"""Every launch plan of the convolution / linear GEMMs (tests/gemm_plan_cases.py) through bre_conv_gemm, element by element against
float64.  Per case:
  * operands: tensor-core cases on the TF32 grid (every product exact), SIMT / linear cases plain fp32; rows of A and columns of B
    scaled by powers of two in 2^[-10, 10], so that a small output element cannot hide behind a large one;
  * guards: every operand and the output sit inside 4096 NaNs on each side, the output is prefilled with NaN; afterwards the guards
    are still NaN bit for bit (no store outside the output) and the output holds no NaN (every element written, no load outside
    the operands multiplied in);
  * bound: |out - ref| <= (K_total + 2) 2^-23 (|A| * |B|) for every element, ref and |A| * |B| in float64;
  * plan: what the launch recorded (engine.last_gemm_plan) is the table's plan, the restated one (scripts/profile_gemms.py) and the
    one the planner gave before the launch (engine.gemm_plan);
  * a second launch gives the same bits.
Then one case per mode with off-grid tensor-core operands (the bound widened by the 2^-10 operand truncation), and the tensor-core
cases once more on the cp.async producer (BRE_TC_TMA=0, read once per process, hence a subprocess)."""
import os
import subprocess
import sys
import zlib

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "scripts"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import gemm_plan_cases as T  # noqa: E402
import profile_gemms as P  # noqa: E402
from breaching_b200 import engine as E  # noqa: E402
from oracle.sweep_check import rna  # noqa: E402

DEV = "cuda:0"
U = 2.0 ** -23
TRUNC = 2.0 ** -10   # tensor cores read an fp32 operand off the TF32 grid with its 13 low mantissa bits dropped
GUARD = 4096         # floats of NaN before and after every buffer (a multiple of 4: 16-byte alignment is kept)
TC_CASES = [c for c in T.CASES if c[4][0] == "tc"]
# one case per mode with operands off the TF32 grid: split-K with a short or empty tail and a split across the sources
OFF_GRID = [c for c in TC_CASES if c[1] == (3, 9, 11, 64, 64, 3, 1, 1) and c[2] == 2]


def _nan_bits():
    return torch.full((1,), float("nan"), device=DEV).view(torch.int32)


def guarded(t):
    """(buffer, view): `t` copied into the middle of a NaN-filled buffer with GUARD floats on each side."""
    n = t.numel()
    buf = torch.full((2 * GUARD + n,), float("nan"), device=DEV)
    view = buf[GUARD:GUARD + n].view(t.shape)
    view.copy_(t)
    return buf, view


def guards_intact(buf):
    bits, nan = buf.view(torch.int32), _nan_bits()
    return bool((bits[:GUARD] == nan).all()) and bool((bits[-GUARD:] == nan).all())


def _pow2(n, gen):
    return torch.pow(2.0, torch.randint(-10, 11, (n,), generator=gen, device=DEV).float())


def operands(case, on_grid=True):
    """Per source: (A, B) as bre_conv_gemm takes them, scaled by powers of two along the GEMM rows of A and columns of B."""
    mode, geom, nsrc, backend, _ = case
    N, H, W, Ci, Co, R, st, pd = geom
    Ho, Wo = (H + 2 * pd - R) // st + 1, (W + 2 * pd - R) // st + 1
    gen = torch.Generator(device=DEV).manual_seed(zlib.crc32(T.label(case).encode()))
    tf32 = T.plan(case)["family"] == "tc" and on_grid

    def randn(*shape):
        t = torch.randn(*shape, generator=gen, device=DEV)
        return rna(t).float() if tf32 else t

    out = []
    for _ in range(nsrc):
        if mode == 0:     # A = im2col(x): rows are output pixels -> scale the input pixels; B columns = output channels
            a = randn(N, H, W, Ci) * _pow2(N * H * W, gen).view(N, H, W, 1)
            b = randn(Co, R, R, Ci) * _pow2(Co, gen).view(Co, 1, 1, 1)
        elif mode == 1:   # A = gathered dout pixels; B columns = input channels of the weight
            a = randn(N, Ho, Wo, Co) * _pow2(N * Ho * Wo, gen).view(N, Ho, Wo, 1)
            b = randn(Co, R, R, Ci) * _pow2(Ci, gen)
        else:             # A rows = output channels of dout; B columns = (r, s, c): the input's channels
            a = randn(N, H, W, Ci) * _pow2(Ci, gen)
            b = randn(N, Ho, Wo, Co) * _pow2(Co, gen)
        out.append((a, b))
    return out


def out_shape(mode, geom):
    N, H, W, Ci, Co, R, st, pd = geom
    Ho, Wo = (H + 2 * pd - R) // st + 1, (W + 2 * pd - R) // st + 1
    return {0: (N, Ho, Wo, Co), 1: (N, H, W, Ci), 2: (Co, R, R, Ci)}[mode]


def launch(case, ops):
    """One bre_conv_gemm call on guarded copies of `ops` into a NaN-prefilled guarded output -> (output buffer, view, operand buffers)."""
    mode, geom, nsrc, backend, _ = case
    N, H, W, Ci, Co, R, st, pd = geom
    bufs, views = [], []
    for a, b in ops:
        for t in (a, b):
            buf, view = guarded(t)
            bufs.append(buf)
            views.append(view)
    obuf, out = guarded(torch.full(out_shape(mode, geom), float("nan"), device=DEV))
    two = nsrc == 2
    E.conv_gemm(mode, views[0], views[1], out, N, H, W, Ci, Co, R, R, st, pd, a2=views[2] if two else None, w2=views[3] if two else None,
                backend=backend)
    torch.cuda.synchronize()
    return obuf, out, bufs


def reference(case, ops, absolute=False):
    """float64 sum over the sources (NHWC / OHWI like the kernel's output); absolute=True: the same contraction over |operands|."""
    import torch.nn.functional as F
    from torch.nn.grad import conv2d_input, conv2d_weight

    mode, geom, nsrc, backend, _ = case
    N, H, W, Ci, Co, R, st, pd = geom
    f = (lambda t: t.double().abs()) if absolute else (lambda t: t.double())
    nchw = lambda t: f(t).permute(0, 3, 1, 2)  # noqa: E731
    total = 0
    for a, b in ops:
        if mode == 0:
            total = total + F.conv2d(nchw(a), nchw(b), stride=st, padding=pd)
        elif mode == 1:
            total = total + conv2d_input((N, Ci, H, W), nchw(b), nchw(a), stride=st, padding=pd)
        else:
            total = total + conv2d_weight(nchw(a), (Co, Ci, R, R), nchw(b), stride=st, padding=pd)
    return total.permute(0, 2, 3, 1)


def check(case, want_plan, on_grid=True):
    """Run one case with every check of the module docstring; returns (output on the host, largest error / bound ratio)."""
    mode, geom, nsrc, backend, _ = case
    N, H, W, Ci, Co, R, st, pd = geom
    planned = E.gemm_plan(mode, backend, N, H, W, Ci, Co, R, R, st, pd, nsrc)
    ops = operands(case, on_grid)
    obuf, out, bufs = launch(case, ops)
    rec = E.last_gemm_plan()
    assert rec == want_plan, (rec, want_plan)
    assert planned == rec, (planned, rec)
    assert guards_intact(obuf), "a store outside the output"
    assert all(guards_intact(b) for b in bufs), "an operand's guard changed"
    assert not torch.isnan(out).any(), "an output element not written, or a load outside the operands"
    K = T.gemm_dims(mode, geom)[2] * nsrc
    ref, mag = reference(case, ops), reference(case, ops, absolute=True)
    slack = 0.0 if on_grid else 2 * TRUNC
    bound = ((K + 2) * U + slack) * mag
    err = (out.double() - ref).abs()
    ratio = (err / bound.clamp_min(1e-300)).max().item()
    worst = int((err / bound.clamp_min(1e-300)).argmax())
    print(f"{T.label(case)}: {rec['family']} {rec['tile_rows']} x {rec['tile_width']}, split {rec['splits']}, ring {rec['stages']}, "
          f"{rec['producer']}: max |err| / bound = {ratio:.3g}")
    assert ratio <= 1.0, (ratio, worst, out.flatten()[worst].item(), ref.flatten()[worst].item(), mag.flatten()[worst].item())
    _, again, _ = launch(case, ops)
    assert torch.equal(again.view(torch.int32), out.view(torch.int32)), "not bitwise the same from run to run"
    return out.cpu(), ratio


@pytest.mark.parametrize("case", T.CASES, ids=[T.label(c) for c in T.CASES])
def test_gemm_plan_matches_float64(case):
    mode, geom, nsrc, backend, _ = case
    want = T.plan(case)
    assert P.gemm_plan(mode, geom, nsrc, backend) == want
    check(case, want)


@pytest.mark.parametrize("case", OFF_GRID, ids=[T.label(c) for c in OFF_GRID])
def test_off_grid_operands_within_the_truncation_bound(case):
    assert len(OFF_GRID) == 3
    check(case, T.plan(case), on_grid=False)


def cp_async_results():
    """Every tensor-core case the cp.async producer covers (run with BRE_TC_TMA=0), checked against the restated plan and float64."""
    out = {}
    for case in TC_CASES:
        mode, geom, nsrc, backend, _ = case
        want = P.gemm_plan(mode, geom, nsrc, backend)
        if want is not None:
            assert want["producer"] == "cp.async"
            out[T.label(case)] = check(case, want)
    return out


def tma_outputs(labels):
    return {T.label(c): launch(c, operands(c))[1].cpu() for c in TC_CASES if T.label(c) in labels}


def test_cp_async_producer_within_the_bound(tmp_path):
    path = str(tmp_path / "cp_async.pt")
    code = (f"import sys, torch; sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]; import test_gemm_plans_gpu as t; "
            f"torch.save(t.cp_async_results(), {path!r})")
    res = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, BRE_TC_TMA="0"), capture_output=True, text=True, timeout=1200)
    print(res.stdout[-20000:])
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
    cp = torch.load(path)
    assert len(cp) >= len(TC_CASES) // 2, len(cp)
    tma = tma_outputs(set(cp))
    same = sorted(k for k in cp if torch.equal(cp[k][0].view(torch.int32), tma[k].view(torch.int32)))
    print(f"cp.async producer: {len(cp)} cases within the bound (largest ratio {max(r for _, r in cp.values()):.3g}); "
          f"{len(same)} bitwise equal to the TMA result, {len(cp) - len(same)} not")
    for k in sorted(set(cp) - set(same)):
        print(f"  differs from TMA: {k}")
