"""Per-kernel parity on the GPU: each CUDA kernel, called through the C ABI, against a torch fp32/fp64 restatement."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from breaching_b200 import engine as E  # noqa: E402

DEV = "cuda:0"

def _rand(*shape, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return torch.randn(*shape, generator=g).to(DEV)


def _nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def _relerr(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()


def test_conv_is_deterministic_across_launches():
    N, H, W, Ci, Co, R, st, pd = 1, 7, 7, 512, 512, 3, 1, 1
    x, w = _nhwc(_rand(N, Ci, H, W, seed=1)), _rand(Co, R, R, Ci, seed=2)
    a = torch.empty(N, H, W, Co, device=DEV)
    b = torch.empty_like(a)
    E.conv_gemm(0, x, w, a, N, H, W, Ci, Co, R, R, st, pd)
    E.conv_gemm(0, x, w, b, N, H, W, Ci, Co, R, R, st, pd)
    assert torch.equal(a, b)  # split-K partials are reduced in a fixed order


@pytest.mark.parametrize("n", [1, 1023, 1024, 4097, 11_380_173])
def test_match_reduce(n):
    G, g = _rand(n, seed=1), _rand(n, seed=2)
    nchunks = (n + 1023) // 1024
    w = torch.rand(nchunks, device=DEV)
    sums = E.match_reduce(G, g, w)
    Gd, gd = G.double(), g.double()
    wl = w.double().repeat_interleave(1024)[:n]
    ref = [(Gd * gd).sum(), (Gd * Gd).sum(), (gd * gd).sum(), ((Gd - gd) ** 2).sum(), (wl * (Gd - gd).abs()).sum()]
    for a, b in zip(sums, ref):
        assert math.isclose(a, b.item(), rel_tol=1e-6, abs_tol=1e-6), (sums, [r.item() for r in ref])
    again = E.match_reduce(G, g, w)
    assert again == sums  # deterministic
    m = E.match_reduce(G, g, None, mask_value=0.5)
    mask = (gd.abs() > 0.5)
    assert math.isclose(m[0], (Gd * gd * mask).sum().item(), rel_tol=1e-6)
    assert math.isclose(m[1], ((Gd * mask) ** 2).sum().item(), rel_tol=1e-6)


@pytest.mark.parametrize("p,q,dbl", [(1, 1, False), (2, 0.5, True), (2, 1.25, False), (1, 1, True)])
@pytest.mark.parametrize("shape", [(1, 3, 224, 224), (2, 3, 32, 32), (3, 3, 17, 45)])
def test_total_variation_value_and_gradient(p, q, dbl, shape):
    from oracle import restate

    x = _rand(*shape, seed=3)
    val, grad = E.total_variation(x, scale=0.2, inner_exp=p, outer_exp=q, double_opponents=dbl)
    xd = x.double().cpu().requires_grad_(True)
    ref = restate.total_variation(xd, scale=0.2, inner_exp=p, outer_exp=q, double_opponents=dbl)
    (gref,) = torch.autograd.grad(ref, xd)
    assert math.isclose(val, ref.item(), rel_tol=2e-5), (val, ref.item())
    assert _relerr(grad.cpu(), gref) < 5e-5
    base = grad.clone()  # accumulate on top of an existing gradient: result must be exactly doubled
    _, acc = E.total_variation(x, scale=0.2, inner_exp=p, outer_exp=q, double_opponents=dbl, grad=base)
    assert _relerr(acc.cpu(), 2 * gref) < 5e-5


@pytest.mark.gpu
@pytest.mark.parametrize("rows,Ci,Co,dual", [(32, 96, 50304, False), (32, 96, 50304, True), (5, 64, 9000, True), (17, 128, 8192, False)])
def test_tall_linear_dgrad_matches_float64(rows, Ci, Co, dual):
    """dgrad of a linear layer with a very long reduction (the token models' 96 -> 50257 decoder, tag.yaml / BASELINE config 5):
    chunked fp32 register reduction + fixed-order fold (csrc/linear_small.cu) against float64; run twice: bitwise reproducible."""
    from breaching_b200 import engine as E

    dev = torch.device("cuda:0")
    g = torch.Generator(device="cpu").manual_seed(rows * 1000 + Ci)
    dy = torch.randn(rows, Co, generator=g).to(dev)
    w = (torch.randn(Co, Ci, generator=g) / 8).to(dev)
    dy2 = torch.randn(rows, Co, generator=g).to(dev) if dual else None
    w2 = (torch.randn(Co, Ci, generator=g) / 8).to(dev) if dual else None
    want = dy.double() @ w.double()
    if dual:
        want = want + dy2.double() @ w2.double()
    for backend in (0, 1):
        out = torch.full((rows, Ci), float("nan"), device=dev)
        E.conv_gemm(1, dy, w, out, rows, 1, 1, Ci, Co, 1, 1, 1, 0, a2=dy2, w2=w2, backend=backend)
        again = torch.empty_like(out)
        E.conv_gemm(1, dy, w, again, rows, 1, 1, Ci, Co, 1, 1, 1, 0, a2=dy2, w2=w2, backend=backend)
        torch.cuda.synchronize()
        assert torch.equal(out, again)
        rel = ((out.double() - want).norm() / want.norm()).item()
        assert rel < 2e-6, (backend, rel)


@pytest.mark.gpu
@pytest.mark.parametrize("rows,Ci,Co", [(32, 96, 288), (32, 96, 1536), (20, 96, 96), (32, 1536, 96), (1, 512, 397), (8, 2048, 397)])
def test_small_row_linear_kernels_match_float64(rows, Ci, Co):
    """Linear layers on <= 32 rows (classification heads, token-model projections at batch 1) through the engine's dispatch rule
    (`bre_conv_gemm` backend 2: matrix-vector kernels for short reductions, the GEMM back ends otherwise): fprop / dgrad / wgrad with
    one and two sources against float64."""
    from breaching_b200 import engine as E

    dev = torch.device("cuda:0")
    g = torch.Generator(device="cpu").manual_seed(rows + Ci + Co)
    x, x2 = (torch.randn(rows, Ci, generator=g).to(dev) for _ in range(2))
    w, w2 = ((torch.randn(Co, Ci, generator=g) / Ci ** 0.5).to(dev) for _ in range(2))
    dy, dy2 = (torch.randn(rows, Co, generator=g).to(dev) for _ in range(2))
    geom = (rows, 1, 1, Ci, Co, 1, 1, 1, 0)

    def rel(a, b):
        return ((a.double() - b).norm() / b.norm()).item()

    for backend, tol in ((0, 2e-6), (2, 2e-3)):   # 2 = engine dispatch: TF32 products where the tensor-core kernel takes the shape
        out = torch.empty(rows, Co, device=dev)
        E.conv_gemm(0, x, w, out, *geom, backend=backend)
        assert rel(out, x.double() @ w.double().T) < tol, ("fprop", backend)
        E.conv_gemm(0, x, w, out, *geom, a2=x2, w2=w2, backend=backend)
        assert rel(out, x.double() @ w.double().T + x2.double() @ w2.double().T) < tol, ("fprop2", backend)
        din = torch.empty(rows, Ci, device=dev)
        E.conv_gemm(1, dy, w, din, *geom, backend=backend)
        assert rel(din, dy.double() @ w.double()) < tol, ("dgrad", backend)
        E.conv_gemm(1, dy, w, din, *geom, a2=dy2, w2=w2, backend=backend)
        assert rel(din, dy.double() @ w.double() + dy2.double() @ w2.double()) < tol, ("dgrad2", backend)
        dw = torch.empty(Co, Ci, device=dev)
        E.conv_gemm(2, x, dy, dw, *geom, backend=backend)
        assert rel(dw, dy.double().T @ x.double()) < tol, ("wgrad", backend)
        # two sources: the tangent weight gradient of a FedAvg step, wgrad(a, d_T) + wgrad(a', d_B)
        E.conv_gemm(2, x, dy, dw, *geom, a2=x2, w2=dy2, backend=backend)
        assert rel(dw, dy.double().T @ x.double() + dy2.double().T @ x2.double()) < tol, ("wgrad2", backend)
