"""Token-sequence kernels of the transformer / TAG path (csrc/tokens.cu: LayerNorm and multi-head self-attention in all four
sweeps) against the float64 formulas of oracle/transformer_interp.py -- which are themselves verified against autograd's
double backward and the reference's TAG closure (tests/test_transformer_interp.py)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from breaching_b200 import engine as E  # noqa: E402
from oracle import transformer_interp as TI  # noqa: E402

DEV = torch.device("cuda:0")


def _relerr(a, b):
    return ((a.double().cpu() - b.double().cpu()).norm() / (b.double().cpu().norm() + 1e-30)).item()


@pytest.mark.parametrize("rows,C", [(32, 96), (16, 16), (7, 50), (64, 1536)])
def test_layernorm_four_sweeps(rows, C):
    gen = torch.Generator().manual_seed(rows * 1000 + C)
    r = lambda *s: torch.randn(*s, generator=gen, dtype=torch.double)  # noqa: E731
    x, dy, xd, dyd = r(rows, C), r(rows, C), r(rows, C), r(rows, C)
    gamma, beta, vg, vb = 1 + 0.2 * r(C), 0.1 * r(C), r(C), r(C)
    eps = 1e-5
    y, xh, inv = TI._ln_forward(x, gamma, beta, eps)
    dx, Gg, Gb, t, u = TI._ln_backward(dy[None], xh[None], inv[None], gamma)
    yd, xhd = TI._ln_tangent_forward(xd, xh, inv, gamma, vg, vb)
    dxd = TI._ln_tangent_backward(dyd, dy, t[0], u[0], xd, xh, xhd, inv, gamma, vg)
    f = lambda v: v.float().to(DEV).contiguous()  # noqa: E731
    stats = torch.empty(rows, 2, device=DEV)
    out0 = E.token_layernorm(0, f(x), f(gamma), f(beta), stats, eps=eps)
    assert _relerr(out0, y) < 1e-5
    out1, gg, gb = E.token_layernorm(1, f(x), f(gamma), f(beta), stats, in1=f(dy), eps=eps, want_param_grad=True)
    assert _relerr(out1, dx[0]) < 2e-5 and _relerr(gg, Gg) < 2e-5 and _relerr(gb, Gb) < 2e-5
    out2 = E.token_layernorm(2, f(x), f(gamma), f(beta), stats, in1=f(xd), v_gamma=f(vg), v_beta=f(vb), eps=eps)
    assert _relerr(out2, yd) < 2e-5
    out3 = E.token_layernorm(3, f(x), f(gamma), f(beta), stats, in1=f(dyd), in2=f(dy), in3=f(xd), v_gamma=f(vg), v_beta=f(vb), eps=eps)
    assert _relerr(out3, dxd) < 5e-5


# (1, 33, 2, 8): one row past a lane stride; (2, 64, 4, 16): two full strides; (1, 100, 2, 12): 198 400 B of shared memory, just
# under the kernel's 200 KB opt-in
@pytest.mark.parametrize("B,T,heads,dh", [(1, 32, 8, 12), (2, 8, 4, 4), (3, 5, 2, 7), (1, 33, 2, 8), (2, 64, 4, 16), (1, 100, 2, 12)])
def test_attention_four_sweeps(B, T, heads, dh):
    gen = torch.Generator().manual_seed(B * 100 + T)
    d = heads * dh
    r = lambda *s: torch.randn(*s, generator=gen, dtype=torch.double)  # noqa: E731
    qkv, qkvd, dO, dOd = r(B * T, 3 * d), r(B * T, 3 * d), r(B * T, d), r(B * T, d)

    def heads_of(t):   # [B*T, d] -> [B, h, T, dh]
        return t.view(B, T, heads, dh).transpose(1, 2)

    def merge(t):
        return t.transpose(1, 2).reshape(B * T, d)

    Q, K, V = (heads_of(t) for t in qkv.split(d, dim=1))
    Qd, Kd, Vd = (heads_of(t) for t in qkvd.split(d, dim=1))
    s = 1.0 / dh ** 0.5
    P = torch.softmax(Q @ K.transpose(-1, -2) * s, dim=-1)
    O = merge(P @ V)
    dOh, dOdh = heads_of(dO), heads_of(dOd)
    dV = P.transpose(-1, -2) @ dOh
    dP = dOh @ V.transpose(-1, -2)
    rr = (dP * P).sum(-1, keepdim=True)
    dS = P * (dP - rr)
    dqkv = torch.cat([merge(dS @ K * s), merge(dS.transpose(-1, -2) @ Q * s), merge(dV)], dim=1)
    Sd = (Qd @ K.transpose(-1, -2) + Q @ Kd.transpose(-1, -2)) * s
    Pd = P * (Sd - (P * Sd).sum(-1, keepdim=True))
    Od = merge(Pd @ V + P @ Vd)
    dVd = Pd.transpose(-1, -2) @ dOh + P.transpose(-1, -2) @ dOdh
    dPd = dOdh @ V.transpose(-1, -2) + dOh @ Vd.transpose(-1, -2)
    rd = (dPd * P + dP * Pd).sum(-1, keepdim=True)
    dSd = Pd * (dP - rr) + P * (dPd - rd)
    dqkvd = torch.cat([merge((dSd @ K + dS @ Kd) * s), merge((dSd.transpose(-1, -2) @ Q + dS.transpose(-1, -2) @ Qd) * s), merge(dVd)],
                      dim=1)
    f = lambda v: v.float().to(DEV).contiguous()  # noqa: E731
    Pg, Pdg = torch.empty(B, heads, T, T, device=DEV), torch.empty(B, heads, T, T, device=DEV)
    out0 = E.token_attention(0, f(qkv), B, T, heads, Pg, Pdg)
    assert _relerr(out0, O) < 1e-5 and _relerr(Pg, P) < 1e-5
    out1 = E.token_attention(1, f(qkv), B, T, heads, Pg, Pdg, in1=f(dO))
    assert _relerr(out1, dqkv) < 2e-5
    out2 = E.token_attention(2, f(qkv), B, T, heads, Pg, Pdg, in1=f(qkvd))
    assert _relerr(out2, Od) < 2e-5 and _relerr(Pdg, Pd) < 2e-5
    out3 = E.token_attention(3, f(qkv), B, T, heads, Pg, Pdg, in1=f(dOd), in2=f(dO), in3=f(qkvd))
    assert _relerr(out3, dqkvd) < 5e-5


def test_attention_head_over_the_shared_memory_limit_is_rejected():
    """T = 128, dh = 12 needs 8 T dh + 4 T^2 floats = 311 296 B: an error naming the limit, not a launch."""
    B, T, heads, dh = 1, 128, 2, 12
    qkv = torch.randn(B * T, 3 * heads * dh, device=DEV)
    P, Pd = torch.empty(B, heads, T, T, device=DEV), torch.empty(B, heads, T, T, device=DEV)
    with pytest.raises(E.EngineError, match="311296 B of shared memory"):
        E.token_attention(0, qkv, B, T, heads, P, Pd)


@pytest.mark.parametrize("sweep", [0, 1, 2, 3])
def test_token_kernels_round_their_output_on_request(sweep):
    """``round_out`` stores exactly the TF32 rounding (cvt.rna) of what the kernel stores without it."""
    from oracle.sweep_check import on_grid, rna

    gen = torch.Generator().manual_seed(41 + sweep)
    rows, C, B, T, heads = 24, 48, 2, 12, 4
    r = lambda *s: torch.randn(*s, generator=gen).to(DEV)  # noqa: E731
    x, a1, a2, a3, g, b, vg, vb = r(rows, C), r(rows, C), r(rows, C), r(rows, C), 1 + 0.1 * r(C), r(C), r(C), r(C)
    stats = torch.empty(rows, 2, device=DEV)
    E.token_layernorm(0, x, g, b, stats)
    kw = dict(in1=a1, in2=a2, in3=a3, v_gamma=vg, v_beta=vb)
    plain = E.token_layernorm(sweep, x, g, b, stats, **kw)
    rounded = E.token_layernorm(sweep, x, g, b, stats, round_out=True, **kw)
    assert not on_grid(plain.cpu()) and torch.equal(rounded.cpu().double(), rna(plain.cpu().double()))
    qkv, qkvd, dO, dOd = r(B * T, 3 * C), r(B * T, 3 * C), r(B * T, C), r(B * T, C)
    P, Pd = torch.empty(B, heads, T, T, device=DEV), torch.empty(B, heads, T, T, device=DEV)
    E.token_attention(0, qkv, B, T, heads, P, Pd)
    E.token_attention(2, qkv, B, T, heads, P, Pd, in1=qkvd)
    ins = {0: {}, 1: dict(in1=dO), 2: dict(in1=qkvd), 3: dict(in1=dOd, in2=dO, in3=qkvd)}[sweep]
    Pk, Pdk = P.clone(), Pd.clone()   # sweeps 0 / 2 rewrite P / P'; the same values either way
    plain = E.token_attention(sweep, qkv, B, T, heads, P, Pd, **ins)
    rounded = E.token_attention(sweep, qkv, B, T, heads, Pk, Pdk, round_out=True, **ins)
    assert not on_grid(plain.cpu()) and torch.equal(rounded.cpu().double(), rna(plain.cpu().double()))


@pytest.mark.parametrize("backend", ["simt", "tc"])
def test_transformer_closure_on_the_engine_matches_reference_tag_fixture(backend):
    """BASELINE config 5 in miniature on the CUDA engine: the layer program of ``compiler.compile_transformer`` (positional
    embedding, QKV / output / feed-forward / decoder GEMMs, multi-head attention, LayerNorm, residuals, next-token
    cross-entropy with the joint attacker's soft labels) through all four sweeps -- objective value, gradient w.r.t. the
    candidate embeddings and w.r.t. the label logits against the *reference's* TAG closure (tag.yaml)."""
    import os
    import sys

    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from helpers import case_from_fixture, cfg_from_fixture, load_golden
    from breaching_b200 import compiler

    fx = load_golden("trial_joint_tag_transformer.pt")
    model, loss_fn, payload, shared, true = case_from_fixture(fx)
    cfg = cfg_from_fixture(fx)
    names = [n for n, _ in model.named_parameters()]
    grads = list(shared[0]["gradients"])
    grads.pop(names.index("encoder.weight"))                       # base_attack.py:88-95
    params = [p.detach() for n, p in model.named_parameters() if n != "encoder.weight"]
    B, T, d = fx["x0"].shape
    V = fx["l0"].shape[-1]
    prog = compiler.compile_transformer(model, B, T)
    eng = E.Engine(None, (B * T, d, 1, 1), cfg, DEV, backend=backend, program=prog)
    eng.load_model(params=params)
    L = len(grads)
    tag_weights = torch.arange(L, 0, -1, dtype=torch.float32) / L  # objectives.py:115-124, scale_scheme linear
    eng.load_targets([g.to(DEV) for g in grads], torch.zeros(B * T, dtype=torch.long), tensor_weights=tag_weights)
    q = fx["l0"].to(DEV).softmax(dim=-1)
    eng.load_soft_labels(q.reshape(B * T, V))
    val, gx = eng.objective_and_gradient(fx["x0"].to(DEV).reshape(B * T, d, 1, 1))
    gq = eng.label_gradient((B, T, V))
    gl = q * (gq - (q * gq).sum(dim=-1, keepdim=True))
    tol_v, tol_g = (2e-4, 2e-3) if backend == "simt" else (5e-3, 3e-2)
    assert abs(val - fx["objective0"]) < tol_v * abs(fx["objective0"]), (val, fx["objective0"], eng.last_terms())
    assert _relerr(gx.reshape(B, T, d), fx["raw_grad_x0"]) < tol_g, _relerr(gx.reshape(B, T, d), fx["raw_grad_x0"])
    assert _relerr(gl, fx["raw_grad_l0"]) < tol_g, _relerr(gl, fx["raw_grad_l0"])
    eng.close()


def test_tag_attack_through_the_attacker_api():
    """tag.yaml end to end (prologue in embedding space, joint loop with AdamW / clip / warm-up, scoring, token recovery)
    against the reference trajectory of the miniature config-5 fixture."""
    import copy
    import math
    import os
    import sys

    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from helpers import case_from_fixture, cfg_from_fixture, load_golden
    from breaching_b200.attacks import prepare_attack

    fx = load_golden("trial_joint_tag_transformer.pt")
    model, loss_fn, payload, shared, true = case_from_fixture(fx)
    cfg = cfg_from_fixture(fx)
    attacker = prepare_attack(model, loss_fn, cfg, dict(device=DEV, dtype=torch.float, backend="simt"))
    assert type(attacker).__name__ == "OptimizationJointAttacker"
    rec_models, template, stats, shared2 = attacker._prepare_text(payload, copy.deepcopy(shared))
    engine = attacker._get_text_engine(rec_models, shared2)
    best, best_l = attacker._run_joint_trial(engine, fx["x0"].to(DEV), fx["l0"].to(DEV), stats, 0, iterations=fx["iters"])
    for a, b in zip(stats["Trial_0_Val"], fx["history"]):
        assert math.isclose(a, b, rel_tol=2e-3, abs_tol=1e-5), (stats["Trial_0_Val"], fx["history"])
    cfg.optim.max_iterations = 3
    rec, st = prepare_attack(model, loss_fn, cfg, dict(device=DEV, dtype=torch.float)).reconstruct(payload, copy.deepcopy(shared), {})
    assert rec["data"].shape == true["data"].shape and rec["data"].dtype == torch.long and "raw_embeddings" in rec


@pytest.mark.parametrize("backend", ["simt", "tc"])
def test_full_size_config5_closure_on_the_engine(backend):
    """BASELINE config 5 at full size (50 257 tokens, 96 dims, 8 heads, 3 layers, 32 positions) on the CUDA engine against the
    closure of the reference's TAG attacker (tests/golden/trial_joint_tag_config5.pt)."""
    import os
    import sys

    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from helpers import case_from_fixture, cfg_from_fixture, load_golden
    from breaching_b200 import compiler

    fx = load_golden("trial_joint_tag_config5.pt")
    gen = torch.Generator().manual_seed(fx["l0_seed"])
    x0 = torch.randn(list(fx["x0"].shape), generator=gen)
    l0 = torch.randn([1, 32, fx["case"]["ntokens"]], generator=gen)
    assert torch.equal(x0, fx["x0"])
    model, loss_fn, payload, shared, true = case_from_fixture(fx)
    cfg = cfg_from_fixture(fx)
    names = [n for n, _ in model.named_parameters()]
    grads = list(shared[0]["gradients"])
    grads.pop(names.index("encoder.weight"))
    params = [p.detach() for n, p in model.named_parameters() if n != "encoder.weight"]
    B, T, d = x0.shape
    V = l0.shape[-1]
    eng = E.Engine(None, (B * T, d, 1, 1), cfg, DEV, backend=backend, program=compiler.compile_transformer(model, B, T))
    eng.load_model(params=params)
    L = len(grads)
    eng.load_targets([g.to(DEV) for g in grads], torch.zeros(B * T, dtype=torch.long),
                     tensor_weights=torch.arange(L, 0, -1, dtype=torch.float32) / L)
    q = l0.to(DEV).softmax(dim=-1)
    eng.load_soft_labels(q.reshape(B * T, V))
    val, gx = eng.objective_and_gradient(x0.to(DEV).reshape(B * T, d, 1, 1))
    gq = eng.label_gradient((B, T, V))
    gl = q * (gq - (q * gq).sum(dim=-1, keepdim=True))
    tol_v, tol_g = (2e-4, 2e-3) if backend == "simt" else (5e-3, 3e-2)
    assert abs(val - fx["objective0"]) < tol_v * abs(fx["objective0"]), (val, fx["objective0"], eng.last_terms())
    assert _relerr(gx.reshape(B, T, d), fx["raw_grad_x0"]) < tol_g
    assert _relerr(gl[:, :, ::97], fx["raw_grad_l0_sample"]) < tol_g
    assert abs(float(gl.norm()) - fx["raw_grad_l0_norm"]) < tol_g * fx["raw_grad_l0_norm"]
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("rows,d,V,limited", [(32, 96, 50257, False), (7, 16, 50, False), (40, 96, 3000, True)])
def test_token_recovery_kernel_matches_the_reference_formula(rows, d, V, limited):
    """bre_token_match against `_postprocess_text_data._max_similarity` (base_attack.py:126-133, squared norms) in float64; half of
    the rows are exact vocabulary entries plus noise (the case the attack cares about), the rest random."""
    from breaching_b200 import engine as E
    from breaching_b200.attacks import host

    dev = torch.device("cuda:0")
    g = torch.Generator(device="cpu").manual_seed(rows * 7 + V)
    emb = torch.randn(V, d, generator=g)
    picks = torch.randint(0, V, (rows,), generator=g)
    rec = torch.randn(rows, d, generator=g)
    rec[::2] = emb[picks[::2]] + 0.05 * torch.randn(len(picks[::2]), d, generator=g)
    subset = torch.unique(torch.cat([picks, torch.randint(0, V, (200,), generator=g)])) if limited else None

    def scores(r, e):
        r = r.double() - r.double().mean(dim=-1, keepdim=True)
        e = e.double() - e.double().mean(dim=-1, keepdim=True)
        return r @ e.T / r.pow(2).sum(-1)[:, None] / e.pow(2).sum(-1)[None, :]

    want = scores(rec, emb if subset is None else emb[subset])
    got = E.token_match(rec.to(dev), emb.to(dev), None if subset is None else subset.to(dev)).cpu()
    assert got.dtype == torch.int64 and got.shape == (rows,)
    best = want.max(dim=1)[0]
    chosen = want[torch.arange(rows), got]
    assert torch.all(chosen >= best - 1e-6 * best.abs().clamp_min(1e-12)), (chosen, best)
    if subset is None and d >= 64:
        assert torch.equal(got[::2], picks[::2])                      # the noisy vocabulary entries are found again
    # the host-side dispatch (attacks/host.py) gives the same tokens on device tensors as its formula does on host tensors
    dev_tokens = host._max_similarity(rec.to(dev), emb.to(dev), None if subset is None else subset.to(dev)).cpu()
    cpu_tokens = host._max_similarity(rec, emb, subset)
    assert torch.equal(dev_tokens, got)
    agree = (dev_tokens == cpu_tokens).float().mean().item()
    assert agree >= 0.95, agree                                       # fp32 near-ties of the random half may flip
