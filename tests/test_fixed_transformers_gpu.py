"""The reference's fixed-position transformers on the GPU: the cluster-split attention kernel (heads wider than one CTA's shared
memory: transformer1's one head of 200, transformerS's one head of 512) in all four sweeps, and the constant positional add of
transformer3f / transformer1 / transformerS through the engine's sweeps, the attacker and full-size reconstructions."""
import copy
import math
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from breaching_b200 import compiler, synthetic  # noqa: E402
from breaching_b200 import engine as E  # noqa: E402
from helpers import EngineSource, cfg_from_fixture, load_golden, sweep_objective  # noqa: E402
from oracle.sweep_check import SweepChecker  # noqa: E402

DEV = torch.device("cuda:0")
FIXTURES = ["transformer3f", "transformer1", "transformerS"]


def _relerr(a, b):
    return ((a.double().cpu() - b.double().cpu()).norm() / (b.double().cpu().norm() + 1e-30)).item()


def _attention_case(B, T, heads, dh, seed):
    """Random operands and the float64 statement of the four sweeps (as test_tokens_gpu.py states them)."""
    gen = torch.Generator().manual_seed(seed)
    d = heads * dh
    r = lambda *s: torch.randn(*s, generator=gen, dtype=torch.double)  # noqa: E731
    qkv, qkvd, dO, dOd = r(B * T, 3 * d), r(B * T, 3 * d), r(B * T, d), r(B * T, d)
    hs = lambda t: t.view(B, T, heads, dh).transpose(1, 2)  # noqa: E731
    merge = lambda t: t.transpose(1, 2).reshape(B * T, d)  # noqa: E731
    Q, K, V = (hs(t) for t in qkv.split(d, dim=1))
    Qd, Kd, Vd = (hs(t) for t in qkvd.split(d, dim=1))
    s = 1.0 / dh ** 0.5
    P = torch.softmax(Q @ K.transpose(-1, -2) * s, dim=-1)
    dOh, dOdh = hs(dO), hs(dOd)
    dP = dOh @ V.transpose(-1, -2)
    rr = (dP * P).sum(-1, keepdim=True)
    dS = P * (dP - rr)
    Sd = (Qd @ K.transpose(-1, -2) + Q @ Kd.transpose(-1, -2)) * s
    Pd = P * (Sd - (P * Sd).sum(-1, keepdim=True))
    dPd = dOdh @ V.transpose(-1, -2) + dOh @ Vd.transpose(-1, -2)
    rd = (dPd * P + dP * Pd).sum(-1, keepdim=True)
    dSd = Pd * (dP - rr) + P * (dPd - rd)
    want = {
        0: merge(P @ V),
        1: torch.cat([merge(dS @ K * s), merge(dS.transpose(-1, -2) @ Q * s), merge(P.transpose(-1, -2) @ dOh)], dim=1),
        2: merge(Pd @ V + P @ Vd),
        3: torch.cat([merge((dSd @ K + dS @ Kd) * s), merge((dSd.transpose(-1, -2) @ Q + dS.transpose(-1, -2) @ Qd) * s),
                      merge(Pd.transpose(-1, -2) @ dOh + P.transpose(-1, -2) @ dOdh)], dim=1),
    }
    f = lambda v: v.float().to(DEV).contiguous()  # noqa: E731
    ins = {0: {}, 1: dict(in1=f(dO)), 2: dict(in1=f(qkvd)), 3: dict(in1=f(dOd), in2=f(dO), in3=f(qkvd))}
    return f(qkv), ins, want, P, Pd


def _run_sweeps(B, T, heads, qkv, ins, cluster, round_out=False):
    Pg, Pdg = torch.empty(B, heads, T, T, device=DEV), torch.empty(B, heads, T, T, device=DEV)
    outs = {}
    for sweep in (0, 1, 2, 3):
        outs[sweep] = E.token_attention(sweep, qkv, B, T, heads, Pg, Pdg, round_out=round_out, cluster=cluster, **ins[sweep])
        if sweep == 0:
            outs["P"] = Pg.clone()
        if sweep == 2:
            outs["Pd"] = Pdg.clone()
    return outs


CLUSTER_SHAPES = [(1, 32, 1, 200, c) for c in (2, 4, 8)] + [(1, 16, 1, 512, c) for c in (2, 4, 8)] + \
                 [(1, 32, 1, 512, c) for c in (4, 8)] + [(1, 32, 8, 12, c) for c in (2, 4)] + \
                 [(2, 8, 2, 30, 4), (1, 32, 1, 200, 3)]   # the last CTA takes the remainder: 30 = 3 x 8 + 6, 200 = 2 x 67 + 66


@pytest.mark.parametrize("B,T,heads,dh,c", CLUSTER_SHAPES)
def test_cluster_attention_four_sweeps(B, T, heads, dh, c):
    qkv, ins, want, P, Pd = _attention_case(B, T, heads, dh, seed=T * 1000 + dh * 10 + c)
    assert E.token_attention_plan(T, dh, c) == c
    out = _run_sweeps(B, T, heads, qkv, ins, c)
    assert _relerr(out[0], want[0]) < 1e-5 and _relerr(out["P"], P) < 1e-5
    assert _relerr(out[1], want[1]) < 2e-5
    assert _relerr(out[2], want[2]) < 2e-5 and _relerr(out["Pd"], Pd) < 2e-5
    assert _relerr(out[3], want[3]) < 5e-5


@pytest.mark.parametrize("B,T,heads,dh", [(1, 32, 8, 12), (2, 16, 2, 40), (1, 32, 1, 64)])
def test_forced_clusters_agree_with_the_resident_kernel(B, T, heads, dh):
    qkv, ins, _, _, _ = _attention_case(B, T, heads, dh, seed=7 + dh)
    resident = _run_sweeps(B, T, heads, qkv, ins, 1)
    for c in (2, 4):
        split = _run_sweeps(B, T, heads, qkv, ins, c)
        for k in resident:
            assert _relerr(split[k], resident[k]) < 3e-6, (c, k, _relerr(split[k], resident[k]))


def test_cluster_attention_is_deterministic_and_rounds_on_request():
    from oracle.sweep_check import on_grid, rna

    B, T, heads, dh = 1, 32, 1, 200
    qkv, ins, _, _, _ = _attention_case(B, T, heads, dh, seed=99)
    a, b = _run_sweeps(B, T, heads, qkv, ins, 0), _run_sweeps(B, T, heads, qkv, ins, 0)
    assert all(torch.equal(a[k], b[k]) for k in a)
    rounded = _run_sweeps(B, T, heads, qkv, ins, 0, round_out=True)
    for sweep in (0, 1, 2, 3):
        assert not on_grid(a[sweep].cpu()) and torch.equal(rounded[sweep].cpu().double(), rna(a[sweep].cpu().double()))


def test_attention_dispatch_and_refusal():
    assert E.token_attention_plan(32, 12) == 1               # transformer3 / transformer3f: the resident kernel, as before
    assert E.token_attention_plan(32, 200) == 2              # transformer1
    assert E.token_attention_plan(16, 512) == 2              # transformerS at T = 16
    assert E.token_attention_plan(32, 512) == 3              # transformerS at T = 32: smallest cluster whose slices fit
    assert E.token_attention_plan(128, 12) is None           # the T^2 working set alone is over the limit
    assert E.token_attention_plan(32, 200, 1) is None        # forced resident kernel that does not fit
    qkv = torch.randn(32, 3 * 200, device=DEV)
    P = torch.empty(1, 1, 32, 32, device=DEV)
    with pytest.raises(E.EngineError, match="221184 B of shared memory"):
        E.token_attention(0, qkv, 1, 32, 1, P, P, cluster=1)
    qkv = torch.randn(128, 3 * 24, device=DEV)
    P = torch.empty(1, 2, 128, 128, device=DEV)
    with pytest.raises(E.EngineError, match="311296 B of shared memory.*per CTA"):
        E.token_attention(0, qkv, 1, 128, 2, P, P)


# ---- the constant positional add through the engine ------------------------------------------------------------------------
def _fixture_case(name):
    fx = load_golden("fixed_transformers.pt")[name]
    model, loss_fn, payload, shared, true = synthetic.make_text_case(**fx["case"])
    checksum = float(sum(p.detach().double().sum() for p in model.parameters()))
    assert abs(checksum - fx["weight_checksum"]) <= 1e-6 * max(1.0, abs(fx["weight_checksum"]))
    names = [n for n, _ in model.named_parameters()]
    grads = list(shared[0]["gradients"])
    grads.pop(names.index("encoder.weight"))
    params = [p.detach() for n, p in model.named_parameters() if n != "encoder.weight"]
    return fx, model, loss_fn, payload, shared, grads, params


def _engine(model, B, T, cfg, grads, params, backend):
    d = model.decoder.in_features
    prog = compiler.compile_transformer(model, B, T)
    eng = E.Engine(None, (B * T, d, 1, 1), cfg, DEV, backend=backend, program=prog)
    eng.load_model(params=params)
    L = len(grads)
    eng.load_targets([g.to(DEV) for g in grads], torch.zeros(B * T, dtype=torch.long),
                     tensor_weights=torch.arange(L, 0, -1, dtype=torch.float32) / L)
    return eng, prog


@pytest.mark.parametrize("backend", ["simt", "tc"])
@pytest.mark.parametrize("name", FIXTURES)
def test_closure_matches_the_reference_fixture(name, backend):
    fx, model, _, _, _, grads, params = _fixture_case(name)
    cfg = cfg_from_fixture(fx)
    B, T, d = fx["x0"].shape
    V = fx["l0"].shape[-1]
    eng, _ = _engine(model, B, T, cfg, grads, params, backend)
    try:
        q = fx["l0"].to(DEV).softmax(dim=-1)
        eng.load_soft_labels(q.reshape(B * T, V))
        val, gx = eng.objective_and_gradient(fx["x0"].to(DEV).reshape(B * T, d, 1, 1))
        gq = eng.label_gradient((B, T, V))
        gl = q * (gq - (q * gq).sum(dim=-1, keepdim=True))
        tol_v, tol_g = (2e-4, 2e-3) if backend == "simt" else (5e-3, 3e-2)
        assert abs(val - fx["objective0"]) < tol_v * abs(fx["objective0"]), (val, fx["objective0"])
        assert _relerr(gx.reshape(B, T, d), fx["raw_grad_x0"]) < tol_g, _relerr(gx.reshape(B, T, d), fx["raw_grad_x0"])
        assert _relerr(gl, fx["raw_grad_l0"]) < tol_g, _relerr(gl, fx["raw_grad_l0"])
    finally:
        eng.close()


class FixedPositionChecker(SweepChecker):
    """SweepChecker plus the constant positional add: F adds the table, B and TB pass the delta to the candidate unchanged, TF
    stores the candidate's zero tangent."""

    def forward(self):
        super().forward()
        for i, op in enumerate(self.prog.ops):
            if op.kind == compiler.OP_POSCONST:
                x, y = self.T("val", op.tin), self.T("val", op.tout)
                pos = self._pos_rows(op.table.double(), x)
                ref = x + pos
                self._cmp(i, "F", f"val[t{op.tout}]", y, ref, 2 * 2.0 ** -24 * (x.abs() + pos.abs()) + self._rounded(y, ref))

    def _reverse(self, sweep):
        contrib = super()._reverse(sweep)
        for i, op in enumerate(self.prog.ops):
            if op.kind == compiler.OP_POSCONST:
                dout = self.T("tangent_delta" if sweep == "TB" else "delta", op.tout)
                contrib.setdefault(op.tin, []).append((i, dout, 0.0, dout.abs()))
        return contrib

    def tangent_forward(self):
        super().tangent_forward()
        for i, op in enumerate(self.prog.ops):
            if op.kind == compiler.OP_POSCONST:
                y = self.T("tangent", op.tout)
                self._cmp(i, "TF", f"tangent[t{op.tout}]", y, torch.zeros_like(y), 0.0)


@pytest.mark.parametrize("backend", ["simt", "tc"])
@pytest.mark.parametrize("name", FIXTURES)
def test_every_sweep_buffer_is_locally_exact(name, backend):
    fx, model, _, _, _, grads, params = _fixture_case(name)
    cfg = cfg_from_fixture(fx)
    B, T = fx["case"]["batch"], fx["case"]["seq_len"]
    d, V = model.decoder.in_features, model.decoder.out_features
    eng, prog = _engine(model, B, T, cfg, grads, params, backend)
    try:
        gen = torch.Generator().manual_seed(29)
        x = torch.randn(B * T, d, 1, 1, generator=gen)
        q = torch.randn(B * T, V, generator=gen).softmax(dim=-1)
        eng.load_soft_labels(q.to(DEV))
        eng.objective_and_gradient(x.to(DEV))
        lg = eng.label_gradient((B * T, V)).cpu()
        chk = FixedPositionChecker(prog, params, [None] * len(prog.ops), grads, q, sweep_objective(cfg), EngineSource(eng))
        chk.check(raise_on_failure=False)
        chk.check_label_gradient(lg, raise_on_failure=False)
    finally:
        eng.close()
    assert not chk.findings, "\n".join(repr(f) for f in chk.findings[:20])
    kinds = {k for k, _ in chk.ratios}
    assert {"posconst", "layernorm", "attention", "linear", "bnact", "label"} <= kinds and "posadd" not in kinds
    assert {("posconst", "F"), ("posconst", "TF")} <= set(chk.ratios)
    if backend == "tc":
        assert chk.off_grid == set()


@pytest.mark.parametrize("name", FIXTURES)
def test_trajectory_matches_the_reference_and_the_graph_equals_eager(name):
    from breaching_b200.attacks import prepare_attack

    fx, model, loss_fn, payload, shared, _, _ = _fixture_case(name)
    cfg = cfg_from_fixture(fx)
    attacker = prepare_attack(model, loss_fn, cfg, dict(device=DEV, dtype=torch.float, backend="simt"))
    rec_models, template, stats, shared2 = attacker._prepare_text(payload, copy.deepcopy(shared))
    engine = attacker._get_text_engine(rec_models, shared2)
    attacker._run_joint_trial(engine, fx["x0"].to(DEV), fx["l0"].to(DEV), stats, 0, iterations=fx["iters"])
    for a, b in zip(stats["Trial_0_Val"], fx["history"]):
        assert math.isclose(a, b, rel_tol=2e-3, abs_tol=1e-5), (stats["Trial_0_Val"], fx["history"])
    assert len(stats["Trial_0_Val"]) == fx["iters"]
    # the captured iteration and the eager one compute the same bits
    B, T, d = fx["x0"].shape
    runs = []
    for graph in (1, 0):
        engine.set_option("use_graph", graph)
        engine.begin_joint_trial(fx["x0"].reshape(B * T, d, 1, 1), fx["l0"], fx["lrs"])
        engine.run(fx["iters"])
        engine.sync()
        runs.append((engine.history(), engine.best().cpu(), engine.joint_labels().cpu()))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1]) and torch.equal(runs[0][2], runs[1][2])
    engine.close()


@pytest.mark.parametrize("preset", ["transformer3f", "transformer1", "transformerS"])
def test_full_size_reconstruct_returns_tokens(preset):
    """The reference's presets at full size (GPT-2 vocabulary of 50 257, 32 positions, tag.yaml), a few iterations end to end."""
    from breaching_b200 import get_attack_config
    from breaching_b200.attacks import prepare_attack

    dims = {"transformer3f": (96, 8, 1536, 3), "transformer1": (200, 1, 200, 1), "transformerS": (512, 1, 512, 1)}[preset]
    model, loss_fn, payload, shared, true = synthetic.make_text_case(batch=1, seq_len=32, seed=5, ntokens=50257, ninp=dims[0],
                                                                     nhead=dims[1], nhid=dims[2], nlayers=dims[3], positional="fixed")
    cfg = get_attack_config("tag", {"optim.max_iterations": 4})
    rec, stats = prepare_attack(model, loss_fn, cfg, dict(device=DEV, dtype=torch.float)).reconstruct(payload, copy.deepcopy(shared), {})
    assert rec["data"].shape == true["data"].shape and rec["data"].dtype == torch.long
    assert int(rec["data"].min()) >= 0 and int(rec["data"].max()) < 50257
    assert all(math.isfinite(v) for v in stats["Trial_0_Val"])
