"""Every buffer of the four sweeps of one engine evaluation against a float64 restatement of its own op, computed from the
engine's own inputs to that op (oracle/sweep_check.py), on both GEMM back ends.  Each kernel is judged alone, against
rounding-error bounds derived per element, so an error confined to one BN layer, one pooling op, one residual accumulation or
one GEMM epilogue is reported at that op."""
import copy
import os
import resource
import sys
import time

import pytest
import torch

pytestmark = pytest.mark.gpu

from breaching_b200 import compiler as C  # noqa: E402
from breaching_b200 import get_attack_config, synthetic  # noqa: E402
from breaching_b200.engine import Engine  # noqa: E402
from helpers import EngineSource, masked_targets, odd_case, sweep_objective, tensor_weights  # noqa: E402
from oracle.sweep_check import SweepChecker, SweepCheckError  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "scripts")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

DEV = torch.device("cuda:0")
KINDS = ["euclidean", "l1", "tag-euclidean", "cosine-similarity", "angular", "fast-cosine-similarity", "masked-cosine-similarity"]


def build_case(name):
    """(model, input shape, labels, target gradients, attack config, feature targets or None)."""
    cfg = get_attack_config("invertinggradients")
    feats = None
    if name == "odd":
        model, shape, labels, grads = odd_case()
        return model, shape, labels, grads, cfg, None
    size, data, no_buffers, arch = 64, "imagenet", False, name
    if name in ("convnet-tiny", "linear", "trainbn-convnet-tiny"):
        size, data = 32, "cifar"
    if name.startswith("trainbn-"):
        no_buffers, arch = True, name[len("trainbn-"):]
    if name.startswith("priors"):   # "priors" or "priors:<objective>[:<tag scale scheme>]"
        arch = "resnet18"
        over = {"objective.task_regularization": 0.1, "regularization.norm.scale": 1e-3, "regularization.deep_inversion.scale": 1e-3,
                "regularization.features.scale": 0.1}
        parts = name.split(":")[1:]
        if parts:
            over["objective.type"] = parts[0]
        if len(parts) > 1:
            over["objective.scale_scheme"] = parts[1]
        cfg = get_attack_config("invertinggradients", over)
        feats = torch.randn(2, 512, generator=torch.Generator().manual_seed(2))
    if name == "linear":
        cfg = get_attack_config("invertinggradients", {"regularization.norm.scale": 1e-2})
    model, _, _, shared, true = synthetic.make_case(arch, data, batch=2, seed=17, bn_random=True, image_size=size, classes=10,
                                                    no_buffers=no_buffers)
    if not no_buffers:
        model.eval()
    grads = shared[0]["gradients"]
    if cfg.objective.type == "masked-cosine-similarity":
        grads = masked_targets(grads)
    return model, (2, 3, size, size), true["labels"], grads, cfg, feats


def make_engine(model, shape, cfg, labels, grads, backend, feats=None, options=()):
    eng = Engine(copy.deepcopy(model).to(DEV), shape, cfg, DEV, backend=backend)
    for k, v in options:
        eng.set_option(k, v)
    eng.load_model()
    eng.load_targets([g.to(DEV) for g in grads], labels.to(DEV), tensor_weights=tensor_weights(cfg, len(grads)))
    if feats is not None:
        eng.load_feature_targets(feats.to(DEV))
    return eng


def candidate(shape, seed=4):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed))


def check_evaluation(eng, x, model, grads, labels, cfg, feats, label):
    """Evaluate at ``x`` and check every buffer of the four sweeps, every objective term and the returned objective, then the
    euclidean and cosine scores at ``x``."""
    value, _ = eng.objective_and_gradient(x.to(DEV))
    terms = eng.last_terms()
    bn = [None if m is None or m.running_mean is None else (m.running_mean.double(), m.running_var.double())
          for m in C.bn_modules(model, eng.prog)]
    src = EngineSource(eng)
    chk = SweepChecker(eng.prog, list(model.parameters()), bn, grads, labels, sweep_objective(cfg, feats), src)
    chk.fused = [i for i in range(len(eng.prog.ops)) if eng.debug_op(i)["fused"]]
    chk.stem = sorted(src.stem)
    try:
        chk.check(raise_on_failure=False)
        chk.check_terms(terms, value, raise_on_failure=False)
        for kind in ("euclidean", "cosine-similarity"):
            chk.check_score(eng.score(x.to(DEV), kind), kind, raise_on_failure=False)
        if chk.findings:
            raise SweepCheckError("\n".join(repr(f) for f in chk.findings[:20]))
    finally:
        # largest error / bound ratio per op kind and sweep (headroom of the bounds)
        print(f"\n[{label}] " + ", ".join(f"{k}/{s}: {r:.3g}" for (k, s), r in sorted(chk.ratios.items())) +
              f"; tensor-core ops reading an off-grid activation: {sorted(chk.off_grid)}; fused BN ops: {chk.fused}; stem columns: {chk.stem}")
    # the activations of tensor-core GEMMs are stored on the TF32 grid, except the pooling outputs (not rounded on store)
    assert chk.off_grid <= pool_fed(eng.prog), sorted(chk.off_grid)
    return chk


def pool_fed(prog):
    """The conv / linear ops whose input is a max-pool or average-pool output."""
    pooled = {op.tout for op in prog.ops if op.kind in (C.OP_MAXPOOL, C.OP_AVGPOOL)}
    return {i for i, op in enumerate(prog.ops) if op.kind in (C.OP_CONV, C.OP_LINEAR) and op.tin in pooled}


def check_engine(name, backend, options=(), env=None, monkeypatch=None):
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    model, shape, labels, grads, cfg, feats = build_case(name)
    eng = make_engine(model, shape, cfg, labels, grads, backend, feats, options)
    try:
        return check_evaluation(eng, candidate(shape), model, grads, labels, cfg, feats, f"{name} / {backend} {dict(options)} {env or ''}")
    finally:
        eng.close()


CASES = ["convnet-tiny", "resnet18", "resnet50", "trainbn-convnet-tiny", "trainbn-resnet18", "linear", "odd", "priors"]


@pytest.mark.parametrize("backend", ["simt", "tc"])
@pytest.mark.parametrize("name", CASES)
def test_every_sweep_buffer_is_locally_exact(name, backend, monkeypatch):
    chk = check_engine(name, backend, monkeypatch=monkeypatch)
    if name == "odd":   # the case exists to reach these: BN / ReLU / add ops accumulating into an input / residual delta,
        ops, tens = chk.prog.ops, chk.prog.tensors   # with scalar (C % 4 != 0) and float4 (C % 4 == 0) kernels
        reached = {(f, tens[op.tout].C % 4 == 0) for op in ops if op.kind == C.OP_BNACT for f in ("in", "res") if getattr(op, f"acc_{f}")}
        assert reached == {("in", False), ("in", True), ("res", False), ("res", True)}, reached
    if backend == "tc" and name in ("resnet18", "resnet50", "priors"):
        assert chk.stem == [0]


@pytest.mark.parametrize("backend", ["simt", "tc"])
@pytest.mark.parametrize("kind", KINDS + ["tag-euclidean:exp"])
def test_every_objective_is_locally_exact(kind, backend, monkeypatch):
    """The seven matching objectives on ResNet-18 64 x 64 with every prior and task regularisation: the direction v, every buffer
    it feeds and the terms.  tag-euclidean gets the attack's per-tensor weights (linear and exp); masked-cosine's targets sit on
    both sides of the mask threshold and fill whole masked chunks."""
    chk = check_engine(f"priors:{kind}", backend, monkeypatch=monkeypatch)
    assert ("objective", "V") in chk.ratios and ("terms", "match") in chk.ratios


def test_stem_without_column_path(monkeypatch):
    assert check_engine("resnet18", "tc", env={"BRE_STEM_COLS": "0"}, monkeypatch=monkeypatch).stem == []


def test_precise_first_layers(monkeypatch):
    assert check_engine("resnet18", "tc", options=(("precise_first", 2),), monkeypatch=monkeypatch).stem == []


def test_in_kernel_bn_gradient_reduction(monkeypatch):
    """BRE_DEFER_BN=0: the BN gamma / beta gradients reduced inside the backward kernels, and every sweep after them."""
    check_engine("resnet18", "tc", env={"BRE_DEFER_BN": "0"}, monkeypatch=monkeypatch)


def test_fused_bn_epilogue(monkeypatch):
    """fuse_bnact: the conv + BN pair of the tensor-core epilogue is checked as one op where the pre-BN tangent is not stored."""
    chk = check_engine("resnet18", "tc", options=(("fuse_bnact", 1),), monkeypatch=monkeypatch)
    assert chk.fused and set(chk.src.unwritten) <= {chk.prog.ops[i].tin for i in chk.fused}


def test_tf32_direction_shadow_is_what_the_gemms_read():
    """debug_param("v_operand") is the TF32 shadow for tensor-core weights and the fp32 arena elsewhere."""
    model, shape, labels, grads, cfg, feats = build_case("resnet18")
    eng = make_engine(model, shape, cfg, labels, grads, "tc")
    eng.objective_and_gradient(candidate(shape).to(DEV))
    from oracle.sweep_check import on_grid, rna

    shadowed = 0
    for j in range(len(eng.prog.params)):
        w, wo = eng.debug_param("W", j), eng.debug_param("W_operand", j)
        vo = eng.debug_param("v_operand", j)
        if torch.equal(wo, w):
            continue
        shadowed += 1
        assert torch.equal(wo.double(), rna(w.double())) and on_grid(vo), j
    assert shadowed > 0
    eng.close()


# ---- the benchmarked workloads at full size ------------------------------------------------------------------------------------
def covered_plans(prog):
    """(mode, tile rows, tile width, split, ring depth, per parity class) of every tensor-core GEMM launch of one evaluation, by the
    launch rules of csrc/igemm_tc.cu as scripts/profile_gemms.py restates them."""
    import bench
    from profile_gemms import ring_plan, split_plan

    plans = set()
    for o in bench.gemm_ops(prog, "tc"):
        g = o["geom"]
        rows = [(0, 1), (2, 1)] + ([(0, 1)] if o["first"] else [(1, 1), (0, 2)]) + [(1, 2)]
        for mode, nsrc in rows:
            _, bn, splits, _ = split_plan(mode, g, nsrc)
            bm, depth = ring_plan(mode, g, nsrc)
            plans.add((("fprop", "dgrad", "wgrad")[mode], bm, bn, splits, depth, mode == 1 and g[6] == 2))
    return plans


@pytest.mark.parametrize("at", ["randn", "warm"])
@pytest.mark.parametrize("backend", ["simt", "tc"])
@pytest.mark.parametrize("config", [1, 2, 3])
def test_benchmark_config_at_full_size(config, backend, at):
    """BASELINE configs 1-3 built exactly as bench.py builds them (the shared BN buffers copied into the model for config 3), at a
    seeded randn candidate and at the candidate after 4 trial iterations (boxed and sign-stepped: pixels on the box faces, TV
    differences exactly zero)."""
    import bench

    t0 = time.time()
    case = bench.build_case(config)
    model, _, payload, shared, true, cfg = case
    m = copy.deepcopy(model)
    if shared[0]["buffers"] is not None:
        for buf, src in zip(m.buffers(), shared[0]["buffers"]):
            buf.data.copy_(src)
    m.eval()
    runner = bench.EngineRunner(config, case, DEV, backend, 0)
    shape = bench.candidate_shape(config, payload, shared)
    plans = covered_plans(runner.prog)
    try:
        if at == "warm":
            runner.warm(4)
            x = runner.eng.candidate().cpu()
        else:
            x = candidate(shape, seed=config)
        check_evaluation(runner.eng, x, m, shared[0]["gradients"], true["labels"], cfg, None, f"config {config} / {backend} / {at}")
    finally:
        runner.eng.close()
        print(f"config {config} / {backend} / {at}: {time.time() - t0:.1f} s, peak host RSS of the process "
              f"{resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2 ** 20:.2f} GB; tensor-core launch plans "
              f"(mode, rows, width, split, ring, parity classes): {sorted(plans)}")
    if at == "warm" and cfg.optim.get("boxed", False):   # the sign(0) paths: pixels on the box faces
        assert int((x == x.amax()).sum()) > 1 or int((x == x.amin()).sum()) > 1
    if config == 2:
        assert any(p[1] == 64 and p[4] == 8 for p in plans), plans
        assert any(p[1] == 128 and p[2] == 32 and p[3] == 8 for p in plans), plans
