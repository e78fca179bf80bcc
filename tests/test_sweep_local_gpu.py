"""Every buffer of the four sweeps of one engine evaluation against a float64 restatement of its own op, computed from the
engine's own inputs to that op (oracle/sweep_check.py), on both GEMM back ends.  Each kernel is judged alone, against
rounding-error bounds derived per element, so an error confined to one BN layer, one pooling op, one residual accumulation or
one GEMM epilogue is reported at that op."""
import copy
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from breaching_b200 import compiler as C  # noqa: E402
from breaching_b200 import get_attack_config, synthetic  # noqa: E402
from breaching_b200.engine import Engine  # noqa: E402
from helpers import EngineSource, odd_case, sweep_objective  # noqa: E402
from oracle.sweep_check import SweepChecker  # noqa: E402

DEV = torch.device("cuda:0")


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
    if name == "priors":
        arch = "resnet18"
        cfg = get_attack_config("invertinggradients", {"objective.task_regularization": 0.1, "regularization.norm.scale": 1e-3,
                                                        "regularization.deep_inversion.scale": 1e-3,
                                                        "regularization.features.scale": 0.1})
        feats = torch.randn(2, 512, generator=torch.Generator().manual_seed(2))
    if name == "linear":
        cfg = get_attack_config("invertinggradients", {"regularization.norm.scale": 1e-2})
    model, _, _, shared, true = synthetic.make_case(arch, data, batch=2, seed=17, bn_random=True, image_size=size, classes=10,
                                                    no_buffers=no_buffers)
    if not no_buffers:
        model.eval()
    return model, (2, 3, size, size), true["labels"], shared[0]["gradients"], cfg, feats


def make_engine(model, shape, cfg, labels, grads, backend, feats=None, options=()):
    eng = Engine(copy.deepcopy(model).to(DEV), shape, cfg, DEV, backend=backend)
    for k, v in options:
        eng.set_option(k, v)
    eng.load_model()
    eng.load_targets([g.to(DEV) for g in grads], labels.to(DEV))
    if feats is not None:
        eng.load_feature_targets(feats.to(DEV))
    return eng


def candidate(shape, seed=4):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed))


def check_engine(name, backend, options=(), env=None, monkeypatch=None):
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    model, shape, labels, grads, cfg, feats = build_case(name)
    eng = make_engine(model, shape, cfg, labels, grads, backend, feats, options)
    eng.objective_and_gradient(candidate(shape).to(DEV))
    bn = [None if m is None or m.running_mean is None else (m.running_mean.double(), m.running_var.double())
          for m in C.bn_modules(model, eng.prog)]
    src = EngineSource(eng)
    chk = SweepChecker(eng.prog, list(model.parameters()), bn, grads, labels, sweep_objective(cfg, feats), src)
    chk.fused = [i for i in range(len(eng.prog.ops)) if eng.debug_op(i)["fused"]]
    chk.stem = sorted(src.stem)
    try:
        chk.check()
    finally:
        # largest error / bound ratio per op kind and sweep (headroom of the bounds)
        print(f"\n[{name} / {backend} {dict(options)} {env or ''}] " +
              ", ".join(f"{k}/{s}: {r:.3g}" for (k, s), r in sorted(chk.ratios.items())) +
              f"; tensor-core ops reading an off-grid activation: {sorted(chk.off_grid)}; fused BN ops: {chk.fused}; stem columns: {chk.stem}")
        eng.close()
    return chk


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
