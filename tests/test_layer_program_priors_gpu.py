"""Every prior on every network of tests/layer_program_cases.py, checked against float64 buffer by buffer and term by term
(oracle/sweep_check.py through test_sweep_local_gpu.check_evaluation), on both GEMM back ends: task-loss regularisation, the
features prior on the head's input (spatial heads permute the targets from CHW to HWC), the norm prior at p = 1, 2, 3 (the fused
RGB kernel or the kernel of other channel counts), TV as ``modern`` configures it on 3-channel candidates, DeepInversion on
eval-mode BN, and orthogonality on batches of two or more.  Together the cases reach the three branches of ``Engine::priors()``.

Networks local to this file reach the DeepInversion statistics paths of ``Engine::build_di_tables``: per-layer float4 and scalar
kernels in one network, and on the batched path a 320-channel layer (two finalize groups), a share clamped to the 4-block floor and
a batch-1 BN on a 1x1 map (M = 1: the variance is exactly 0).  Two of the networks go through two FedAvg local steps with
DeepInversion and task-loss regularisation, and networks that register their modules in another order than they run them are
refused the priors that would single out another layer than the reference does."""
import copy
import math

import pytest
import torch
from torch import nn

pytestmark = pytest.mark.gpu

import test_fedavg_priors_gpu as FP  # noqa: E402
from breaching_b200 import compiler as C  # noqa: E402
from breaching_b200 import get_attack_config  # noqa: E402
from breaching_b200.attacks.host import measured_features  # noqa: E402
from breaching_b200.engine import Engine, EngineError, make_cfg  # noqa: E402
from helpers import BNRegisteredLate, LinearRegisteredLast, registration_case  # noqa: E402
from layer_program_cases import CASES, build  # noqa: E402
from oracle import restate  # noqa: E402
from test_layer_programs_gpu import fedavg_case  # noqa: E402
from test_sweep_local_gpu import DEV, candidate, check_evaluation, make_engine  # noqa: E402

NUM_SMS = 132   # csrc/common.cuh kNumSMs: the batched statistics launch deals 16 blocks per SM to the BN inputs

# networks that reach the DeepInversion statistics paths: name -> (purpose, factory, input shape)
DI_NETS = {
    "di-mixed": ("a 64-channel (float4) and a 6-channel (scalar) BN: the whole network takes the per-layer statistics kernels",
                 lambda: nn.Sequential(nn.Conv2d(3, 64, 3, 1, 1), nn.BatchNorm2d(64), nn.ReLU(), nn.Conv2d(64, 6, 3, 2, 1),
                                       nn.BatchNorm2d(6), nn.ReLU(), nn.Flatten(), nn.Linear(6 * 5 * 5, 10)),
                 (2, 3, 10, 10)),
    "di-edges": ("batch 1, batched statistics: a 320-channel BN on a 32 x 32 map next to a 320-channel BN on the 1 x 1 map of the "
                 "average pool (M = 1, its share clamped to 4 blocks; 2 finalize groups each)",
                 lambda: nn.Sequential(nn.Conv2d(3, 320, 3, 1, 1), nn.BatchNorm2d(320), nn.ReLU(), nn.AdaptiveAvgPool2d(1),
                                       nn.BatchNorm2d(320), nn.Flatten(), nn.Linear(320, 10)),
                 (1, 3, 32, 32)),
}
NO_IMAGE_TERMS = "cand-co32 without image terms"
ENTRIES = list(CASES) + [NO_IMAGE_TERMS] + list(DI_NETS)
P_NORM = (1.0, 2.0, 3.0)
TV_MODERN = {"regularization.total_variation.scale": 0.1, "regularization.total_variation.inner_exp": 2,
             "regularization.total_variation.outer_exp": 0.5, "regularization.total_variation.double_opponents": True}


def build_entry(name, seed=11):
    """(model in eval mode with random BN, input shape, labels, target gradients, engine options)."""
    if name == NO_IMAGE_TERMS:
        return build("cand-co32")
    if name in CASES:
        return build(name)
    _, factory, shape = DI_NETS[name]
    torch.manual_seed(seed)
    model = factory().eval()
    gen = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, nn.BatchNorm2d):
                m.weight.copy_(1.0 + 0.2 * torch.randn(m.weight.shape, generator=gen))
                m.bias.copy_(0.1 * torch.randn(m.bias.shape, generator=gen))
                m.running_mean.copy_(0.1 * torch.randn(m.running_mean.shape, generator=gen))
                m.running_var.copy_(1.0 + 0.3 * torch.rand(m.running_var.shape, generator=gen))
    x = torch.randn(shape, generator=gen)
    y = torch.randint(0, 10, (shape[0],), generator=gen)
    grads = torch.autograd.grad(nn.functional.cross_entropy(model(x), y), list(model.parameters()))
    return model, shape, y, [g.detach() for g in grads], ()


def prior_overrides(name, prog, shape, with_di_and_features=True):
    """invertinggradients with every prior the network supports (module docstring); p of the norm prior rotates over the entries."""
    over = {"objective.task_regularization": 0.1, "regularization.total_variation.scale": 0.0}
    if name != NO_IMAGE_TERMS:
        over.update({"regularization.norm.scale": 1e-2, "regularization.norm.pnorm": P_NORM[ENTRIES.index(name) % 3]})
        if shape[1] == 3:
            over.update(TV_MODERN)
    if with_di_and_features:
        over["regularization.features.scale"] = 0.1
        if any(op.kind == C.OP_BNACT and op.has_bn and not op.bn_train for op in prog.ops):
            over["regularization.deep_inversion.scale"] = 1e-3
    if shape[0] >= 2:
        over["regularization.orthogonality.scale"] = 1.0
    return over


def priors_branch(cfg, shape):
    """The branch of ``Engine::priors()`` an evaluation takes, and whether orthogonality runs (it needs two images)."""
    c = make_cfg(cfg)
    image = c.tv_scale != 0 or c.norm_scale != 0
    branch = "orthogonality alone" if not image else "non-RGB norm kernel" if shape[1] != 3 else "RGB fused kernel"
    return branch, bool(c.orthogonality) and shape[0] >= 2


def di_plan(prog):
    """DeepInversion statistics as ``Engine::build_di_tables`` chooses them: the batched slab kernels iff every BN input has
    ``C % 4 == 0`` and ``C >= 4``, else per layer (float4 where C allows, scalar elsewhere).  Per BN layer: (C, M, kernel, block
    share of the batched launch before the 4-block floor, finalize groups of 256 channels)."""
    ins = [prog.tensors[op.tin] for op in prog.ops if op.kind == C.OP_BNACT and op.has_bn]
    vec = [t.C % 4 == 0 and t.C >= 4 for t in ins]
    total = sum(t.N * t.C * t.H * t.W for t in ins)
    layers = [(t.C, t.N * t.H * t.W, "float4" if v else "scalar", int(t.N * t.C * t.H * t.W / total * 16 * NUM_SMS + 0.5),
               -(-t.C // 256)) for t, v in zip(ins, vec)]
    return ("batched" if all(vec) else "per-layer"), layers


def feature_targets(prog, seed=5):
    """Seeded random feature targets [N, F] in torch flatten order for the input of the features prior's Linear."""
    t = prog.tensors[prog.ops[prog.feature_op].tin]
    return torch.randn(t.N, t.C * t.H * t.W, generator=torch.Generator().manual_seed(seed))


def test_the_entries_reach_every_path():
    """From the programs alone: the DI statistics paths (both choices, a per-layer scalar and float4 layer, a clamped share, several
    finalize groups, M = 1) and the three branches of ``Engine::priors()``, each with orthogonality."""
    paths, layers, branches = set(), set(), set()
    for name in ENTRIES:
        model, shape, *_ = build_entry(name)
        prog = C.compile_model(model, shape)
        cfg = get_attack_config("invertinggradients", prior_overrides(name, prog, shape))
        branches.add(priors_branch(cfg, shape))
        if any(op.kind == C.OP_BNACT and op.has_bn and not op.bn_train for op in prog.ops):
            path, per = di_plan(prog)
            paths.add(path)
            for c, m, kernel, share, groups in per:
                layers |= {(path, kernel)} | ({("clamped",)} if path == "batched" and share < 4 else set())
                layers |= ({("groups > 1",)} if path == "batched" and groups > 1 else set()) | ({("M = 1",)} if m == 1 else set())
            print(f"{name}: DI {path}, layers (C, M, kernel, share, groups) {per}")
        print(f"{name}: priors() branch {priors_branch(cfg, shape)}")
    assert paths == {"batched", "per-layer"}
    assert {("per-layer", "float4"), ("per-layer", "scalar"), ("clamped",), ("groups > 1",), ("M = 1",)} <= layers, layers
    assert {("orthogonality alone", True), ("non-RGB norm kernel", True), ("RGB fused kernel", True)} <= branches, branches


@pytest.mark.parametrize("backend", ["simt", "tc"])
@pytest.mark.parametrize("name", ENTRIES)
def test_every_prior_of_the_case(name, backend):
    model, shape, labels, grads, options = build_entry(name)
    prog = C.compile_model(model, shape)
    train_bn = any(op.kind == C.OP_BNACT and op.bn_train for op in prog.ops)
    if train_bn:   # no running statistics: DeepInversion and the features prior are refused at creation
        cfg = get_attack_config("invertinggradients", {**prior_overrides(name, prog, shape),
                                                       "regularization.deep_inversion.scale": 1e-3})
        with pytest.raises(EngineError, match="DeepInversion / feature priors need running statistics"):
            make_engine(model, shape, cfg, labels, grads, backend, options=options)
    cfg = get_attack_config("invertinggradients", prior_overrides(name, prog, shape, with_di_and_features=not train_bn))
    feats = None if train_bn else feature_targets(prog)
    di = di_plan(prog)[0] if make_cfg(cfg).di_scale > 0 else "off"
    eng = make_engine(model, shape, cfg, labels, grads, backend, feats, options)
    try:
        chk = check_evaluation(eng, candidate(shape), model, grads, labels, cfg, feats,
                               f"{name} / {backend}, priors() branch {priors_branch(cfg, shape)}, DI statistics {di}")
    finally:
        eng.close()
    obj = chk.obj
    assert obj["norm"] is not None or name == NO_IMAGE_TERMS
    assert (obj["di"] is not None) == (not train_bn and any(op.has_bn for op in prog.ops))
    assert (obj["features"] is not None) == (not train_bn)
    assert bool(obj.get("orthogonality")) == (shape[0] >= 2)
    assert ("terms", "norm") in chk.ratios and ("terms", "task_loss") in chk.ratios


# ---- FedAvg: DeepInversion and task-loss regularisation on the last of two local steps -------------------------------------------
@pytest.mark.parametrize("backend", ["simt", "tc"])
@pytest.mark.parametrize("name", ["stem3-k2s3p0-ties", "di-mixed"])
def test_fedavg_priors_of_the_case(name, backend):
    """The last step's DeepInversion adjoints seed its tangent backward scaled by -1/lr (per-layer statistics on di-mixed)."""
    model, shape, *_ = build_entry(name)
    model, shared, hyper, _, cand, ms = fedavg_case(name, model_shape=(model, shape))
    cfg = get_attack_config("invertinggradients", {"regularization.deep_inversion.scale": 1e-3, "objective.task_regularization": 0.1})
    chk, obj = FP.check_engine(name, backend, case=(model, shared, hyper, cfg, cand, ms))
    assert obj["di"] is not None and obj["task_regularization"] != 0 and obj.get("features") is None
    print(f"{name}: DI {di_plan(chk.prog)[0]}")


# ---- registration order vs. execution order ------------------------------------------------------------------------------------
PRIORS = {BNRegisteredLate: ({"regularization.deep_inversion.scale": 1e-2, "regularization.features.scale": 0.1}, "deep_inversion",
                             r"BatchNorm 'bn2' is registered first but 'bn1' runs first"),
          LinearRegisteredLast: ({"regularization.features.scale": 0.1}, "features",
                                 r"Linear 'proj' is registered last but 'fc' runs last")}


@pytest.mark.parametrize("cls", [BNRegisteredLate, LinearRegisteredLast], ids=["bn", "linear"])
def test_registration_order(cls):
    """A network whose first registered BN / last registered Linear is not the first / last to run is refused the prior, naming
    both layers.  Its twin registered in run order (same parameters and buffers) gets the reference's objective and candidate
    gradient: the fp32 back end against restate.TrialOracle in float64, with the attack's own feature targets."""
    over, key, message = PRIORS[cls]
    cfg = get_attack_config("invertinggradients", over)
    model, shape, labels, grads = registration_case(cls)
    with pytest.raises(EngineError, match=message):
        Engine(copy.deepcopy(model).to(DEV), shape, cfg, DEV, backend="simt")
    model, shape, labels, grads = registration_case(cls, in_order=True)
    feats = measured_features([dict(gradients=grads)], labels)[0]
    eng = make_engine(model, shape, cfg, labels, grads, "simt", feats)
    x = candidate(shape)
    try:
        val, grad = eng.objective_and_gradient(x.to(DEV))
        terms = eng.last_terms()
    finally:
        eng.close()
    orc = restate.TrialOracle(copy.deepcopy(model).double(), nn.CrossEntropyLoss(), cfg, [g.double() for g in grads], labels, None, None,
                              dtype=torch.float64)
    phi, _, raw, ref_terms = orc.closure_gradient(x.double(), 0, 0.0)
    orc.close()
    rel = ((grad.cpu().double() - raw).norm() / raw.norm()).item()
    print(f"\n[{cls.__name__} in run order] objective {val:.9g} (float64 {float(phi):.9g}), {key} {terms[key]:.6g} "
          f"(float64 {ref_terms[key]:.6g}), candidate gradient rel. error {rel:.2e}")
    assert ref_terms[key] > 0
    assert math.isclose(terms[key], ref_terms[key], rel_tol=1e-5), (terms, ref_terms)
    assert math.isclose(val, float(phi), rel_tol=1e-5), (val, float(phi))
    assert rel < 1e-4, rel
