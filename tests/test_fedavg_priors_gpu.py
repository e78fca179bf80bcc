"""FedAvg (multi-step) updates with the priors of the last local step on the engine: task-loss regularisation and DeepInversion
enter the last step's tangent-backward stream as seeds scaled by -1/lr (DESIGN.md section 3.1).  Against the reference's own
outputs (tests/golden/trial_fedavg_{taskreg,di}_*.pt), buffer by buffer against float64 (oracle/fedavg_priors.PriorMultiStepChecker),
through the attacker API, and with the priors off the iteration issues exactly the launches it did before they existed."""
import copy
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from breaching_b200 import compiler as C  # noqa: E402
from breaching_b200 import get_attack_config, synthetic  # noqa: E402
from breaching_b200.attacks import prepare_attack  # noqa: E402
from breaching_b200.engine import Engine, EngineError  # noqa: E402
from breaching_b200.schedule import lr_table  # noqa: E402
from helpers import case_from_fixture, cfg_from_fixture, load_golden, sweep_objective  # noqa: E402
from oracle.fedavg_priors import PriorMultiStepChecker  # noqa: E402
from oracle.sweep_check import on_grid  # noqa: E402
from test_sweep_multistep_gpu import WHICH, EngineGlue, EngineStepSource, read_params, read_tensors  # noqa: E402

DEV = torch.device("cuda:0")
FIXTURES = ["fedavg_taskreg_convnet", "fedavg_di_convnet", "fedavg_di_resnet18"]
PRIORS = {"regularization.features.scale": 0.0, "regularization.deep_inversion.scale": 0.01, "objective.task_regularization": 0.1}
# launches per iteration of BASELINE config 4 (ResNet-18 224 x 224, 4 local steps, `modern` without priors) before the priors of
# FedAvg existed, measured on an H100 80GB HBM3 with the parent of the change that added them
CONFIG4_LAUNCHES = {"tc": 916, "simt": 877}


def _relerr(a, b):
    return ((a.double().cpu() - b.double().cpu()).norm() / (b.double().cpu().norm() + 1e-30)).item()


def _engine(fx, backend):
    model, loss_fn, payload, shared, true = case_from_fixture(fx)
    cfg = cfg_from_fixture(fx)
    local = shared[0]["metadata"]["local_hyperparams"]
    meta = payload[0]["metadata"]
    eng = Engine(copy.deepcopy(model).to(DEV).eval(), (local["data_per_step"], *fx["x0"].shape[1:]), cfg, DEV, backend=backend)
    eng.load_model()
    eng.load_targets([g.to(DEV) for g in shared[0]["gradients"]], local["labels"][0], mean=meta.mean, std=meta.std)
    eng.set_local_steps(fx["x0"].shape[0], local["steps"], local["lr"], local["labels"])
    return eng, cfg


def _tf32(t):
    """``t`` rounded to nearest onto the TF32 grid, with an identity gradient."""
    r = torch.bitwise_and(t.contiguous().view(torch.int32) + 0x1000, -0x2000).view(torch.float32)
    return t + (r - t).detach()


def _reference_tf32_deviation(fx):
    """rel. l2 distance between the reference algorithm in eager PyTorch on the GPU with TF32 convolutions (the reference's default
    GPU numerics; every convolution reads its operands on the TF32 grid) and the fp32 fixture.  The DeepInversion hooks of the oracle
    fire on the module that torch.func.functional_call evaluates, so the last local step's statistics win, as in the fixture."""
    from oracle import restate

    model, loss_fn, payload, shared, true = case_from_fixture(fx)
    cfg = cfg_from_fixture(fx)
    meta = payload[0]["metadata"]
    dm = torch.tensor(meta.mean, device=DEV)[None, :, None, None]
    ds = torch.tensor(meta.std, device=DEV)[None, :, None, None]
    local = copy.deepcopy(shared[0]["metadata"]["local_hyperparams"])
    local["labels"] = [lab.to(DEV) for lab in local["labels"]]
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    conv_forward = torch.nn.Conv2d._conv_forward
    torch.nn.Conv2d._conv_forward = lambda self, x, w, b: conv_forward(self, _tf32(x), _tf32(w), b)
    try:
        orc = restate.TrialOracle(copy.deepcopy(model).to(DEV).eval(), loss_fn, cfg, [g.to(DEV) for g in shared[0]["gradients"]],
                                  torch.cat(local["labels"]), dm, ds, local_hyperparams=local)
        _, _, raw, _ = orc.closure_gradient(fx["x0"].to(DEV), 0, 0.0)
        orc.close()
    finally:
        torch.nn.Conv2d._conv_forward = conv_forward
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
    return _relerr(raw, fx["raw_grad0"])


@pytest.mark.parametrize("backend", ["simt", "tc"])
@pytest.mark.parametrize("name", FIXTURES)
def test_closure_matches_reference_fixture(name, backend):
    fx = load_golden(f"trial_{name}.pt")
    eng, cfg = _engine(fx, backend)
    val, grad = eng.objective_and_gradient(fx["x0"].to(DEV))
    terms = eng.last_terms()
    tol_v, tol_g = (2e-3, 1e-2) if backend == "simt" else (2e-2, 5e-2)
    if backend == "tc":
        tol_g = max(tol_g, 1.5 * _reference_tf32_deviation(fx))
    assert math.isclose(val, fx["objective0"], rel_tol=tol_v, abs_tol=1e-6), (val, fx["objective0"], terms)
    # the reported terms: the last local step's task loss (weighted into the value) and the DeepInversion term of its forward
    assert math.isclose(terms["task_loss"], fx["task_loss0"], rel_tol=1e-3 if backend == "simt" else 1e-2)
    di = fx["overrides"].get("regularization.deep_inversion.scale", 0.0) > 0
    assert (terms["deep_inversion"] > 0) == di, terms
    tau = fx["overrides"]["objective.task_regularization"]
    parts = terms["match"] + terms["total_variation"] + terms["norm"] + terms["deep_inversion"] + tau * terms["task_loss"]
    assert math.isclose(val, parts, rel_tol=1e-6), (val, terms)
    rel = _relerr(grad, fx["raw_grad0"])
    assert rel < tol_g, (rel, tol_g)
    eng.close()


@pytest.mark.parametrize("name", FIXTURES)
def test_trajectory_matches_reference_fixture(name):
    fx = load_golden(f"trial_{name}.pt")
    eng, cfg = _engine(fx, "simt")
    opt = cfg.optim
    eng.begin_trial(fx["x0"].to(DEV), lr_table(opt.step_size, opt.step_size_decay, opt.warmup, opt.max_iterations))
    eng.run(fx["iters"])
    eng.sync()
    hist = eng.history().tolist()
    assert len(hist) == fx["iters"]
    for a, b in zip(hist, fx["history"]):
        assert math.isclose(a, b, rel_tol=2e-3, abs_tol=1e-5), (hist, fx["history"])
    assert (eng.candidate().cpu() - fx["candidate_final"]).abs().mean().item() < 5e-3
    eng.close()


# ---- every buffer of every step against float64 ----------------------------------------------------------------------------
def build_case(name):
    """(model, shared, local hyper-parameters, attack config, candidate, mean / std)."""
    if name.startswith("fixture:"):
        fx = load_golden(f"trial_{name[8:]}.pt")
        model, loss_fn, payload, shared, true = case_from_fixture(fx)
        cfg, x = cfg_from_fixture(fx), fx["x0"]
    else:
        size = 224 if name == "config4" else 64
        model, loss_fn, payload, shared, true = synthetic.make_fedavg_case(
            "resnet18", "imagenet", num_data_points=4, steps=4, data_per_step=1, lr=1e-3, seed=3 if size == 64 else 233,
            image_size=size if size == 64 else None, classes=10 if size == 64 else None)
        over = dict(PRIORS) if name != "config4" else {"regularization.features.scale": 0.0, "regularization.deep_inversion.scale": 0.01}
        cfg = get_attack_config("modern", over)
        x = torch.randn(4, 3, size, size, generator=torch.Generator().manual_seed(3))
    meta = payload[0]["metadata"]
    return model.eval(), shared, shared[0]["metadata"]["local_hyperparams"], cfg, x, (meta.mean, meta.std)


def make_engine(case, backend):
    model, shared, local, cfg, x, (mean, std) = case
    eng = Engine(copy.deepcopy(model).to(DEV).eval(), (local["data_per_step"], *x.shape[1:]), cfg, DEV, backend=backend)
    eng.load_model()
    eng.load_targets([g.to(DEV) for g in shared[0]["gradients"]], local["labels"][0], mean=mean, std=std)
    eng.set_local_steps(x.shape[0], local["steps"], local["lr"], local["labels"])
    return eng


def check_engine(name, backend, keep_tangents=False, case=None):
    """``case``: a tuple as build_case returns it, instead of the named one."""
    case = build_case(name) if case is None else case
    model, shared, local, cfg, x, _ = case
    K, dps = local["steps"], local["data_per_step"]
    eng = make_engine(case, backend)
    n = len(eng.prog.params)
    xd = x.to(DEV)
    fwd, rev, unwritten, D = [], [], [], {}
    for k in range(K):
        eng.set_option("debug_multistep_stop", k + 1)
        eng.objective_and_gradient(xd)
        f = read_tensors(eng, ("val", "delta"))
        f.update(read_params(eng, ("G",)))
        fwd.append(f)
        D[k + 1] = [eng.debug_step_param("D", 0, j) for j in range(n)]
    for k in range(K):
        eng.set_option("debug_multistep_stop", K + 1 + k)
        eng.objective_and_gradient(xd)
        r = read_tensors(eng, WHICH)
        r.update(read_params(eng, ("v", "v_operand") + (("G",) if k > 0 else ())))
        rev.append(r)
        unwritten.append({op.tin for i, op in enumerate(eng.prog.ops) if eng.debug_op(i)["tangent_in_unwritten"]})
    eng.set_option("debug_multistep_stop", 0)
    _, grad = eng.objective_and_gradient(xd)
    W = [[eng.debug_step_param("W", k, j) for j in range(n)] for k in range(K + 1)]
    Wo = [[eng.debug_step_param("W_operand", k, j) for j in range(n)] for k in range(K + 1)]
    stem = {i for i in range(len(eng.prog.ops)) if eng.debug_op(i)["stem_columns"]}
    prog = eng.prog
    eng.close()
    glue = EngineGlue(W, Wo, D, x, grad.cpu(), [(k * dps) % x.shape[0] for k in range(K)],
                      float(torch.tensor(local["lr"], dtype=torch.float32)))
    bn = [None if m is None or m.running_mean is None else (m.running_mean.double(), m.running_var.double())
          for m in C.bn_modules(model, prog)]
    srcs = [EngineStepSource(fwd[k], rev[k], k, glue, stem, unwritten[k]) for k in range(K)]
    obj = sweep_objective(cfg)
    chk = PriorMultiStepChecker(prog, bn, shared[0]["gradients"], local["labels"], obj, srcs, glue)
    try:
        chk.check()
    finally:
        print(f"\n[{name} / {backend}] " + ", ".join(f"{k}/{s}: {r:.3g}" for (k, s), r in sorted(chk.ratios.items())) +
              f"; off-grid (step, op): {sorted(chk.off_grid)}")
    return (chk, obj, rev) if keep_tangents else (chk, obj)


@pytest.mark.parametrize("backend", ["simt", "tc"])
@pytest.mark.parametrize("name", ["fixture:fedavg_di_convnet", "resnet18-64"])
def test_every_step_buffer_with_priors(name, backend):
    """fedavg-convnet (3 steps x 2 images, the last slice wraps) and ResNet-18 at 64 x 64 (4 steps x 1 image), DI and tau on."""
    chk, obj = check_engine(name, backend)
    assert obj["di"] is not None and obj["task_regularization"] != 0


def test_config4_with_deep_inversion_every_step_buffer():
    """BASELINE config 4 at full size with DeepInversion on, tensor cores.  The seeded tangent deltas of the last step (every BN
    input: a tensor-core dgrad operand) are stored on the TF32 grid, and the seeds add no off-grid operand: the only ones the
    checker lists are the activations of the convolution fed by the max-pool, at every step, as without priors (the case
    oracle/sweep_check.py documents)."""
    chk, _, rev = check_engine("config4", "tc", keep_tangents=True)
    prog = chk.prog
    pool_outputs = {op.tout for op in prog.ops if op.kind == C.OP_MAXPOOL}
    pooled = {i for i, op in enumerate(prog.ops) if op.kind == C.OP_CONV and op.tin in pool_outputs}
    assert {i for _, i in chk.off_grid} <= pooled, sorted(chk.off_grid)
    for op in prog.ops:
        if op.kind == C.OP_BNACT and op.has_bn:
            assert on_grid(rev[-1][("tangent_delta", op.tin)]), op.tin


# ---- neutrality, API, refusal ------------------------------------------------------------------------------------------------
def _config4_engine(backend, overrides):
    model, loss_fn, payload, shared, true = synthetic.make_fedavg_case("resnet18", "imagenet", num_data_points=4, steps=4,
                                                                       data_per_step=1, lr=1e-3, seed=233)
    cfg = get_attack_config("modern", overrides)
    local = shared[0]["metadata"]["local_hyperparams"]
    meta = payload[0]["metadata"]
    eng = Engine(copy.deepcopy(model).to(DEV).eval(), (1, 3, 224, 224), cfg, DEV, backend=backend)
    eng.load_model()
    eng.load_targets([g.to(DEV) for g in shared[0]["gradients"]], local["labels"][0], mean=meta.mean, std=meta.std)
    eng.set_local_steps(4, 4, float(local["lr"]), local["labels"])
    eng.begin_trial(torch.randn(4, 3, 224, 224, generator=torch.Generator().manual_seed(0)).to(DEV), lr_table(0.1, "cosine-decay", 50, 24000, 8))
    eng.run(2)
    eng.sync()
    return eng


@pytest.mark.parametrize("backend", ["tc", "simt"])
def test_priors_off_keep_the_launch_sequence(backend):
    """tau = 0 and DI scale 0: the config-4 iteration issues exactly the launches it issued before the priors existed; with both
    priors on, the DeepInversion statistics add two (the batched statistics and the finalisation); the task seed replaces the
    logits seed kernel."""
    eng = _config4_engine(backend, {"regularization.features.scale": 0.0})
    assert eng.launches_per_iteration() == CONFIG4_LAUNCHES[backend]
    eng.close()
    eng = _config4_engine(backend, dict(PRIORS))
    assert eng.launches_per_iteration() == CONFIG4_LAUNCHES[backend] + 2
    assert all(math.isfinite(h) for h in eng.history().tolist())
    eng.close()


def _fedavg_case():
    return synthetic.make_fedavg_case("resnet18", "imagenet", num_data_points=4, steps=4, data_per_step=1, lr=1e-3, seed=3,
                                      image_size=64, classes=10)


@pytest.mark.parametrize("preset,overrides", [
    ("modern", {"regularization.features.scale": 0.0, "regularization.deep_inversion.scale": 0.01}),
    ("seethroughgradients", {"optim.langevin_noise": 0.0}),      # euclidean + DI + norm + TV
    ("modern", {"regularization.features.scale": 0.0, "objective.task_regularization": 0.1}),
])
def test_through_the_attacker_api(preset, overrides):
    model, loss_fn, payload, shared, true = _fedavg_case()
    cfg = get_attack_config(preset, {**overrides, "optim.max_iterations": 12, "optim.callback": 6, "optim.warmup": 2})
    attacker = prepare_attack(model, loss_fn, cfg, dict(device=DEV, dtype=torch.float))
    rec, stats = attacker.reconstruct(payload, copy.deepcopy(shared), {}, dryrun=False)
    assert rec["data"].shape == (4, 3, 64, 64) and len(stats["Trial_0_Val"]) == 12
    assert math.isfinite(stats["opt_value"]) and torch.isfinite(rec["data"]).all()


def test_zero_local_learning_rate_with_a_prior_is_refused():
    model, loss_fn, payload, shared, true = _fedavg_case()
    local = shared[0]["metadata"]["local_hyperparams"]
    meta = payload[0]["metadata"]
    for over in ({"objective.task_regularization": 0.1}, {"regularization.deep_inversion.scale": 0.01}):
        cfg = get_attack_config("modern", {"regularization.features.scale": 0.0, **over})
        eng = Engine(copy.deepcopy(model).to(DEV).eval(), (1, 3, 64, 64), cfg, DEV)
        eng.load_model()
        eng.load_targets([g.to(DEV) for g in shared[0]["gradients"]], local["labels"][0], mean=meta.mean, std=meta.std)
        with pytest.raises(EngineError, match="nonzero local learning rate"):
            eng.set_local_steps(4, 4, 0.0, local["labels"])
        eng.close()
