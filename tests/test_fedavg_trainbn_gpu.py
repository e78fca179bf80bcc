"""FedAvg (multi-step) updates of train-mode BatchNorm networks on the engine: without BN buffers every local step normalises with
its own batch statistics, and the reverse pass of step k reads that step's constants and sweep-B sums while the gamma / beta
tangents of its Hessian-vector product come out of the tangent-backward statistics kernel (DESIGN.md section 3.1).  Against the
reference's own outputs (tests/golden/trial_fedavg_trainbn_*.pt), buffer by buffer against float64
(fedavg_trainbn_oracle.TrainBnMultiStepChecker), at BASELINE config-4 size against float64 autograd, through the attacker API,
and the refusals that remain."""
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
from fedavg_trainbn_oracle import TrainBnMultiStepChecker  # noqa: E402
from helpers import case_from_fixture, cfg_from_fixture, load_golden, sweep_objective  # noqa: E402
from oracle import restate  # noqa: E402
from oracle.sweep_check import SweepCheckError  # noqa: E402
from test_fedavg_priors_gpu import _tf32  # noqa: E402
from test_fedavg_trainbn_cpu import train_mode  # noqa: E402
from test_sweep_multistep_gpu import WHICH, EngineGlue, EngineStepSource, read_params, read_tensors  # noqa: E402

DEV = torch.device("cuda:0")
# the ResNet-18 fixture (one image per step at 64 x 64: its last stage normalises over 2 x 2 pixels) amplifies fp32 rounding too
# much for a comparison of two fp32 implementations; it is checked on the CPU (oracle against the reference) and buffer by buffer
# here, and BASELINE config 4 covers ResNet-18 on both back ends
FIXTURES = ["fedavg_trainbn_convnet", "fedavg_trainbn_taskreg_convnet"]
PLAIN = {"regularization.features.scale": 0.0}


def _relerr(a, b):
    return ((a.double().cpu() - b.double().cpu()).norm() / (b.double().cpu().norm() + 1e-30)).item()


def _engine(model, local, x_shape, cfg, meta, gradients, backend):
    eng = Engine(train_mode(model).to(DEV), (local["data_per_step"], *x_shape[1:]), cfg, DEV, backend=backend)
    assert any(op.bn_train for op in eng.prog.ops)
    eng.load_model()
    eng.load_targets([g.to(DEV) for g in gradients], local["labels"][0], mean=meta.mean, std=meta.std)
    eng.set_local_steps(x_shape[0], local["steps"], local["lr"], local["labels"])
    return eng


def _fixture_engine(fx, backend):
    model, loss_fn, payload, shared, true = case_from_fixture(fx)
    assert payload[0]["buffers"] is None and shared[0]["buffers"] is None
    cfg = cfg_from_fixture(fx)
    local = shared[0]["metadata"]["local_hyperparams"]
    return _engine(model, local, fx["x0"].shape, cfg, payload[0]["metadata"], shared[0]["gradients"], backend), cfg


def _reference_gradient(model, loss_fn, cfg, shared, meta, x, tf32=False, dtype=torch.float32):
    """The reference closure's candidate gradient in eager PyTorch on the GPU (oracle.restate), train mode; ``tf32``: every
    convolution reads its operands on the TF32 grid (the reference's default GPU numerics)."""
    local = copy.deepcopy(shared[0]["metadata"]["local_hyperparams"])
    local["labels"] = [lab.to(DEV) for lab in local["labels"]]
    dm = torch.tensor(meta.mean, device=DEV, dtype=dtype)[None, :, None, None]
    ds = torch.tensor(meta.std, device=DEV, dtype=dtype)[None, :, None, None]
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    conv_forward = torch.nn.Conv2d._conv_forward
    if tf32:
        torch.nn.Conv2d._conv_forward = lambda self, x_, w, b: conv_forward(self, _tf32(x_), _tf32(w), b)
    try:
        orc = restate.TrialOracle(train_mode(model).to(DEV, dtype), loss_fn, cfg, [g.to(DEV, dtype) for g in shared[0]["gradients"]],
                                  torch.cat(local["labels"]), dm, ds, dtype=dtype, local_hyperparams=local)
        val, _, raw, _ = orc.closure_gradient(x.to(DEV, dtype), 0, 0.0)
        orc.close()
    finally:
        torch.nn.Conv2d._conv_forward = conv_forward
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
    return float(val), raw


@pytest.mark.parametrize("backend", ["simt", "tc"])
@pytest.mark.parametrize("name", FIXTURES)
def test_closure_matches_reference_fixture(name, backend):
    fx = load_golden(f"trial_{name}.pt")
    eng, cfg = _fixture_engine(fx, backend)
    val, grad = eng.objective_and_gradient(fx["x0"].to(DEV))
    terms = eng.last_terms()
    tol_v, tol_g = (2e-3, 1e-2) if backend == "simt" else (2e-2, 5e-2)
    if backend == "tc":
        model, loss_fn, payload, shared, true = case_from_fixture(fx)
        _, raw = _reference_gradient(model, loss_fn, cfg, shared, payload[0]["metadata"], fx["x0"], tf32=True)
        tol_g = max(tol_g, 1.5 * _relerr(raw, fx["raw_grad0"]))
    assert math.isclose(val, fx["objective0"], rel_tol=tol_v, abs_tol=1e-6), (val, fx["objective0"], terms)
    assert math.isclose(terms["task_loss"], fx["task_loss0"], rel_tol=1e-3 if backend == "simt" else 5e-2)
    rel = _relerr(grad, fx["raw_grad0"])
    assert rel < tol_g, (rel, tol_g)
    eng.close()


@pytest.mark.parametrize("name", FIXTURES)
def test_trajectory_matches_reference_fixture(name):
    """The fixture's first two iterations (batch statistics over two images make later fp32 iterates of two implementations
    drift apart), and the captured graph and eager launches give bitwise the same history and candidate."""
    fx = load_golden(f"trial_{name}.pt")
    runs = []
    for graph in (1, 0):
        eng, cfg = _fixture_engine(fx, "simt")
        eng.set_option("use_graph", graph)
        opt = cfg.optim
        eng.begin_trial(fx["x0"].to(DEV), lr_table(opt.step_size, opt.step_size_decay, opt.warmup, opt.max_iterations))
        eng.run(fx["iters"])
        eng.sync()
        runs.append((eng.history().clone(), eng.candidate().cpu().clone()))
        eng.close()
    hist = runs[0][0].tolist()
    assert len(hist) == fx["iters"]
    for a, b in zip(hist[:2], fx["history"][:2]):
        assert math.isclose(a, b, rel_tol=2e-3, abs_tol=1e-5), (hist, fx["history"])
    assert all(math.isfinite(h) for h in hist)
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


# ---- every buffer of every step against float64 ----------------------------------------------------------------------------
def build_case(name):
    """(model, shared, local hyper-parameters, attack config, candidate, metadata)."""
    if name.startswith("fixture:"):
        fx = load_golden(f"trial_{name[8:]}.pt")
        model, loss_fn, payload, shared, true = case_from_fixture(fx)
        cfg, x = cfg_from_fixture(fx), fx["x0"]
    else:   # BASELINE config 4 without buffers: ResNet-18 at 224 x 224, 4 steps x 1 image
        model, loss_fn, payload, shared, true = synthetic.make_fedavg_case("resnet18", "imagenet", num_data_points=4, steps=4,
                                                                           data_per_step=1, lr=1e-3, seed=233, no_buffers=True)
        cfg = get_attack_config("modern", dict(PLAIN))
        x = torch.randn(4, 3, 224, 224, generator=torch.Generator().manual_seed(3))
    return model, loss_fn, shared, shared[0]["metadata"]["local_hyperparams"], cfg, x, payload[0]["metadata"]


def check_engine(name, backend):
    model, loss_fn, shared, local, cfg, x, meta = build_case(name)
    K, dps = local["steps"], local["data_per_step"]
    eng = _engine(model, local, x.shape, cfg, meta, shared[0]["gradients"], backend)
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
    value, grad = eng.objective_and_gradient(xd)
    terms = eng.last_terms()
    W = [[eng.debug_step_param("W", k, j) for j in range(n)] for k in range(K + 1)]
    Wo = [[eng.debug_step_param("W_operand", k, j) for j in range(n)] for k in range(K + 1)]
    stem = {i for i in range(len(eng.prog.ops)) if eng.debug_op(i)["stem_columns"]}
    prog = eng.prog
    eng.close()
    glue = EngineGlue(W, Wo, D, x, grad.cpu(), [(k * dps) % x.shape[0] for k in range(K)],
                      float(torch.tensor(local["lr"], dtype=torch.float32)))
    srcs = [EngineStepSource(fwd[k], rev[k], k, glue, stem, unwritten[k]) for k in range(K)]
    chk = TrainBnMultiStepChecker(prog, [None] * len(prog.ops), shared[0]["gradients"], local["labels"], sweep_objective(cfg), srcs, glue)
    try:
        chk.check(raise_on_failure=False)
        chk.check_terms(terms, value, raise_on_failure=False)
        if chk.findings:
            raise SweepCheckError("\n".join(repr(f) for f in chk.findings[:20]))
    finally:
        print(f"\n[{name} / {backend}] " + ", ".join(f"{k}/{s}: {r:.3g}" for (k, s), r in sorted(chk.ratios.items())) +
              f"; off-grid (step, op): {sorted(chk.off_grid)}")
    return chk


@pytest.mark.parametrize("backend", ["simt", "tc"])
@pytest.mark.parametrize("name", ["fixture:fedavg_trainbn_convnet", "fixture:fedavg_trainbn_taskreg_convnet", "fixture:fedavg_trainbn_resnet18",
                                  "config4"])
def test_every_step_buffer(name, backend):
    """Every step's sweeps, the gamma / beta tangents of every train-mode BN at steps k > 0 included, and the glue."""
    chk = check_engine(name, backend)
    train = [i for i, op in enumerate(chk.prog.ops) if op.kind == C.OP_BNACT and op.has_bn and op.bn_train]
    assert train and any(sweep == "TG" for _, sweep in chk.ratios)


# ---- config-4 size: the closure against float64 ------------------------------------------------------------------------------
@pytest.mark.parametrize("backend", ["simt", "tc"])
def test_config4_closure(backend):
    """fp32 back end: within float64 noise of the float64 closure; TF32 back end: within a small multiple of the reference's own
    TF32 deviation (eager PyTorch on the GPU, every convolution on TF32 operands)."""
    model, loss_fn, shared, local, cfg, x, meta = build_case("config4")
    eng = _engine(model, local, x.shape, cfg, meta, shared[0]["gradients"], backend)
    val, grad = eng.objective_and_gradient(x.to(DEV))
    eng.close()
    val64, raw64 = _reference_gradient(model, loss_fn, cfg, shared, meta, x, dtype=torch.float64)
    rel = _relerr(grad, raw64)
    if backend == "simt":
        _, raw32 = _reference_gradient(model, loss_fn, cfg, shared, meta, x)
        bound = max(1e-4, 4 * _relerr(raw32, raw64))   # fp32 rounding of the reference's own eager run
        tol_v = 1e-4
    else:
        _, raw_tf32 = _reference_gradient(model, loss_fn, cfg, shared, meta, x, tf32=True)
        bound = 3 * _relerr(raw_tf32, raw64)
        tol_v = 1e-2
    print(f"\nconfig4 train-mode FedAvg / {backend}: rel. gradient error {rel:.3g} (bound {bound:.3g})")
    assert math.isclose(val, val64, rel_tol=tol_v), (val, val64)
    assert rel < bound, (rel, bound)


# ---- API, refusals -----------------------------------------------------------------------------------------------------------
def test_through_the_attacker_api():
    model, loss_fn, payload, shared, true = synthetic.make_fedavg_case("resnet18", "imagenet", num_data_points=4, steps=4,
                                                                       data_per_step=1, lr=1e-3, seed=3, image_size=64, classes=10,
                                                                       no_buffers=True)
    cfg = get_attack_config("modern", {**PLAIN, "optim.max_iterations": 12, "optim.callback": 6, "optim.warmup": 2})
    attacker = prepare_attack(model, loss_fn, cfg, dict(device=DEV, dtype=torch.float))
    rec, stats = attacker.reconstruct(payload, copy.deepcopy(shared), {}, dryrun=False)
    assert rec["data"].shape == (4, 3, 64, 64) and len(stats["Trial_0_Val"]) == 12
    assert math.isfinite(stats["opt_value"]) and torch.isfinite(rec["data"]).all()


def test_one_value_per_channel_is_refused():
    """ResNet-18 at 32 x 32 with one image per step: its last stage would normalise over 1 x 1 pixels.  No user can train such a
    step (torch refuses it, see test_fedavg_trainbn_cpu.py), and the engine refuses to run one, naming the layer."""
    model, loss_fn, payload, shared, true = synthetic.make_fedavg_case("resnet18", "imagenet", num_data_points=2, steps=1,
                                                                       data_per_step=2, lr=1e-2, seed=6, image_size=32, classes=10,
                                                                       no_buffers=True)
    meta, y = payload[0]["metadata"], true["labels"]
    eng = Engine(train_mode(model).to(DEV), (1, 3, 32, 32), get_attack_config("modern", dict(PLAIN)), DEV)
    eng.load_model()
    eng.load_targets([g.to(DEV) for g in shared[0]["gradients"]], y[:1], mean=meta.mean, std=meta.std)
    with pytest.raises(EngineError, match=r"train-mode BatchNorm layer at op \d+ \(512 channels at 1x1\) sees one value per channel"):
        eng.set_local_steps(2, 2, 1e-2, [y[:1], y[1:2]])
    eng.close()


def test_statistics_priors_are_still_refused():
    """DeepInversion and the features prior need running statistics (refused at engine creation); the features prior is also not
    defined for multi-step updates."""
    model, loss_fn, payload, shared, true = synthetic.make_fedavg_case("resnet18", "imagenet", num_data_points=4, steps=4,
                                                                       data_per_step=1, lr=1e-3, seed=3, image_size=64, classes=10,
                                                                       no_buffers=True)
    for over in ({"regularization.features.scale": 0.0, "regularization.deep_inversion.scale": 0.01}, {}):
        with pytest.raises(EngineError, match="need running statistics"):
            Engine(train_mode(model).to(DEV), (1, 3, 64, 64), get_attack_config("modern", over), DEV)
