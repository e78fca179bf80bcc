"""Every buffer of every local step of a multi-step (FedAvg) evaluation against float64 (oracle/sweep_check.MultiStepChecker), on
both GEMM back ends.  The engine's option ``debug_multistep_stop`` stops the evaluation after step k's forward / backward sweeps
(its activations, deltas, G_k) and after its tangent sweeps (tangents, tangent deltas, the direction u_{k+1} it used and its
tangent weight gradients); a full evaluation gives W_0..W_K, their operand forms and the final candidate gradient.  Each step's
kernels are judged on the engine's own inputs, and the glue between the steps (weight updates, D, the adjoint updates, the
candidate-gradient assembly) by one-rounding relations."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

from breaching_b200 import compiler as C  # noqa: E402
from breaching_b200 import get_attack_config, synthetic  # noqa: E402
from breaching_b200.engine import Engine, EngineError  # noqa: E402
from breaching_b200.schedule import lr_table  # noqa: E402
from helpers import case_from_fixture, cfg_from_fixture, load_golden, sweep_objective  # noqa: E402
from oracle.sweep_check import MultiStepChecker, SweepCheckError  # noqa: E402

DEV = torch.device("cuda:0")
WHICH = ("val", "delta", "tangent", "tangent_delta")


def build_case(name):
    """(model, shared, local hyper-parameters, attack config, candidate [N, 3, H, W], mean / std)."""
    if name == "fedavg-convnet":
        fx = load_golden("trial_fedavg_convnet.pt")
        model, loss_fn, payload, shared, true = case_from_fixture(fx)
        cfg, x = cfg_from_fixture(fx), fx["x0"]
    else:
        size = 224 if name == "config4" else 64
        model, loss_fn, payload, shared, true = synthetic.make_fedavg_case(
            "resnet18", "imagenet", num_data_points=4, steps=4, data_per_step=1, lr=1e-3, seed=3 if size == 64 else 233,
            image_size=size if size == 64 else None, classes=10 if size == 64 else None)
        cfg = get_attack_config("modern", {"regularization.features.scale": 0.0})
        x = torch.randn(4, 3, size, size, generator=torch.Generator().manual_seed(3))
    meta = payload[0]["metadata"]
    return model.eval(), shared, shared[0]["metadata"]["local_hyperparams"], cfg, x, (meta.mean, meta.std)


def make_engine(case, backend, options=()):
    model, shared, local, cfg, x, (mean, std) = case
    eng = Engine(copy.deepcopy(model).to(DEV).eval(), (local["data_per_step"], *x.shape[1:]), cfg, DEV, backend=backend)
    for k, v in options:
        eng.set_option(k, v)
    eng.load_model()
    eng.load_targets([g.to(DEV) for g in shared[0]["gradients"]], local["labels"][0], mean=mean, std=std)
    eng.set_local_steps(x.shape[0], local["steps"], local["lr"], local["labels"])
    return eng


def read_tensors(eng, which):
    out = {}
    for w in which:
        for tid in range(len(eng.prog.tensors)):
            if tid == 0 and w in ("tangent", "delta"):   # the candidate has no tangent; its delta is not a step buffer
                continue
            out[(w, tid)] = eng.debug_tensor(w, tid)
    return out


def read_params(eng, which):
    return {(w, j): eng.debug_param(w, j) for w in which for j in range(len(eng.prog.params))}


class EngineStepSource:
    """Step k of a multi-step evaluation: forward / backward buffers from the stop after its backward sweep, tangent buffers from
    the stop after its tangent sweeps."""

    def __init__(self, fwd, rev, k, glue, stem, unwritten):
        self.fwd, self.rev, self.k, self.glue = fwd, rev, k, glue
        self.has_tangent_G = k > 0
        self.stem, self.unwritten = stem, unwritten

    def rounds_operands(self, i):
        return i in self.stem

    def tensor(self, which, tid):
        t = (self.fwd if which in ("val", "delta") else self.rev).get((which, tid))
        return None if t is None else t.double()

    def param(self, which, idx):
        if which == "W_operand":
            return self.glue.W_operand[self.k][idx].double()
        if which == "TG":
            return self.rev[("G", idx)].double()
        return (self.fwd if which == "G" else self.rev)[(which, idx)].double()


class EngineGlue:
    def __init__(self, W, W_operand, D, x, grad, offsets, lr):
        self.W, self.W_operand, self.D, self.x, self.grad, self.offsets, self.lr = W, W_operand, D, x, grad, offsets, lr

    def shadowed(self, j):
        return not torch.equal(self.W_operand[0][j], self.W[0][j])


def check_engine(name, backend, options=(), env=None, monkeypatch=None, case=None):
    """``case``: a tuple as build_case returns it, instead of the named one."""
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    case = build_case(name) if case is None else case
    model, shared, local, cfg, x, _ = case
    K, dps = local["steps"], local["data_per_step"]
    eng = make_engine(case, backend, options)
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
        # the stops see the same forward buffers: nothing of the evaluation before a stop depends on where it stops
        for key, t in fwd[k].items():
            if key[0] in ("val", "delta"):
                assert torch.equal(t, r[key]), (k, key)
    eng.set_option("debug_multistep_stop", 0)
    value, grad = eng.objective_and_gradient(xd)
    terms = eng.last_terms()
    W = [[eng.debug_step_param("W", k, j) for j in range(n)] for k in range(K + 1)]
    Wo = [[eng.debug_step_param("W_operand", k, j) for j in range(n)] for k in range(K + 1)]
    stem = {i for i in range(len(eng.prog.ops)) if eng.debug_op(i)["stem_columns"]}
    prog = eng.prog
    scores = []   # (kind, score, the D its pass accumulated)
    for kind in ("euclidean", "cosine-similarity"):
        sc = eng.score(xd, kind)
        scores.append((kind, sc, [eng.debug_step_param("D", 0, j) for j in range(n)]))
    offsets = [(k * dps) % x.shape[0] for k in range(K)]
    eng.close()
    glue = EngineGlue(W, Wo, D, x, grad.cpu(), offsets, float(torch.tensor(local["lr"], dtype=torch.float32)))
    bn = [None if m is None or m.running_mean is None else (m.running_mean.double(), m.running_var.double())
          for m in C.bn_modules(model, prog)]
    srcs = [EngineStepSource(fwd[k], rev[k], k, glue, stem, unwritten[k]) for k in range(K)]
    chk = MultiStepChecker(prog, bn, shared[0]["gradients"], local["labels"], sweep_objective(cfg), srcs, glue)
    chk.stem, chk.unwritten = sorted(stem), unwritten
    try:
        chk.check(raise_on_failure=False)
        chk.check_terms(terms, value, raise_on_failure=False)
        for kind, sc, Ds in scores:
            chk.check_score(sc, kind, Ds, raise_on_failure=False)
        if chk.findings:
            raise SweepCheckError("\n".join(repr(f) for f in chk.findings[:20]))
    finally:
        print(f"\n[{name} / {backend} {dict(options)} {env or ''}] " +
              ", ".join(f"{k}/{s}: {r:.3g}" for (k, s), r in sorted(chk.ratios.items())) +
              f"; off-grid (step, op): {sorted(chk.off_grid)}; stem columns: {chk.stem}; unstored tangents per step: {unwritten}")
    return chk


@pytest.mark.parametrize("backend", ["simt", "tc"])
def test_fedavg_convnet_every_step_buffer(backend):
    """The fedavg_convnet fixture: 3 steps x 2 images over 4 images, the third step wraps onto images 0-1."""
    chk = check_engine("fedavg-convnet", backend)
    assert chk.glue.offsets == [0, 2, 0]


@pytest.mark.parametrize("backend", ["simt", "tc"])
def test_config4_structure_every_step_buffer(backend):
    """BASELINE config 4 at 64 x 64: ResNet-18, 4 steps x 1 image, `modern` without the features prior."""
    chk = check_engine("resnet18-64", backend)
    if backend == "tc":
        assert chk.stem == [0]


@pytest.mark.parametrize("switch", ["fuse_bnact", "overlap_wgrad", "stem_cols"])
def test_tensor_core_switches_every_step_buffer(switch, monkeypatch):
    """Each switch in both settings (the default is the control): the fused BN epilogue, whose pre-BN tangent a step k > 0 must
    store for its gamma tangent; the tangent weight gradients on the side stream; the stem off its column path."""
    for value in (0, 1):
        if switch == "stem_cols":
            chk = check_engine("resnet18-64", "tc", env={"BRE_STEM_COLS": str(value)}, monkeypatch=monkeypatch)
            assert chk.stem == ([0] if value else [])
            continue
        chk = check_engine("resnet18-64", "tc", options=((switch, value),))
        if switch == "fuse_bnact" and value:
            assert chk.unwritten[0] and not any(chk.unwritten[1:]), chk.unwritten


def test_config4_at_full_size_every_step_buffer():
    """BASELINE config 4 itself: ResNet-18 at 224 x 224, 4 steps x 1 image, tensor cores."""
    check_engine("config4", "tc")


def _everything(eng):
    out = read_tensors(eng, WHICH)
    out.update(read_params(eng, ("G", "v", "v_operand", "W", "W_operand")))
    return out


def test_multistep_stop_is_neutral():
    """Stopped evaluations leave no trace: after every stop and a reset to 0, objective, gradient and every buffer are bitwise
    those of a fresh engine.  ``run`` refuses while a stop is set."""
    case = build_case("fedavg-convnet")
    x, K = case[4].to(DEV), case[2]["steps"]
    fresh = make_engine(case, "tc")
    val0, grad0 = fresh.objective_and_gradient(x)
    ref = _everything(fresh)
    fresh.close()
    eng = make_engine(case, "tc")
    for s in range(1, 2 * K + 1):
        eng.set_option("debug_multistep_stop", s)
        eng.objective_and_gradient(x)
    eng.begin_trial(x, lr_table(0.1, "step-lr", 0, 24000, 4))
    with pytest.raises(EngineError):
        eng.run(1)
    eng.set_option("debug_multistep_stop", 0)
    val1, grad1 = eng.objective_and_gradient(x)
    assert val1 == val0 and torch.equal(grad1, grad0)
    got = _everything(eng)
    for key, t in ref.items():
        assert torch.equal(got[key], t), key
    eng.close()
