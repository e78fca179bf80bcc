"""FedAvg (multi-step) updates with the priors of the last local step -- task-loss regularisation and DeepInversion -- on the
CPU: the reference's own outputs (tests/golden/trial_fedavg_{taskreg,di}_*.pt) against the oracle restatement; the float64
restatement of the engine's evaluation (``oracle.fedavg_priors.PriorMultiStepInterpreter``: the priors enter the last step's tangent backward as seeds
scaled by -1/lr) against float64 autograd of the reference closure; and the multi-step checker on its buffers, including a
corrupted seed reported at exactly the (step, op, sweep) that produced it."""
import copy
import math

import pytest
import torch

from breaching_b200 import compiler, get_attack_config, synthetic
from helpers import load_golden, oracle_for_fixture, sweep_objective
from oracle import restate
from oracle.fedavg_priors import PriorMultiStepChecker, PriorMultiStepInterpreter, PriorStepSource
from oracle.sweep_check import InterpreterGlue

FEDAVG_PRIOR_FIXTURES = ["fedavg_taskreg_convnet", "fedavg_di_convnet", "fedavg_di_resnet18"]
PRIORS = {"regularization.features.scale": 0.0, "regularization.deep_inversion.scale": 0.01, "objective.task_regularization": 0.1}
TASK_ONLY = {"regularization.features.scale": 0.0, "objective.task_regularization": 0.1}
CASES = {
    # 3 steps x 2 images over 4 images: step 2 wraps onto images 0-1
    "convnet-tiny": (dict(model_name="convnet-tiny", data="cifar", num_data_points=4, steps=3, data_per_step=2, lr=0.05, seed=4,
                          bn_random=True), PRIORS),
    "convnet-tiny-task": (dict(model_name="convnet-tiny", data="cifar", num_data_points=4, steps=3, data_per_step=2, lr=0.05, seed=4,
                               bn_random=True), TASK_ONLY),
    "resnet18": (dict(model_name="resnet18", data="imagenet", num_data_points=4, steps=4, data_per_step=1, lr=1e-2, seed=6,
                      bn_random=True, image_size=32, classes=10), PRIORS),
    # K = 1: no adjoint update, only the candidate term of the seeds
    "convnet-tiny-k1": (dict(model_name="convnet-tiny", data="cifar", num_data_points=2, steps=1, data_per_step=2, lr=0.05, seed=4,
                             bn_random=True), PRIORS),
}


@pytest.mark.parametrize("name", FEDAVG_PRIOR_FIXTURES)
def test_oracle_reproduces_reference_fixture(name):
    """The tolerances of tests/test_golden_oracle.py: trajectories to 2e-4, the first candidate to 1e-4."""
    fx = load_golden(f"trial_{name}.pt")
    orc, cfg, labels = oracle_for_fixture(fx)
    assert labels.tolist() == fx["labels"].tolist()
    phi0, _, raw, terms = orc.closure_gradient(fx["x0"], 0, 0.0)
    assert math.isclose(float(phi0), fx["objective0"], rel_tol=1e-5, abs_tol=1e-7)
    assert math.isclose(terms["task_loss"], fx["task_loss0"], rel_tol=1e-5, abs_tol=1e-7)
    assert ((raw - fx["raw_grad0"]).norm() / fx["raw_grad0"].norm()).item() < 1e-4
    best, hist, trace = orc.run(fx["x0"], iterations=fx["iters"], record=True)
    assert len(hist) == len(fx["history"])
    for a, b in zip(hist, fx["history"]):
        assert math.isclose(a, b, rel_tol=2e-4, abs_tol=1e-6), (hist, fx["history"])
    assert (trace[0]["candidate"] - fx["candidate_after_1"]).abs().max().item() < 1e-4
    assert (trace[-1]["candidate"] - fx["candidate_final"]).abs().mean().item() < 2e-3
    assert math.isclose(orc.score(best, fx["scoring"]), fx["score"], rel_tol=5e-2, abs_tol=1e-5)
    orc.close()


def _case(name):
    kw, over = CASES[name]
    model, loss_fn, payload, shared, true = synthetic.make_fedavg_case(**kw)
    cfg = get_attack_config("modern", dict(over))
    local = shared[0]["metadata"]["local_hyperparams"]
    x = torch.randn(true["data"].shape, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    return model.eval(), loss_fn, payload, shared, cfg, local, x


def run_multistep(name, tamper=None):
    model, loss_fn, payload, shared, cfg, local, x = _case(name)
    m64 = copy.deepcopy(model).double().eval()
    prog = compiler.compile_model(m64, (local["data_per_step"], *x.shape[1:]))
    mi = PriorMultiStepInterpreter(m64, prog, local["lr"])
    mi.tamper = tamper
    g64 = [g.double() for g in shared[0]["gradients"]]
    obj = sweep_objective(cfg)
    val, grad = mi.run(x, local["labels"], g64, obj)
    bn = [None if (m is None or m.running_mean is None) else (m.running_mean.double(), m.running_var.double())
          for m in compiler.bn_modules(m64, prog)]
    chk = PriorMultiStepChecker(prog, bn, g64, local["labels"], obj,
                                [PriorStepSource(mi, k) for k in range(local["steps"])], InterpreterGlue(mi, x, grad))
    return mi, chk, val, grad, (model, loss_fn, payload, shared, cfg, local, x)


@pytest.mark.parametrize("name", list(CASES))
def test_interpreter_matches_reference_autograd(name):
    mi, _, val, grad, (model, loss_fn, payload, shared, cfg, local, x) = run_multistep(name)
    meta = payload[0]["metadata"]
    dm = torch.tensor(meta.mean, dtype=torch.float64)[None, :, None, None]
    ds = torch.tensor(meta.std, dtype=torch.float64)[None, :, None, None]
    orc = restate.TrialOracle(copy.deepcopy(model).double().eval(), loss_fn, cfg, [g.double() for g in shared[0]["gradients"]],
                              torch.cat(local["labels"]), dm, ds, dtype=torch.float64, local_hyperparams=local)
    phi, _, raw, terms = orc.closure_gradient(x, 0, 0.0)
    orc.close()
    assert abs(float(val) - float(phi)) <= 1e-10 * max(1.0, abs(float(phi))), (float(val), float(phi))
    assert ((grad - raw).norm() / raw.norm()).item() < 1e-10
    # the priors are really on: without them the value and gradient differ
    assert mi.seeds is not None and terms["task_loss"] > 0
    if "deep_inversion" in terms:
        assert terms["deep_inversion"] > 0


@pytest.mark.parametrize("name", list(CASES))
def test_checker_holds_on_interpreter_buffers(name):
    _, chk, _, _, _ = run_multistep(name)
    chk.check()
    worst = max(chk.ratios.values())
    assert worst < 1e-6, sorted(chk.ratios.items(), key=lambda kv: -kv[1])[:5]


def test_zero_step_size_with_a_prior_is_refused():
    model, loss_fn, payload, shared, cfg, local, x = _case("convnet-tiny-task")
    m64 = copy.deepcopy(model).double().eval()
    prog = compiler.compile_model(m64, (local["data_per_step"], *x.shape[1:]))
    with pytest.raises(ValueError, match="lr must be nonzero"):
        PriorMultiStepInterpreter(m64, prog, 0.0).run(x, local["labels"], [g.double() for g in shared[0]["gradients"]], sweep_objective(cfg))


# ---- tampers: each is reported at exactly the (step, op, sweep) it corrupts -----------------------------------------------
def _flagged(name, tamper):
    _, chk, _, _, _ = run_multistep(name, tamper)
    return {(f.step, f.op, f.sweep) for f in chk.check(raise_on_failure=False)}, chk


def _bn_ops(prog):
    return {i for i, op in enumerate(prog.ops) if op.kind == compiler.OP_BNACT and op.has_bn}


def test_seed_at_the_wrong_step_is_reported():
    """The task-loss seed given to step K - 2 instead of the last step: both logits seeds are wrong."""
    def tamper(step, sweep, oi, key, stored, contribution=None):
        if sweep == "SEED":
            return contribution if step == 1 else None
        return stored

    found, chk = _flagged("convnet-tiny-task", tamper)
    head = len(chk.prog.ops) - 1
    assert found == {(2, head, "TB"), (1, head, "TB")}, found


def test_seed_without_the_step_size_factor_is_reported():
    """The seeds without their -1/lr factor (the prior adjoints as in a single-step evaluation): the logits seed of the last step
    and every DeepInversion adjoint at its BN inputs."""
    lr = CASES["convnet-tiny"][0]["lr"]

    def tamper(step, sweep, oi, key, stored, contribution=None):
        if sweep == "SEED" and stored is not None:
            c, inject = stored
            return c * -lr, {t: a * -lr for t, a in inject.items()}
        return stored

    found, chk = _flagged("convnet-tiny", tamper)
    assert found == {(2, len(chk.prog.ops) - 1, "TB")} | {(2, i, "TB") for i in _bn_ops(chk.prog)}, found


def test_prior_on_the_candidate_only_is_reported():
    """u_last formed without the priors' parameter gradients (tau G_last + dR_DI / dW_last): the adjoint update of the last step."""
    lr = CASES["convnet-tiny"][0]["lr"]
    plain, _, _, _, _ = run_multistep("convnet-tiny", lambda step, sweep, oi, key, stored, contribution=None:
                                      None if sweep == "SEED" else stored)
    tg_plain = plain.steps[2].TG

    def tamper(step, sweep, oi, key, stored, contribution=None):
        if sweep == "U" and step == 2:
            return [s + lr * (c - c0) for s, c, c0 in zip(stored, contribution, tg_plain)]
        return stored

    found, _ = _flagged("convnet-tiny", tamper)
    assert found == {(2, -1, "U")}, found


def test_deep_inversion_statistics_of_the_wrong_step_are_reported():
    """The DeepInversion adjoints built from step 1's forward instead of the last step's: every BN input of the last step."""
    def tamper(step, sweep, oi, key, stored, contribution=None):
        return 1 if sweep == "DI" else stored

    found, chk = _flagged("convnet-tiny", tamper)
    assert found == {(2, i, "TB") for i in _bn_ops(chk.prog)}, found
