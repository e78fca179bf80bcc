"""The multi-step (FedAvg) interpreter and checker on the CPU: the float64 restatement of the engine's multi-step evaluation
(oracle/program_interp.MultiStepInterpreter) equals float64 autograd of the reference's ``_grad_fn_multi_step``; every
relation of the multi-step checker (oracle/sweep_check.MultiStepChecker) holds to rounding level on its buffers; and a buffer
corrupted the way a faulty kernel or a faulty step of the glue would corrupt it is reported at exactly the (step, op, sweep)
that produced it."""
import copy

import pytest
import torch

from breaching_b200 import compiler, get_attack_config, synthetic
from helpers import sweep_objective
from oracle import program_interp as PI
from oracle import restate
from oracle.sweep_check import InterpreterGlue, InterpreterStepSource, MultiStepChecker

CASES = {
    # the fedavg_convnet fixture case: 3 steps x 2 images over 4 images, so step 2 wraps onto images 0-1
    "convnet-tiny": dict(model_name="convnet-tiny", data="cifar", num_data_points=4, steps=3, data_per_step=2, lr=0.05, seed=4,
                         bn_random=True),
    "resnet18": dict(model_name="resnet18", data="imagenet", num_data_points=4, steps=4, data_per_step=1, lr=1e-2, seed=6,
                     bn_random=True, image_size=32, classes=10),
}


def _case(name):
    model, loss_fn, payload, shared, true = synthetic.make_fedavg_case(**CASES[name])
    cfg = get_attack_config("modern", {"regularization.features.scale": 0.0})
    local = shared[0]["metadata"]["local_hyperparams"]
    x = torch.randn(true["data"].shape, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    return model.eval(), loss_fn, payload, shared, cfg, local, x


def run_multistep(name, tamper=None):
    model, loss_fn, payload, shared, cfg, local, x = _case(name)
    m64 = copy.deepcopy(model).double().eval()
    prog = compiler.compile_model(m64, (local["data_per_step"], *x.shape[1:]))
    mi = PI.MultiStepInterpreter(m64, prog, local["lr"])
    mi.tamper = tamper
    g64 = [g.double() for g in shared[0]["gradients"]]
    obj = sweep_objective(cfg)
    val, grad = mi.run(x, local["labels"], g64, obj)
    bn = [None if (m is None or m.running_mean is None) else (m.running_mean.double(), m.running_var.double())
          for m in compiler.bn_modules(m64, prog)]
    chk = MultiStepChecker(prog, bn, g64, local["labels"], obj,
                           [InterpreterStepSource(mi, k) for k in range(local["steps"])], InterpreterGlue(mi, x, grad))
    return mi, chk, val, grad, (model, loss_fn, payload, shared, cfg, local, x)


@pytest.mark.parametrize("name", list(CASES))
def test_multistep_interpreter_matches_reference_autograd(name):
    mi, _, val, grad, (model, loss_fn, payload, shared, cfg, local, x) = run_multistep(name)
    meta = payload[0]["metadata"]
    dm = torch.tensor(meta.mean, dtype=torch.float64)[None, :, None, None]
    ds = torch.tensor(meta.std, dtype=torch.float64)[None, :, None, None]
    orc = restate.TrialOracle(copy.deepcopy(model).double().eval(), loss_fn, cfg, [g.double() for g in shared[0]["gradients"]],
                              torch.cat(local["labels"]), dm, ds, dtype=torch.float64, local_hyperparams=local)
    phi, _, raw, _ = orc.closure_gradient(x, 0, 0.0)
    orc.close()
    assert abs(float(val) - float(phi)) <= 1e-10 * max(1.0, abs(float(phi))), (float(val), float(phi))
    rel = ((grad - raw).norm() / raw.norm()).item()
    assert rel < 1e-10, rel
    if name == "convnet-tiny":
        assert mi.offsets == [0, 2, 0]   # the third step wraps onto images 0-1


@pytest.mark.parametrize("name", list(CASES))
def test_checker_holds_on_interpreter_buffers(name):
    _, chk, _, _, _ = run_multistep(name)
    chk.check()
    worst = max(chk.ratios.values())
    assert worst < 1e-6, sorted(chk.ratios.items(), key=lambda kv: -kv[1])[:5]
    sweeps = {s for _, s in chk.ratios}
    assert {"F", "B", "V", "TF", "TB", "TG", "W", "Wt", "D", "U", "Ut", "GX"} <= sweeps, sweeps


def _flagged(chk):
    return {(f.step, f.op, f.sweep) for f in chk.check(raise_on_failure=False)}


def test_gamma_tangent_without_pre_bn_term_is_reported():
    """The shape of the old fuse_bnact defect: the BN gamma tangent of a step k > 0 without its pre-BN-tangent term."""
    holder = {}

    def tamper(step, sweep, oi, key, stored, contribution=None):
        if step == 2 and sweep == "TG" and oi == holder["i"] and key == holder["op"].gamma:
            it, op = holder["mi"].steps[2], holder["op"]
            return stored - (it.du_B[oi] * it.ta[op.tin] * it._bn_consts(oi, op)[1]).sum(dim=(0, 2, 3))
        return stored

    holder["mi"], chk = _rerun("resnet18", tamper)
    prog = chk.prog
    holder["i"] = [j for j, op in enumerate(prog.ops) if op.kind == compiler.OP_BNACT and op.has_bn][3]
    holder["op"] = prog.ops[holder["i"]]
    assert _flagged(chk) == {(2, holder["i"], "TG")}


def test_single_source_tangent_wgrad_is_reported():
    """A tangent weight gradient without its second source wgrad(a', d_B), at the first conv that does not read the candidate."""
    holder = {}

    def tamper(step, sweep, oi, key, stored, contribution=None):
        op = holder["op"]
        if step == 1 and sweep == "TG" and oi == holder["i"] and key == op.w:
            it = holder["mi"].steps[1]
            return stored - torch.nn.grad.conv2d_weight(it.ta[op.tin], stored.shape, it.d_B[op.tout], stride=op.stride, padding=op.pad)
        return stored

    holder["mi"], chk = _rerun("convnet-tiny", tamper)
    holder["i"] = [j for j, op in enumerate(chk.prog.ops) if op.kind == compiler.OP_CONV and op.tin != 0][0]
    holder["op"] = chk.prog.ops[holder["i"]]
    assert _flagged(chk) == {(1, holder["i"], "TG")}


def _rerun(name, tamper):
    """run_multistep with a tamper hook that may read the interpreter it runs in (``holder`` pattern)."""
    model, loss_fn, payload, shared, cfg, local, x = _case(name)
    m64 = copy.deepcopy(model).double().eval()
    prog = compiler.compile_model(m64, (local["data_per_step"], *x.shape[1:]))
    mi = PI.MultiStepInterpreter(m64, prog, local["lr"])
    mi.tamper = tamper
    g64 = [g.double() for g in shared[0]["gradients"]]
    obj = sweep_objective(cfg)
    bn = [None if (m is None or m.running_mean is None) else (m.running_mean.double(), m.running_var.double())
          for m in compiler.bn_modules(m64, prog)]
    return mi, _Deferred(mi, x, local, prog, bn, g64, obj)


class _Deferred:
    """The checker of a tampered run, built once the run (started by ``_flagged``) has finished."""

    def __init__(self, mi, x, local, prog, bn, g64, obj):
        self.mi, self.x, self.local, self.prog, self.bn, self.g64, self.obj = mi, x, local, prog, bn, g64, obj

    def check(self, raise_on_failure=True):
        _, grad = self.mi.run(self.x, self.local["labels"], self.g64, self.obj)
        chk = MultiStepChecker(self.prog, self.bn, self.g64, self.local["labels"], self.obj,
                               [InterpreterStepSource(self.mi, k) for k in range(self.local["steps"])],
                               InterpreterGlue(self.mi, self.x, grad))
        return chk.check(raise_on_failure=raise_on_failure)


def test_overwritten_wrapped_gradient_slice_is_reported():
    """Step 0 overwrites the candidate-gradient slice that the wrapped step 2 already accumulated into."""
    def tamper(step, sweep, oi, key, stored, contribution=None):
        return contribution if (step == 0 and sweep == "GX") else stored

    _, chk = _rerun("convnet-tiny", tamper)
    assert _flagged(chk) == {(None, -1, "GX")}


def test_adjoint_update_with_stale_tangent_G_is_reported():
    """u_1 formed with the tangent parameter gradients of step 2 instead of step 1."""
    lr = CASES["convnet-tiny"]["lr"]
    seen = {}

    def tamper(step, sweep, oi, key, stored, contribution=None):
        if sweep == "U":
            seen[step] = contribution
            if step == 1:
                return [s + lr * (c - old) for s, c, old in zip(stored, contribution, seen[2])]
        return stored

    _, chk = _rerun("convnet-tiny", tamper)
    assert _flagged(chk) == {(1, -1, "U")}


def test_weights_from_the_wrong_step_gradient_are_reported():
    """W_2 formed from G_0 instead of G_1."""
    lr = CASES["convnet-tiny"]["lr"]
    seen = {}

    def tamper(step, sweep, oi, key, stored, contribution=None):
        if sweep == "W":
            seen[step] = contribution
            if step == 1:
                return [s + lr * (c - old) for s, c, old in zip(stored, contribution, seen[0])]
        return stored

    _, chk = _rerun("convnet-tiny", tamper)
    assert _flagged(chk) == {(1, -1, "W")}
