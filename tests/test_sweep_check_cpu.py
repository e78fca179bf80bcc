"""The layer-local sweep checker (oracle/sweep_check.py) on the float64 four-sweep interpreter: every relation it checks holds
to rounding level on the interpreter's own buffers, and a buffer corrupted the way a faulty kernel would corrupt it (the
ops that read it see the corrupted value) is reported at exactly the op and sweep that produced it."""
import copy

import pytest
import torch

from breaching_b200 import compiler, get_attack_config, synthetic
from helpers import odd_case, sweep_objective
from oracle import program_interp as PI
from oracle.sweep_check import InterpreterSource, SweepChecker


def _synthetic(name, size, no_buffers=False, seed=11):
    data = "cifar" if size == 32 else "imagenet"
    model, _, _, shared, true = synthetic.make_case(name, data, batch=2, seed=seed, bn_random=True, image_size=size, classes=10,
                                                    no_buffers=no_buffers)
    return model, (2, 3, size, size), true["labels"], shared[0]["gradients"]


def _case(name):
    if name == "odd":
        return odd_case()
    if name == "convnet-tiny":
        return _synthetic("convnet-tiny", 32)
    if name == "trainbn-convnet-tiny":
        return _synthetic("convnet-tiny", 32, no_buffers=True)
    return _synthetic(name, 32)


def run_interpreter(model, shape, labels, grads, obj, seed=3, tamper=None):
    """float64 four sweeps + priors; returns the checker fed with the interpreter's buffers."""
    m64 = copy.deepcopy(model).double()
    prog = compiler.compile_model(m64, shape)
    it = PI.ProgramInterpreter(m64, prog)
    it.tamper = tamper
    x = torch.randn(shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)

    def inject_fn(it_):
        inj = {}
        parts = []
        if obj.get("di") is not None:
            parts.append(it_.deep_inversion(obj["di"]["scale"], obj["di"]["first_bn_multiplier"])[1])
        if obj.get("features") is not None:
            parts.append(it_.feature_regularization(obj["features"]["measured"], obj["features"]["scale"])[1])
        for p in parts:
            for k, v in p.items():
                inj[k] = inj.get(k, 0) + v
        return inj or None

    g64 = [g.double() for g in grads]
    _, dx, _, _ = it.matching_gradient(x, labels, g64, obj["kind"], scale=obj["scale"], task_regularization=obj["task_regularization"],
                                       inject_fn=inject_fn)
    from oracle import restate

    xd = x.clone().requires_grad_(True)
    prior = xd.sum() * 0
    if obj.get("tv") is not None:
        prior = prior + restate.total_variation(xd, scale=obj["tv"]["scale"])
    if obj.get("norm") is not None:
        prior = prior + restate.norm_regularization(xd, scale=obj["norm"]["scale"], pnorm=obj["norm"]["p"])
    (gp,) = torch.autograd.grad(prior, xd)
    return SweepChecker(prog, it.P, it.bn, g64, labels, obj, InterpreterSource(it, dx + gp)), prog


def _objective(name):
    if name == "resnet18":   # every prior the checker knows
        cfg = get_attack_config("invertinggradients", {"objective.task_regularization": 0.1, "regularization.norm.scale": 1e-3,
                                                        "regularization.deep_inversion.scale": 1e-3,
                                                        "regularization.features.scale": 0.1})
        feats = torch.randn(2, 512, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
        return sweep_objective(cfg, features=feats)
    return sweep_objective(get_attack_config("invertinggradients"))


CASES = ["convnet-tiny", "resnet18", "resnet50", "trainbn-convnet-tiny", "odd"]


@pytest.mark.parametrize("name", CASES)
def test_interpreter_buffers_satisfy_every_relation(name):
    model, shape, labels, grads = _case(name)
    chk, prog = run_interpreter(model, shape, labels, grads, _objective(name))
    chk.check()
    # float64 buffers against fp32 rounding bounds: every relation holds far below its bound (~1e-12 relative)
    worst = max(chk.ratios.values())
    assert worst < 1e-6, sorted(chk.ratios.items(), key=lambda kv: -kv[1])[:5]
    kinds = {k for k, _ in chk.ratios}
    assert {"conv", "bnact", "linear"} <= kinds
    sweeps = {s for _, s in chk.ratios}
    assert sweeps == {"F", "B", "V", "TF", "TB"}


def _flagged(chk):
    return {(f.op, f.sweep) for f in chk.check(raise_on_failure=False)}


@pytest.mark.parametrize("name", ["convnet-tiny", "odd", "resnet18"])
def test_scaled_tangent_channel_is_reported_at_its_producer(name):
    model, shape, labels, grads = _case(name)
    prog = compiler.compile_model(copy.deepcopy(model).double(), shape)
    target = [i for i, op in enumerate(prog.ops) if op.kind == compiler.OP_CONV][2]

    def tamper(sweep, i, tid, stored, contribution=None):
        if sweep == "TF" and i == target:
            stored = stored.clone()
            stored[:, 1] *= 1.001
        return stored

    chk, _ = run_interpreter(model, shape, labels, grads, _objective(name), tamper=tamper)
    assert _flagged(chk) == {(target, "TF")}


@pytest.mark.parametrize("name", ["convnet-tiny", "odd", "resnet18"])
def test_swapped_delta_pixels_are_reported_where_the_delta_is_final(name):
    model, shape, labels, grads = _case(name)
    prog = compiler.compile_model(copy.deepcopy(model).double(), shape)
    t = [op.tout for op in prog.ops if op.kind == compiler.OP_BNACT][1]
    last = min(i for i, op in enumerate(prog.ops) if t in (op.tin, op.res))

    def tamper(sweep, i, tid, stored, contribution=None):
        if sweep == "B" and i == last and tid == t:
            stored = stored.clone()
            flat = stored[0, 0].flatten()
            nz = flat.nonzero().flatten()
            j, k = int(nz[0]), int(nz[-1])
            assert flat[j] != flat[k]
            flat[j], flat[k] = flat[k].clone(), flat[j].clone()
            stored[0, 0] = flat.view_as(stored[0, 0])
        return stored

    chk, _ = run_interpreter(model, shape, labels, grads, _objective(name), tamper=tamper)
    assert _flagged(chk) == {(last, "B")}


def _branch_point(prog, kind):
    """(op index, tensor) of an accumulation: ``conv``: the residual branch point of the first residual op (a conv accumulates into
    its delta); ``bnact-in`` / ``bnact-res``: a BN / ReLU / add op with ``acc_in`` / ``acc_res``, ``-scalar`` on C % 4 != 0 channels
    (scalar kernels), ``-vec`` on C % 4 == 0 (float4 kernels)."""
    consumers = lambda t: [i for i, op in enumerate(prog.ops) if t in (op.tin, op.res)]  # noqa: E731
    if kind == "conv":
        first_res = next(op for op in prog.ops if op.res >= 0)
        t = next(t for t in (first_res.res, first_res.tin) if len(consumers(t)) == 2)
        return min(consumers(t)), t
    field, width = kind.split("-")[1:]
    for i, op in enumerate(prog.ops):
        vec = prog.tensors[op.tout].C % 4 == 0
        if op.kind == compiler.OP_BNACT and getattr(op, f"acc_{field}") and vec == (width == "vec"):
            t = op.tin if field == "in" else op.res
            assert min(consumers(t)) == i   # this op's write makes the buffer final
            return i, t
    raise AssertionError(f"no {kind} accumulation in the program")


@pytest.mark.parametrize("name,kind", [("resnet18", "conv"), ("odd", "conv"), ("odd", "bnact-in-scalar"), ("odd", "bnact-res-scalar"),
                                       ("odd", "bnact-in-vec"), ("odd", "bnact-res-vec")])
@pytest.mark.parametrize("sweep", ["B", "TB"])
def test_dropped_accumulation_is_reported(name, kind, sweep):
    """The last consumer of a tensor with two consumers overwrites the delta instead of accumulating into it."""
    model, shape, labels, grads = _case(name)
    prog = compiler.compile_model(copy.deepcopy(model).double(), shape)
    last, t = _branch_point(prog, kind)

    def tamper(sweep_, i, tid, stored, contribution=None):
        return contribution if (sweep_ == sweep and i == last and tid == t) else stored

    chk, _ = run_interpreter(model, shape, labels, grads, _objective(name), tamper=tamper)
    assert _flagged(chk) == {(last, sweep)}


@pytest.mark.parametrize("kind", ["euclidean", "l1", "tag-euclidean"])
def test_other_objectives_direction(kind):
    model, shape, labels, grads = _case("convnet-tiny")
    obj = sweep_objective(get_attack_config("invertinggradients", {"objective.type": kind, "objective.scale": 0.5}))
    chk, _ = run_interpreter(model, shape, labels, grads, obj)
    chk.check()
    assert chk.ratios[("objective", "V")] < 1e-6
