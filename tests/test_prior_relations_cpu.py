"""The orthogonality relation of the float64 sweep checker (oracle/sweep_check.orthogonality_relation) against autograd of the
reference's OrthogonalityRegularization (oracle/restate.py) in float64; an fp32 emulation of ``orthogonality_kernel`` passes it, and
the faults a kernel could make (the gradient without its ``-x_ik^2`` self term, the value without ``- Q_k``) are reported.  Also the
rule that picks the layers of the DeepInversion and feature priors: the first *registered* BatchNorm2d and the last *registered*
Linear, in the compiler, the checker and the reference's own objective."""
import copy

import pytest
import torch

from breaching_b200 import compiler, get_attack_config
from helpers import BNRegisteredLate, LinearRegisteredLast, registration_case, sweep_objective
from oracle import restate
from oracle.sweep_check import SweepChecker, orthogonality_relation, worst_element
from test_sweep_check_cpu import _case, assemble, interpreter_terms, run_interpreter

SHAPES = [(2, 3, 5, 7), (3, 1, 4, 4), (5, 2, 3, 9), (17, 3, 2, 2)]


def _x(shape, seed=0):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)


def kernel_fp32(x, self_term=True, subtract_q=True):
    """``orthogonality_kernel`` emulated in fp32: per position the batch loop of fp32 squares, adds and fmas, the value in double,
    the gradient ``scale * v * (S - v * v)``; optionally with one of the faults a kernel could make."""
    N = x.shape[0]
    xf = x.reshape(N, -1).to(torch.float32)
    D = xf.shape[1]
    S = torch.zeros(D, dtype=torch.float32)
    Q = torch.zeros(D, dtype=torch.float32)
    for j in range(N):
        v2 = xf[j] * xf[j]
        S = S + v2
        Q = (v2.double() * v2.double() + Q.double()).to(torch.float32)   # fmaf: one rounding
    val = float((S.double() * S.double() - (Q.double() if subtract_q else 0.0)).sum()) / D
    scale = torch.tensor(4.0 / D, dtype=torch.float32)
    grad = (scale * xf) * ((S - xf * xf) if self_term else S)
    return val, grad.double().view_as(x)


@pytest.mark.parametrize("shape", SHAPES)
def test_relation_is_autograd_of_the_reference(shape):
    x = _x(shape).requires_grad_(True)
    ref = restate.orthogonality_regularization(x)
    (g,) = torch.autograd.grad(ref, x)
    val, vb, grad, gb = orthogonality_relation(x.detach())
    assert abs(val - float(ref.detach())) <= 1e-12 * abs(float(ref.detach()))
    assert torch.allclose(grad, g, rtol=1e-12, atol=1e-15)
    assert vb > 0 and bool((gb > 0).all())


def test_single_image_is_exactly_zero():
    val, vb, grad, gb = orthogonality_relation(_x((1, 3, 4, 4)))
    assert (val, vb) == (0.0, 0.0) and not grad.any() and not gb.any()
    assert restate.orthogonality_regularization(_x((1, 3, 4, 4))) == 0


@pytest.mark.parametrize("shape", SHAPES)
def test_fp32_kernel_passes_and_its_faults_are_reported(shape):
    x = _x(shape, seed=1).to(torch.float32).double()
    ref, vb, gref, gb = orthogonality_relation(x)
    val, grad = kernel_fp32(x)
    assert abs(val - ref) <= vb
    assert worst_element(grad, gref, gb)[0] <= 1.0
    _, bad = kernel_fp32(x, self_term=False)
    assert worst_element(bad, gref, gb)[0] > 1.0
    bad_val, _ = kernel_fp32(x, subtract_q=False)
    assert abs(bad_val - ref) > vb


# ---- through the checker: the candidate-gradient relation of sweep TB and the norm slot of the terms -----------------------------
def _ortho_run(name, norm):
    """The float64 interpreter on ``name`` with orthogonality on (and the norm prior if ``norm``); the interpreter's candidate
    gradient gets the orthogonality gradient, as the engine adds it after the other priors."""
    over = {"regularization.orthogonality.scale": 0.5}
    if norm:
        over["regularization.norm.scale"] = 1e-2
    obj = sweep_objective(get_attack_config("invertinggradients", over))
    assert obj["orthogonality"] is True
    model, shape, labels, grads = _case(name)
    chk, _ = run_interpreter(model, shape, labels, grads, obj)
    clean = chk.src.grad_x
    chk.src.grad_x = clean + orthogonality_relation(chk.x0)[2]
    return chk, obj, clean


@pytest.mark.parametrize("fault", [None, "self term", "not added"])
def test_candidate_gradient_relation(fault):
    chk, obj, clean = _ortho_run("odd", norm=True)
    x = chk.x0
    if fault == "self term":
        N = x.shape[0]
        xf = x.reshape(N, -1)
        chk.src.grad_x = clean + (4.0 / xf.shape[1] * xf * (xf * xf).sum(dim=0)).view_as(x)
    elif fault == "not added":
        chk.src.grad_x = clean
    flagged = {(f.op, f.sweep, f.what) for f in chk.check(raise_on_failure=False)}
    if fault is None:
        assert not flagged and chk.ratios[("bnact", "TB")] < 1e-6
    else:
        assert flagged == {(chk.first_consumer[0], "TB", "tangent_delta[t0] (candidate gradient)")}


@pytest.mark.parametrize("fault", [None, "without Q", "overwritten"])
def test_term_is_accumulated_into_the_norm_slot(fault):
    model, shape, labels, grads = _case("resnet18")
    obj = sweep_objective(get_attack_config("invertinggradients", {
        "objective.task_regularization": 0.125, "regularization.total_variation.scale": 0.25, "regularization.norm.scale": 2.0 ** -10,
        "regularization.deep_inversion.scale": 2.0 ** -10, "regularization.features.scale": 0.125,
        "regularization.orthogonality.scale": 1.0}), features=torch.randn(2, 512, generator=torch.Generator().manual_seed(2),
                                                                          dtype=torch.float64))
    chk, _ = run_interpreter(model, shape, labels, grads, obj)
    terms, _ = interpreter_terms(chk, obj)
    x = chk.x0
    N = x.shape[0]
    x2 = x.reshape(N, -1) ** 2
    ortho = float((x2.sum(0) ** 2 - (x2 ** 2).sum(0)).sum()) / x2.shape[1]
    assert ortho == pytest.approx(float(restate.orthogonality_regularization(x)), rel=1e-12)
    if fault == "without Q":
        ortho = float((x2.sum(0) ** 2).sum()) / x2.shape[1]
    if fault != "overwritten":   # the orthogonality kernel overwrote the norm prior's value instead of adding to it
        terms["norm"] += ortho
    else:
        terms["norm"] = ortho
    flagged = {f.sweep for f in chk.check_terms(terms, assemble(terms, obj), raise_on_failure=False)}
    assert flagged == (set() if fault is None else {"norm"})


def test_absent_orthogonality_leaves_the_relations_as_they_were():
    obj = sweep_objective(get_attack_config("invertinggradients"))
    assert "orthogonality" not in obj
    obj = sweep_objective(get_attack_config("invertinggradients", {"regularization.orthogonality.scale": 0.0}))
    assert "orthogonality" not in obj


# ---- which layers the DeepInversion and feature priors read ------------------------------------------------------------------------
def _prog(cls, in_order):
    model, shape, labels, grads = registration_case(cls, in_order)
    return model, compiler.compile_model(model, shape), labels, grads


def test_compiler_and_checker_follow_registration_order():
    for in_order in (False, True):
        model, prog, labels, grads = _prog(BNRegisteredLate, in_order)
        bn_ops = [i for i, op in enumerate(prog.ops) if op.has_bn]
        assert prog.ops[prog.di_first_op].bn_module == ("bn1" if in_order else "bn2")
        assert prog.di_first_op == (bn_ops[1] if not in_order else bn_ops[0])
        chk = SweepChecker(prog, list(model.parameters()), [None] * len(prog.ops), grads, labels, {"kind": "euclidean"}, None)
        assert chk._first_bn() == prog.di_first_op
        model, prog, labels, grads = _prog(LinearRegisteredLast, in_order)
        lin_ops = [i for i, op in enumerate(prog.ops) if op.kind == compiler.OP_LINEAR]
        assert prog.ops[prog.feature_op].module == ("proj" if not in_order else "fc")
        assert prog.feature_op == (lin_ops[0] if not in_order else lin_ops[-1])
        chk = SweepChecker(prog, list(model.parameters()), [None] * len(prog.ops), grads, labels, {"kind": "euclidean"}, None)
        assert chk._feature_op() == prog.feature_op


@pytest.mark.parametrize("cls,key", [(BNRegisteredLate, "deep_inversion"), (LinearRegisteredLast, "features")])
def test_reference_objective_depends_on_registration_order(cls, key):
    """The reference's own objective (restate.TrialOracle, float64) differs between a network and its twin registered in run order
    (same parameters, same buffers, same candidate): the prior singles out another layer."""
    over = {"regularization.deep_inversion.scale": 1e-2} if key == "deep_inversion" else {"regularization.features.scale": 0.1}
    cfg = get_attack_config("invertinggradients", over)
    values = []
    for in_order in (False, True):
        model, shape, labels, grads = registration_case(cls, in_order)
        m64 = copy.deepcopy(model).double()
        orc = restate.TrialOracle(m64, torch.nn.CrossEntropyLoss(), cfg, [g.double() for g in grads], labels, None, None,
                                  dtype=torch.float64)
        _, terms = orc.objective_terms(_x(shape, seed=4))
        orc.close()
        values.append(terms[key])
    assert values[0] != pytest.approx(values[1], rel=1e-3), values
