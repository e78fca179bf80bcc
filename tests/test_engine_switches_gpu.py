"""Engine switches that are meant to leave the numerics alone must leave them bitwise alone: two engines that differ only in one
switch evaluate the same candidate, and the objective, its terms, the gradient, every parameter gradient G, the direction v
(as the GEMMs read it) and all four buffers of every tensor must be identical."""
import copy
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from breaching_b200 import compiler as C  # noqa: E402
from breaching_b200 import get_attack_config, synthetic  # noqa: E402
from breaching_b200.engine import Engine  # noqa: E402
from breaching_b200.schedule import lr_table  # noqa: E402
from helpers import unwritten_tangents  # noqa: E402
from test_sweep_local_gpu import build_case, candidate, make_engine  # noqa: E402

DEV = torch.device("cuda:0")


def fedavg_case():
    model, _, _, shared, _ = synthetic.make_fedavg_case("resnet18", num_data_points=6, steps=3, data_per_step=2, image_size=32,
                                                        bn_random=True)
    return model.eval(), shared


def make(case, backend, options=()):
    if case == "fedavg":
        model, shared = fedavg_case()
        local = shared[0]["metadata"]["local_hyperparams"]
        eng = Engine(copy.deepcopy(model).to(DEV), (2, 3, 32, 32), get_attack_config("invertinggradients"), DEV, backend=backend)
        for k, v in options:
            eng.set_option(k, v)
        eng.load_model()
        eng.load_targets([g.to(DEV) for g in shared[0]["gradients"]], local["labels"][0])
        eng.set_local_steps(6, local["steps"], local["lr"], local["labels"])
        return eng, (6, 3, 32, 32)
    model, shape, labels, grads, cfg, feats = build_case(case)
    return make_engine(model, shape, cfg, labels, grads, backend, feats, options), shape


def snapshot(eng, shape, skip_tangent=()):
    val, grad = eng.objective_and_gradient(candidate(shape).to(DEV))
    skip_tangent = set(skip_tangent) | unwritten_tangents(eng)   # not stored by design (bre_engine_debug_tensor)
    out = {"objective": torch.tensor(val, dtype=torch.float64), "gradient": grad.cpu()}
    out.update({f"terms.{k}": torch.tensor(v, dtype=torch.float64) for k, v in eng.last_terms().items()})
    buffers(eng, out, skip_tangent)
    return out, skip_tangent, [i for i in range(len(eng.prog.ops)) if eng.debug_op(i)["fused"]]


def buffers(eng, out, skip_tangent=(), skip_candidate_val=False):
    for j in range(len(eng.prog.params)):
        out[f"G[{j}]"] = eng.debug_param("G", j)
        out[f"v[{j}]"] = eng.debug_param("v_operand", j)
    for t in range(len(eng.prog.tensors)):
        for which in ("val", "delta", "tangent", "tangent_delta"):
            if (t == 0 and which == "tangent") or (which == "tangent" and t in skip_tangent) or (t == 0 and which == "val" and skip_candidate_val):
                continue
            out[f"{which}[t{t}]"] = eng.debug_tensor(which, t)
    return out


def assert_bitwise(a, b, label):
    assert a.keys() == b.keys()
    diff = [k for k in a if not torch.equal(a[k], b[k])]
    worst = {k: float((a[k].double() - b[k].double()).abs().max()) for k in diff[:8]}
    assert not diff, f"{label}: {len(diff)} of {len(a)} buffers differ, e.g. {worst}"


def compare(case, backend, name, values, env=False, monkeypatch=None):
    runs = []
    for value in values:   # one engine at a time: `pdl` is process-wide
        if env:
            monkeypatch.setenv(name, str(value))
            eng, shape = make(case, backend)
        else:
            eng, shape = make(case, backend, ((name, value),))
        runs.append(snapshot(eng, shape))
        eng.close()
    skip = runs[0][1] | runs[1][1]
    if name == "fuse_bnact":
        # the fused run really fused (train-mode BN never does), and the only tangents it left unstored are fused pre-BN tangents
        assert not runs[0][2] and (bool(runs[1][2]) != case.startswith("trainbn-")), (runs[0][2], runs[1][2])
        assert skip == runs[1][1]
    else:
        assert not skip
    a, b = ({k: v for k, v in r[0].items() if not any(k == f"tangent[t{t}]" for t in skip)} for r in runs)
    assert_bitwise(a, b, f"{case} / {backend}: {name} {values} (unstored tangents skipped: {sorted(skip)})")


@pytest.mark.parametrize("case", ["resnet18", "trainbn-resnet18", "fedavg"])
def test_fuse_bnact_is_bitwise_neutral(case):
    """The FedAvg case is the regression test of the pre-BN tangent: its tangent-backward reduces the tangent of the gamma
    gradient from that tangent in steps k > 0, so the fused epilogue has to store it there."""
    compare(case, "tc", "fuse_bnact", (0, 1))


@pytest.mark.parametrize("backend", ["simt", "tc"])
@pytest.mark.parametrize("case", ["resnet18", "trainbn-resnet18"])
def test_overlap_wgrad_is_bitwise_neutral(case, backend):
    compare(case, backend, "overlap_wgrad", (0, 1))


@pytest.mark.parametrize("case", ["resnet18", "trainbn-resnet18"])
def test_pdl_is_bitwise_neutral(case):
    try:
        compare(case, "tc", "pdl", (0, 1))
    finally:   # process-wide switch: back to the default
        eng, _ = make("convnet-tiny", "simt")
        eng.set_option("pdl", int(os.environ.get("BRE_PDL", "1") != "0"))
        eng.close()


@pytest.mark.parametrize("case", ["resnet18", "trainbn-resnet18"])
def test_deferred_bn_finalisation(case, monkeypatch):
    """Not bitwise by design: the deferred eval-mode BN gamma / beta gradients are reduced over a finer slab grid and folded in
    16 interleaved slices (bn_grad_finalize_kernel), the in-kernel path over the plain slab grid in slab order.  So the sweeps F
    and B (activations, deltas, all other parameter gradients) must be bitwise equal, the BN parameter gradients must agree
    within the summation bound (P + 4) 2^-23 sum |terms| of their reduction, and everything downstream of the direction v
    (which depends on every G) is left to the sweep check of each setting."""
    outs = []
    for value in (0, 1):
        monkeypatch.setenv("BRE_DEFER_BN", str(value))
        eng, shape = make(case, "tc")
        eng.objective_and_gradient(candidate(shape).to(DEV))
        out = {f"G[{j}]": eng.debug_param("G", j) for j in range(len(eng.prog.params))}
        for t in range(len(eng.prog.tensors)):
            out[f"val[t{t}]"], out[f"delta[t{t}]"] = eng.debug_tensor("val", t), eng.debug_tensor("delta", t)
        bounds = {}
        mods = C.bn_modules(build_case(case)[0], eng.prog)
        for op, mod in zip(eng.prog.ops, mods):
            if op.kind == C.OP_BNACT and op.has_bn and not op.bn_train:
                y, d, x = (out[f"{w}[t{t}]"].double() for w, t in (("val", op.tout), ("delta", op.tout), ("val", op.tin)))
                du = (d * (y > 0) if op.relu else d).abs()
                inv = (1.0 / torch.sqrt(mod.running_var.double() + op.eps)).view(1, -1, 1, 1)
                xhat = (x.abs() + mod.running_mean.double().abs().view(1, -1, 1, 1)) * inv
                P_ = du.shape[0] * du.shape[2] * du.shape[3]
                bounds[f"G[{op.gamma}]"] = (P_ + 4) * 2.0 ** -23 * (du * xhat).sum(dim=(0, 2, 3))
                bounds[f"G[{op.beta}]"] = (P_ + 4) * 2.0 ** -23 * du.sum(dim=(0, 2, 3))
        outs.append(out)
        eng.close()
    a, b = outs
    exact = {k: v for k, v in a.items() if k not in bounds}
    assert_bitwise(exact, {k: b[k] for k in exact}, f"{case}: BRE_DEFER_BN, sweeps F / B")
    for k, bound in bounds.items():
        err = (a[k].double() - b[k].double()).abs()
        assert (err <= bound).all(), (k, float(err.max()), float(bound.max()))


@pytest.mark.parametrize("case", ["resnet18", "trainbn-resnet18"])
def test_weight_prefetch_is_bitwise_neutral(case, monkeypatch):
    compare(case, "tc", "BRE_TC_WPREFETCH", (0, 1), env=True, monkeypatch=monkeypatch)


@pytest.mark.parametrize("case", ["resnet18", "trainbn-resnet18", "fedavg"])
def test_graph_replay_is_bitwise_neutral(case):
    """Two optimiser iterations with and without CUDA-graph replay: history, candidate and every buffer of the last evaluation
    (except the candidate's value, which the step has moved on since)."""
    outs = []
    for use_graph in (0, 1):
        eng, shape = make(case, "tc", (("use_graph", use_graph),))
        eng.begin_trial(candidate(shape).to(DEV), lr_table(0.1, "step-lr", 0, 24000, 8))
        eng.run(2)
        eng.sync()
        out = {"history": eng.history().clone(), "candidate": eng.candidate().cpu()}
        outs.append(buffers(eng, out, skip_candidate_val=True))
        eng.close()
    assert_bitwise(outs[0], outs[1], f"{case}: use_graph")
