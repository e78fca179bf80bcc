"""FedAvg (multi-step) updates of train-mode BatchNorm networks on the CPU: no BN buffers from server or user, so every local step
normalises with its own batch statistics.  The reference's own outputs (tests/golden/trial_fedavg_trainbn_*.pt) against the
oracle restatement; the float64 restatement of the engine's evaluation (``fedavg_trainbn_oracle.TrainBnMultiStepInterpreter``)
against float64 autograd of the reference's unrolled local steps -- candidate gradient, the adjoint u_k every step uses and the
tangent parameter gradients H_k u_{k+1}, gamma / beta of every train-mode BN included; and the multi-step checker on its buffers,
including a corrupted gamma tangent reported at exactly the (step, op, sweep) that produced it."""
import copy
import math

import pytest
import torch
import torch.nn.functional as F

from breaching_b200 import compiler, get_attack_config, synthetic
from fedavg_trainbn_oracle import TrainBnMultiStepChecker, TrainBnMultiStepInterpreter
from helpers import load_golden, oracle_for_fixture, sweep_objective
from oracle import restate
from oracle.fedavg_priors import PriorStepSource
from oracle.program_interp import image_prior
from oracle.sweep_check import InterpreterGlue

FIXTURES = ["fedavg_trainbn_convnet", "fedavg_trainbn_taskreg_convnet", "fedavg_trainbn_resnet18"]
PLAIN = {"regularization.features.scale": 0.0}
TASK = {"regularization.features.scale": 0.0, "objective.task_regularization": 0.1}
CONVNET = dict(model_name="convnet-tiny", data="cifar", num_data_points=4, steps=3, data_per_step=2, lr=0.05, seed=4, bn_random=True,
               no_buffers=True)
RESNET = dict(model_name="resnet18", data="imagenet", num_data_points=4, steps=4, data_per_step=1, lr=1e-2, seed=6, bn_random=True,
              image_size=64, classes=10, no_buffers=True)
CASES = {
    # 3 steps x 2 images over 4 images: step 2 wraps onto images 0-1
    "convnet-tiny": (CONVNET, PLAIN),
    "convnet-tiny-task": (CONVNET, TASK),
    # one image per step: the last stage normalises over 2 x 2 pixels
    "resnet18": (RESNET, PLAIN),
    "resnet18-task": (RESNET, TASK),
}


def train_mode(model):
    """The model as the attacker evaluates it without any BN buffers (base_attack.py:192-197)."""
    model = copy.deepcopy(model).train()
    for m in model.modules():
        if hasattr(m, "track_running_stats"):
            m.track_running_stats = False
    return model


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_reproduces_reference_fixture(name):
    """The tolerances of tests/test_golden_oracle.py: trajectories to 2e-4, the first candidate to 1e-4."""
    fx = load_golden(f"trial_{name}.pt")
    orc, cfg, labels = oracle_for_fixture(fx)
    assert orc.model.training and fx["case"]["no_buffers"]
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
    assert payload[0]["buffers"] is None and shared[0]["buffers"] is None
    cfg = get_attack_config("modern", dict(over))
    local = shared[0]["metadata"]["local_hyperparams"]
    x = torch.randn(true["data"].shape, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    return train_mode(model), loss_fn, payload, shared, cfg, local, x


def run_multistep(name, tamper=None):
    model, loss_fn, payload, shared, cfg, local, x = _case(name)
    m64 = model.double()
    prog = compiler.compile_model(m64, (local["data_per_step"], *x.shape[1:]))
    assert any(op.bn_train for op in prog.ops)
    mi = TrainBnMultiStepInterpreter(m64, prog, local["lr"])
    mi.tamper = tamper
    g64 = [g.double() for g in shared[0]["gradients"]]
    obj = sweep_objective(cfg)
    val, grad = mi.run(x, local["labels"], g64, obj)
    bn = [None] * len(prog.ops)   # no running statistics anywhere
    chk = TrainBnMultiStepChecker(prog, bn, g64, local["labels"], obj,
                                  [PriorStepSource(mi, k) for k in range(local["steps"])], InterpreterGlue(mi, x, grad))
    return mi, chk, val, grad, (model, loss_fn, payload, shared, cfg, local, x)


def unrolled_autograd(model, x, local, g, cfg, W_path, D_last):
    """Float64 autograd of the reference's multi-step objective (objectives.py:48-72, train mode): the K local SGD steps kept in
    the graph, the match of W_K - W_0 plus the task term of the last step.  Returns (value, d value / d x, [d value / d W_{k+1}],
    {k: H_k u_{k+1}} for k = 1 .. K - 1, the last one with its task-loss term -tau/lr G_last, drift), ``drift`` the largest
    relative distance between a pinned W_{k+1} and autograd's own W_k - lr G_k at the same W_k.

    The values of the trajectory W_1 .. W_K and of D_K are ``W_path`` / ``D_last`` (the restatement's), the derivatives autograd's:
    with one image per step the step map W_k -> W_{k+1} of a train-mode ResNet-18 amplifies float64 rounding of W_k about a
    thousandfold, so two independent float64 trajectories drift apart by 1e-8 after four steps while every derivative taken at the
    same point agrees to rounding."""
    pin = lambda value, expr: value + (expr - expr.detach())  # noqa: E731
    names = [n for n, _ in model.named_parameters()]
    buffers = dict(model.named_buffers())
    x = x.detach().clone().requires_grad_(True)
    lr, K, dps = local["lr"], local["steps"], local["data_per_step"]
    W, G, seen, drift = [[p.detach().clone().requires_grad_(True) for p in model.parameters()]], [], 0, 0.0
    for k in range(K):
        out = torch.func.functional_call(model, (dict(zip(names, W[k])), buffers), (x[seen:seen + dps],))
        seen = (seen + dps) % x.shape[0]
        loss = F.cross_entropy(out, local["labels"][k])
        G.append(torch.autograd.grad(loss, W[k], create_graph=True))
        step = [(w - lr * gk).detach() for w, gk in zip(W[k], G[k])]
        drift = max(drift, _rel(torch.cat([t.flatten() for t in W_path[k + 1]]), torch.cat([t.flatten() for t in step])))
        W.append([pin(wp, w - lr * gk) for wp, w, gk in zip(W_path[k + 1], W[k], G[k])])
    o = cfg["objective"]
    kw = {k_: o[k_] for k_ in ("tag_scale", "scale_scheme") if k_ in o}
    D = [pin(dp, wk - w0) for dp, wk, w0 in zip(D_last, W[K], W[0])]
    val = restate.matching_objective(o["type"], D, g, scale=restate.cfg_get(o, "scale", 1.0), **kw)
    tau = float(restate.cfg_get(o, "task_regularization", 0.0) or 0.0)
    if tau != 0:
        val = val + tau * loss
    n = len(names)
    flat = torch.autograd.grad(val, [x] + [w for k in range(1, K + 1) for w in W[k]], create_graph=True)
    gx, u = flat[0], [list(flat[1 + (k - 1) * n:1 + k * n]) for k in range(1, K + 1)]
    TG = {}
    for k in range(1, K):
        s = sum((gk * uk.detach()).sum() for gk, uk in zip(G[k], u[k]))
        TG[k] = list(torch.autograd.grad(s, W[k], retain_graph=True))
        if k == K - 1 and tau != 0:
            TG[k] = [t - tau / lr * gk for t, gk in zip(TG[k], G[k])]
    return (val.detach(), gx.detach(), [[t.detach() for t in uk] for uk in u], {k: [t.detach() for t in v] for k, v in TG.items()},
            drift)


def _rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


@pytest.mark.parametrize("name", list(CASES))
def test_interpreter_matches_unrolled_autograd(name):
    mi, _, val, grad, (model, loss_fn, payload, shared, cfg, local, x) = run_multistep(name)
    g64 = [g.double() for g in shared[0]["gradients"]]
    ref_val, ref_gx, ref_u, ref_TG, drift = unrolled_autograd(model.double(), x, local, g64, cfg, mi.W, mi.D[-1])
    pv, gp = image_prior(x, sweep_objective(cfg))
    # one image per step: the batch statistics of ResNet-18's last stage span 2 x 2 pixels, and its Hessian-vector products
    # amplify float64 rounding about a thousandfold
    tol = 1e-12 if name.startswith("convnet") else 1e-11
    assert drift < 1e-14, drift   # the pin absorbs one step's rounding only: the restatement's trajectory is autograd's
    assert abs(float(val - pv) - float(ref_val)) <= 1e-12 * max(1.0, abs(float(ref_val)))
    assert _rel(grad - gp, ref_gx) < tol
    # whole parameter vectors: the biases of convolutions that feed a train-mode BN have a zero gradient, their entries are
    # rounding noise of both computations
    cat = lambda ts, idx=None: torch.cat([t.flatten() for j, t in enumerate(ts) if idx is None or j in idx])  # noqa: E731
    K = local["steps"]
    for k in range(K):   # step k used u_{k+1} = d objective / d W_{k+1}
        assert _rel(cat(mi.steps[k].U), cat(ref_u[k])) < tol, k
    prog = mi.prog
    gb = {j for op in prog.ops if op.kind == compiler.OP_BNACT and op.has_bn and op.bn_train for j in (op.gamma, op.beta)}
    assert gb
    for k in range(1, K):
        assert _rel(cat(mi.steps[k].TG), cat(ref_TG[k])) < tol, k
        assert _rel(cat(mi.steps[k].TG, gb), cat(ref_TG[k], gb)) < tol, k   # BN gamma / beta tangents
    if not name.startswith("convnet"):   # the restatement's own trajectory: see unrolled_autograd
        return
    # against the restatement of the reference closure (oracle.restate, what the fixtures are checked with), priors included
    meta = payload[0]["metadata"]
    dm = torch.tensor(meta.mean, dtype=torch.float64)[None, :, None, None]
    ds = torch.tensor(meta.std, dtype=torch.float64)[None, :, None, None]
    orc = restate.TrialOracle(copy.deepcopy(model).double(), loss_fn, cfg, g64, torch.cat(local["labels"]), dm, ds,
                              dtype=torch.float64, local_hyperparams=local)
    phi, _, raw, terms = orc.closure_gradient(x, 0, 0.0)
    orc.close()
    assert abs(float(val) - float(phi)) <= 1e-10 * max(1.0, abs(float(phi))), (float(val), float(phi))
    assert _rel(grad, raw) < 1e-10


@pytest.mark.parametrize("name", list(CASES))
def test_checker_holds_on_interpreter_buffers(name):
    _, chk, _, _, _ = run_multistep(name)
    chk.check()
    worst = max(chk.ratios.values())
    assert worst < 1e-6, sorted(chk.ratios.items(), key=lambda kv: -kv[1])[:5]
    assert any(sweep == "TG" for _, sweep in chk.ratios), chk.ratios


def test_corrupted_gamma_tangent_is_reported():
    """The gamma tangent of the last train-mode BN at step 1 off by 5 %: exactly that (step, op, sweep)."""
    _, chk0, _, _, _ = run_multistep("convnet-tiny")
    target = max(i for i, op in enumerate(chk0.prog.ops) if op.kind == compiler.OP_BNACT and op.bn_train)
    gamma = chk0.prog.ops[target].gamma

    def tamper(step, sweep, oi, key, stored, contribution=None):
        if step == 1 and sweep == "TG" and oi == target and key == gamma:
            return stored * 1.05
        return stored

    _, chk, _, _, _ = run_multistep("convnet-tiny", tamper)
    found = {(f.step, f.op, f.sweep) for f in chk.check(raise_on_failure=False)}
    assert found == {(1, target, "TG")}, found


def test_one_value_per_channel_is_refused_by_torch_too():
    """What the engine refuses (a train-mode BN over one value per channel: ResNet-18 at 32 x 32 with one image per step) is a
    training step torch refuses as well."""
    model, loss_fn, payload, shared, true = synthetic.make_fedavg_case("resnet18", "imagenet", num_data_points=2, steps=2,
                                                                       data_per_step=2, lr=1e-2, seed=6, image_size=32, classes=10,
                                                                       no_buffers=True)
    with pytest.raises(ValueError, match="more than 1 value per channel"):
        train_mode(model)(true["data"][:1])
