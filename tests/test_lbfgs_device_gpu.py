"""L-BFGS on the device (csrc/lbfgs.cu, the conditional-graph trial of engine.cu): the direction kernels against a float64
two-loop recursion, the curvature push, whole trials against the host loop of attacks/lbfgs.py on the same engine, the early
exits, and which configurations take which path."""
import copy
import ctypes
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from breaching_b200 import engine as E  # noqa: E402
from breaching_b200 import get_attack_config, synthetic  # noqa: E402
from breaching_b200.attacks import lbfgs, prepare_attack  # noqa: E402
from breaching_b200.attacks.optimization_attack import _EngineSum  # noqa: E402
from breaching_b200.schedule import lr_table  # noqa: E402
from helpers import case_from_fixture, cfg_from_fixture, load_golden  # noqa: E402

DEV = torch.device("cuda:0")
H = lbfgs.HISTORY
R = H + 1


class Ring:
    """Caller-owned buffers of bre_lbfgs_direction for a vector of n values; pairs y = a * s from the SPD matrix diag(a)."""

    def __init__(self, n, seed):
        self.n = n
        self.gen = torch.Generator(device=DEV).manual_seed(seed)
        self.a = 0.5 + 1.5 * torch.rand(n, device=DEV, generator=self.gen)   # eigenvalues in [0.5, 2]
        self.S = torch.zeros(R * n, device=DEV)
        self.Y = torch.zeros(R * n, device=DEV)
        self.gram = torch.zeros(2 * R * R + 3 * R, dtype=torch.float64, device=DEV)
        st = E.LbfgsScalars()
        st.h_diag, st.t, st.total_iters = 1.0, 1.0, 1     # total_iters > 0: every call offers its candidate pair (t = 1: s = d)
        self.state = E.lbfgs_state(st)
        self.prev_g = torch.zeros(n, device=DEV)
        self.d = torch.zeros(n, device=DEV)

    def call(self, g, prev_g, d):
        self.prev_g.copy_(prev_g)
        self.d.copy_(d)
        return E.lbfgs_direction(self.S, self.Y, self.gram, self.state, g, self.prev_g, self.d)

    def push(self, k=1):
        for _ in range(k):
            s = torch.randn(self.n, device=DEV, generator=self.gen)
            sc = self.call(self.a * s, torch.zeros_like(s), s)       # y = a s - 0, s = 1 * s: y.s > 0
            assert sc.pushed == 1
        return sc

    def live(self, sc):
        return [(sc.first + k) % R for k in range(sc.count)]


def _two_loop64(S, Y, slots, g):
    """torch.optim.LBFGS's direction in float64 on the stored (fp32) pairs, oldest first; also the magnitude sum of its terms."""
    S, Y, g = S.double(), Y.double(), g.double()
    if not slots:
        return -g, g.abs()
    s_new, y_new = S[slots[-1]], Y[slots[-1]]
    h = float(s_new.dot(y_new) / y_new.dot(y_new))
    rho = {i: 1.0 / float(S[i].dot(Y[i])) for i in slots}
    q = -g
    al = {}
    for i in reversed(slots):
        al[i] = float(S[i].dot(q)) * rho[i]
        q = q - al[i] * Y[i]
    r = q * h
    mag = h * g.abs()
    for i in slots:
        be = float(Y[i].dot(r)) * rho[i]
        r = r + (al[i] - be) * S[i]
        mag = mag + abs(al[i] - be) * S[i].abs() + abs(h * al[i]) * Y[i].abs()
    return r, mag


@pytest.mark.parametrize("n", [10, 3072 + 10, 150528, 1204224])
@pytest.mark.parametrize("pairs", [0, 1, 37, 100, "wrapped"])
def test_direction_matches_float64_two_loop(n, pairs):
    ring = Ring(n, seed=n % 9973 + 7)
    sc = None
    if pairs == "wrapped":
        sc = ring.push(H + 17)
        assert sc.first == 17 and sc.count == H   # 117 pushes through a ring of 101 slots: the oldest live slot moved on
    elif pairs > 0:
        sc = ring.push(pairs)
    if pairs == 0:   # a fresh optimiser: no candidate pair, d = -g
        st = E.LbfgsScalars()
        st.h_diag = 1.0
        ring.state = E.lbfgs_state(st)
    g = torch.randn(n, device=DEV, generator=ring.gen)
    zeros = torch.zeros(n, device=DEV)
    saved = (ring.state.clone(), ring.S.clone(), ring.Y.clone(), ring.gram.clone())
    sc = ring.call(g, zeros, zeros)            # s = 0: the candidate fails the curvature test, the direction uses the ring as it is
    assert sc.pushed == 0
    d1 = ring.d.clone()
    slots = ring.live(sc)
    assert len(slots) == {0: 0, 1: 1, 37: 37, 100: 100, "wrapped": 100}[pairs]
    ref, mag = _two_loop64(ring.S.view(R, n), ring.Y.view(R, n), slots, g)
    # the device forms each d_i once in fp64 and rounds it to fp32 (half an ulp: 2^-24 relative); its Gram entries and S^T g, Y^T g
    # are fp64 sums of exact products of the fp32 operands (relative error <= n 2^-53 of the magnitude of each sum), carried through
    # m <= 100 steps of a recurrence whose multipliers are bounded by the spectrum [0.5, 2] of the pair matrix: 64 (n + 2m) 2^-53
    # times the magnitude of the terms of d_i bounds what fp64 contributes
    tol = 2.0 ** -24 * ref.abs() + 64 * (n + 2 * len(slots)) * 2.0 ** -53 * mag
    err = (d1.double() - ref).abs()
    assert bool((err <= tol).all()), (float(err.max()), float((err / tol.clamp_min(1e-300)).max()))
    assert math.isclose(sc.gtd, float(g.double().dot(d1.double())), rel_tol=1e-9, abs_tol=1e-12)
    # a second launch on the same inputs gives the same bits
    ring.state.copy_(saved[0]); ring.S.copy_(saved[1]); ring.Y.copy_(saved[2]); ring.gram.copy_(saved[3])
    ring.call(g, zeros, zeros)
    assert torch.equal(ring.d, d1)


def test_rejected_pair_leaves_full_ring_unchanged():
    n = 3072 + 10
    ring = Ring(n, seed=5)
    sc = ring.push(H + 5)
    assert sc.count == H
    live = ring.live(sc)
    S, Y = ring.S.view(R, n)[live].clone(), ring.Y.view(R, n)[live].clone()
    gram = ring.gram.clone()
    idx = torch.tensor(live, device=DEV)
    SY, YY = gram[: R * R].view(R, R), gram[R * R: 2 * R * R].view(R, R)
    rho = gram[2 * R * R: 2 * R * R + R]
    s = torch.randn(n, device=DEV, generator=ring.gen)
    after = ring.call(-ring.a * s, torch.zeros(n, device=DEV), s)   # y = -a s: y.s < 0
    assert after.pushed == 0 and after.count == H and after.first == sc.first
    assert torch.equal(ring.S.view(R, n)[live], S) and torch.equal(ring.Y.view(R, n)[live], Y)
    g2 = ring.gram
    SY2, YY2 = g2[: R * R].view(R, R), g2[R * R: 2 * R * R].view(R, R)
    assert torch.equal(SY2[idx][:, idx], SY[idx][:, idx]) and torch.equal(YY2[idx][:, idx], YY[idx][:, idx])
    assert torch.equal(g2[2 * R * R: 2 * R * R + R][idx], rho[idx])
    assert after.h_diag == sc.h_diag


def _attacker_engine(name, overrides=None):
    fx = load_golden(f"trial_{name}.pt")
    model, loss_fn, payload, shared, true = case_from_fixture(fx)
    cfg = cfg_from_fixture(fx)
    for k, v in (overrides or {}).items():
        node = cfg
        *path, last = k.split(".")
        for p in path:
            node = node[p]
        node[last] = v
    attacker = prepare_attack(model, loss_fn, cfg, dict(device=DEV, dtype=torch.float, backend="simt"))
    rec_models, labels, stats, shared2 = attacker.prepare_attack(payload, copy.deepcopy(shared))
    joint = type(attacker).__name__ == "OptimizationJointAttacker"
    engine = attacker._get_engine(rec_models, shared2, torch.zeros(labels.shape[0], dtype=torch.long) if joint else labels)
    return fx, cfg, attacker, engine, joint


def _host_trial(attacker, engine, cfg, joint, x0, l0, table, iters):
    """attacks/lbfgs.run_trial's loop (joint: _run_joint_trial's), recording the optimiser's counters after every step."""
    opt = cfg.optim
    dm, ds = attacker.dm.to(DEV), attacker.ds.to(DEV)
    lo, hi = -dm / ds, (1 - dm) / ds
    if joint:
        flat = torch.cat([x0.reshape(-1), l0.reshape(-1)]).clone()
        x, ell = flat[: x0.numel()].view_as(x0), flat[x0.numel():].view_as(l0)
    else:
        flat = x0.detach().clone().reshape(-1)
        x = flat.view_as(x0)
    optimizer = lbfgs.DeviceLBFGS(flat)
    hist, counts = [], []
    for it in range(iters):
        lr = float(table[it])
        if joint:
            def closure():
                val, gx, gl, _ = attacker._closure(engine, x, ell, it, lr)
                return val, torch.cat([gx.reshape(-1), gl.reshape(-1)])
        else:
            def closure():
                val, grad = engine.objective_and_gradient(x)
                return float(val), lbfgs.postprocess_gradient(grad, opt, it, lr).reshape(-1)
        value = optimizer.step(closure, lr)
        if opt.boxed:
            torch.max(torch.min(x, hi, out=x), lo, out=x)
        hist.append(value)
        counts.append((optimizer.total_iters, optimizer.func_evals))
    return hist, counts


@pytest.mark.parametrize("name", ["lbfgs_convnet", "lbfgs_wei_convnet", "lbfgs_cosine_convnet", "joint_dlg_convnet"])
def test_device_trial_matches_host_lbfgs(name):
    """Same engine, same start: the device trial takes as many inner iterations and closures per recorded iteration as the host
    loop until the objective is below 1e-3 of its start (from there the stop tests compare quantities at float32 noise level),
    its history stays within the fixture tolerances of test_engine_gpu until then and below 1e-3 of the start after it, over 8
    recorded iterations (up to 160 inner iterations: more than the ring holds)."""
    fx, cfg, attacker, engine, joint = _attacker_engine(name)
    iters = 8
    opt = cfg.optim
    table = lr_table(opt.step_size, opt.step_size_decay, opt.warmup, int(opt.max_iterations))
    x0 = fx["x0"].to(DEV)
    l0 = fx["l0"].to(DEV) if joint else None
    host_hist, host_counts = _host_trial(attacker, engine, cfg, joint, x0, l0, table, iters)
    engine.begin_lbfgs_trial(x0, table, label_logits=l0)
    dev_counts = []
    for _ in range(iters):
        engine.run(1)
        c = engine.lbfgs_counters()
        dev_counts.append((c["inner_iterations"], c["closures"]))
    dev_hist = engine.history().tolist()
    assert len(dev_hist) == iters
    start = abs(host_hist[0])
    converged = iters
    for k in range(iters):
        if abs(host_hist[k]) < 1e-3 * start:
            converged = k
            break
        assert dev_counts[k] == host_counts[k], (k, dev_counts, host_counts)
    for k, (a, b) in enumerate(zip(dev_hist, host_hist)):
        if k < converged:
            assert math.isclose(a, b, rel_tol=5e-2, abs_tol=1e-4 * start), (dev_hist, host_hist)
        else:   # below 1e-3 of the start both trajectories move at float32 noise level: both stay there
            assert abs(a) < 1e-3 * start and abs(b) < 1e-3 * start, (dev_hist, host_hist)


def test_zero_gradient_takes_one_closure_per_step():
    model, loss_fn, payload, shared, true = synthetic.make_case("convnet-tiny", "cifar", batch=1, seed=3, bn_random=True)
    cfg = get_attack_config("beyondinfering", {"objective.scale": 0.0, "optim.boxed": False})
    for key in list((cfg.get("regularization") or {}).keys()):
        cfg.regularization[key].scale = 0.0
    cfg.objective.task_regularization = 0.0
    meta = payload[0]["metadata"]
    eng = E.Engine(copy.deepcopy(model).to(DEV).eval(), (1, 3, 32, 32), cfg, DEV, backend="simt")
    eng.load_model()
    eng.load_targets([g.to(DEV) for g in shared[0]["gradients"]], true["labels"].to(DEV), mean=meta.mean, std=meta.std)
    x0 = torch.randn(1, 3, 32, 32, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    eng.begin_lbfgs_trial(x0, [0.1] * 8)
    eng.run(3)
    c = eng.lbfgs_counters()
    assert c["closures"] == 3 and c["inner_iterations"] == 0
    assert torch.equal(eng.candidate(), x0)
    assert eng.history().tolist() == [0.0, 0.0, 0.0]
    eng.close()


def test_non_finite_objective_stops_the_lbfgs_trial():
    model, loss_fn, payload, shared, true = synthetic.make_case("convnet-tiny", "cifar", batch=1, seed=3, bn_random=True)
    cfg = get_attack_config("beyondinfering", {"optim.boxed": False})
    meta = payload[0]["metadata"]
    eng = E.Engine(copy.deepcopy(model).to(DEV).eval(), (1, 3, 32, 32), cfg, DEV, backend="simt")
    eng.load_model()
    eng.load_targets([g.to(DEV) for g in shared[0]["gradients"]], true["labels"].to(DEV), mean=meta.mean, std=meta.std)
    eng.begin_lbfgs_trial(torch.full((1, 3, 32, 32), float("nan"), device=DEV), [0.1] * 8)
    eng.run(4)
    st = eng.status()
    assert st["stopped"] and st["recorded"] == 0 and st["min_objective"] == float("inf")
    eng.close()


def test_device_trial_needs_no_host_closure(monkeypatch):
    """reconstruct() with the beyondinfering preset: no closure on the host, one status poll per `callback` iterations."""
    fx = load_golden("trial_lbfgs_convnet.pt")
    model, loss_fn, payload, shared, true = case_from_fixture(fx)

    def refuse(self, candidate):
        raise AssertionError("host closure called")

    polls = []
    status = E.Engine.status
    monkeypatch.setattr(E.Engine, "objective_and_gradient", refuse)
    monkeypatch.setattr(E.Engine, "status", lambda self: polls.append(1) or status(self))
    T, callback = 6, 2
    cfg = get_attack_config("beyondinfering", {"optim.max_iterations": T, "optim.callback": callback})
    attacker = prepare_attack(model, loss_fn, cfg, dict(device=DEV, dtype=torch.float))
    attacker._score_trial = lambda engine, candidate: 0.0   # the score is an evaluation outside the trial
    rec, stats = attacker.reconstruct(payload, copy.deepcopy(shared), {})
    assert len(stats["Trial_0_Val"]) == T and torch.isfinite(rec["data"]).all()
    assert len(polls) <= math.ceil(T / callback) + 2, len(polls)


def test_routing():
    """Multi-query attacks, augmented configs and Langevin noise keep the host loop; one plain engine takes the device loop."""
    fx = load_golden("trial_lbfgs_convnet.pt")
    model, loss_fn, payload, shared, true = case_from_fixture(fx)

    class Stub:
        def begin_lbfgs_trial(self, *a, **k):
            pass

    def attacker(overrides):
        return prepare_attack(model, loss_fn, get_attack_config("beyondinfering", overrides), dict(device=DEV, dtype=torch.float))

    assert attacker({})._lbfgs_on_device(Stub())
    assert not attacker({})._lbfgs_on_device(_EngineSum([Stub(), Stub()]))
    assert not attacker({"augmentations": {"flip": {}}})._lbfgs_on_device(Stub())
    assert not attacker({"optim.langevin_noise": 0.01})._lbfgs_on_device(Stub())
    # and functionally: with Langevin noise the trial runs the host loop even though the engine offers the device one
    fx, cfg, att, engine, joint = _attacker_engine("lbfgs_convnet", {"optim.langevin_noise": 0.01, "optim.max_iterations": 2})

    def refuse(*a, **k):
        raise AssertionError("device loop taken")

    engine.begin_lbfgs_trial = refuse
    from collections import defaultdict

    stats = defaultdict(list)
    att._run_trial(engine, fx["x0"].to(DEV), stats, 0)
    assert len(stats["Trial_0_Val"]) == 2
