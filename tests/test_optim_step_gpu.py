"""The tail of the iteration on the GPU -- grad_norm_kernel, pixel_step_kernel, commit_kernel and the Langevin-noise generator --
against the float64 restatement of oracle/optim_step.py: stand-alone through ``bre_optimizer_step`` over the case matrix and planted
edges, through the engine with noise on (what the step really receives), and the per-trial noise fields."""
import copy
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import optim_step_cases as K  # noqa: E402
from breaching_b200 import get_attack_config, synthetic  # noqa: E402
from breaching_b200.attacks import prepare_attack  # noqa: E402
from breaching_b200.engine import EngineError, langevin_noise, optimizer_step  # noqa: E402
from breaching_b200.schedule import lr_table  # noqa: E402
from helpers import case_from_fixture, cfg_from_fixture, load_golden  # noqa: E402
from oracle import optim_step as OS  # noqa: E402

DEV = torch.device("cuda:0")
GUARD = 64


# ---- the generator -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed, trial, it", [(0, 0, 0), (K.SEED, 0, 7), (K.SEED, 3, 7), (2 ** 64 - 1, 2 ** 31 - 1, 23_999)])
@pytest.mark.parametrize("n, first", [(1, 0), (257, 0), ((1 << 20) + 3, 0), (4099, (1 << 32) - 2000)])
def test_langevin_noise_matches_the_restatement(seed, trial, it, n, first):
    a = langevin_noise(seed, trial, it, n, first=first, device=DEV)
    b = langevin_noise(seed, trial, it, n, first=first, device=DEV)
    assert torch.equal(a, b)
    ref = OS.gaussian(seed, trial, it, np.arange(n, dtype=np.uint64) + np.uint64(first))
    got = a.cpu().numpy().astype(np.float64)
    bound = OS.Z_ULPS * OS.U * np.abs(ref) + 1e-12
    ratio = float((np.abs(got - ref) / bound).max())
    print(f"noise n={n} first={first} (seed, trial, it)=({seed}, {trial}, {it}): max |error|/bound = {ratio:.3f}")
    assert ratio <= 1.0
    assert np.abs(got).max() <= OS.Z_MAX * (1 + 1e-6)


# ---- stand-alone step ------------------------------------------------------------------------------------------------------------
class DeviceStep:
    """State of one stand-alone sequence on the device; ``step`` runs bre_optimizer_step and returns (before, after) as the checker
    wants them.  The history buffer is followed by a guard region that no call may touch."""

    def __init__(self, ccfg, lr, lo, hi, C, HW, x0, max_hist=64, trial=0):
        self.ccfg, self.C, self.HW, self.max_hist = ccfg, C, HW, max_hist
        dev = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float32)).to(DEV).contiguous()  # noqa: E731
        self.lr, self.lo, self.hi = dev(lr), dev(lo), dev(hi)
        self.x = dev(x0)
        self.m, self.v, self.best = torch.zeros_like(self.x), torch.zeros_like(self.x), self.x.clone()
        self.hist = torch.full((max_hist + GUARD,), -7.0, device=DEV)
        self.sc = dict(fmin=math.inf, it=0, recorded=0, stopped=0, trial=trial)

    def snapshot(self):
        s = {k: getattr(self, k).cpu().numpy().copy() for k in ("x", "m", "v", "best")}
        s.update(self.sc)
        return s

    def step(self, g, gt, obj):
        before = self.snapshot()
        hist_before = self.hist.cpu().numpy().copy()
        scal = dict(self.sc)
        scal.update({k: obj.get(k, 0.0) for k in ("match", "task_loss", "tv", "norm", "di", "feat")})
        gd = torch.as_tensor(g).to(DEV)
        gtd = None if gt is None else torch.as_tensor(gt).to(DEV)
        out = optimizer_step(self.x, self.m, self.v, self.best, gd, self.ccfg, self.lr, self.hist[: self.max_hist], scal, grad_task=gtd,
                             lo=self.lo, hi=self.hi, C=self.C, HW=self.HW)
        self.sc = {k: out[k] for k in ("fmin", "it", "recorded", "stopped", "trial")}
        after = self.snapshot()
        hist_after = self.hist.cpu().numpy()
        changed = np.flatnonzero(hist_after != hist_before)
        slot = before["recorded"]
        assert all(i == slot and i < self.max_hist for i in changed), f"history written at {changed}, expected at most slot {slot}"
        after["hist"] = float(hist_after[slot]) if (after["recorded"] > slot and slot < self.max_hist) else None
        if after["recorded"] > slot and slot >= self.max_hist:
            after.pop("hist")         # full history: nothing to read, and nothing may have been written (checked above)
        after["last_objective"] = out["last_objective"]
        after["grad_norm_sq"] = out["grad_norm_sq"] if self.ccfg.grad_clip >= 0 else None
        return before, after


def run_device_sequence(seq, steps=None):
    dev = DeviceStep(seq.ccfg, seq.lr, seq.lo, seq.hi, seq.C, seq.HW, seq.x0)
    chk = OS.StepChecker(seq.cfg, seq.lr, seq.lo, seq.hi, seq.C, seq.HW)
    for k in range(steps or seq.steps):
        g, gt, obj = seq.inputs(k)
        before, after = dev.step(g, gt, obj)
        chk.check(before, g, gt, obj, after)
    return chk, dev


def test_matrix_size():
    cases = K.matrix()
    print(f"matrix: {len(cases)} cases x {len(K.SMALL_SIZES)} sizes x {K.STEPS} steps, plus the {K.BIG_SIZE} candidate")
    assert len(cases) == 27


@pytest.mark.parametrize("case", K.matrix(), ids=K.case_id)
def test_step_matrix(case):
    worst, either, amb = {}, 0, 0
    for size in K.SMALL_SIZES:
        chk, dev = run_device_sequence(K.Sequence(case, size))
        assert dev.sc["it"] == K.STEPS and dev.sc["recorded"] == K.STEPS
        for key, r in chk.ratios.items():
            worst[key] = max(worst.get(key, 0.0), r)
        either += chk.either_sign
        amb += chk.clip_ambiguous
    print(f"{K.case_id(case)}: max |error|/bound {({k: round(v, 3) for k, v in worst.items()})}, either-sign {either}, clip-ambiguous {amb}")
    assert either <= 4 and max(worst.values()) <= 1.0


BIG_CASES = [dict(optimizer="adam", signed=None, clip="active", noise=0.01, boxed=True, task="tau"),
             dict(optimizer="momgd", signed="hard", clip="active", noise=1.0, boxed=True, task="null")]


@pytest.mark.parametrize("case", BIG_CASES, ids=K.case_id)
def test_step_on_the_full_size_candidate(case):
    """8 x 3 x 224 x 224: more elements than one pass of the grid, and a norm folded over all its blocks (6 steps: the float64 side
    draws 1.2 M Philox values per step in numpy)."""
    chk, dev = run_device_sequence(K.Sequence(case, K.BIG_SIZE, steps=6), steps=6)
    print(f"{K.case_id(case)} {K.BIG_SIZE}: max |error|/bound {chk.ratios}, either-sign {chk.either_sign}")
    assert chk.either_sign <= 8 and max(chk.ratios.values()) <= 1.0


# ---- planted edges -------------------------------------------------------------------------------------------------------------------
def _edge(optimizer="adam", signed=None, clip=None, noise=0.0, boxed=False, tau=0.0, excludes=False, T=K.T_MAX, n_lr=K.N_LR, size=(2, 3, 5)):
    ccfg = K.make_ccfg(optimizer, signed, clip, noise, boxed, tau, excludes, T)
    images, C, HW = size
    n = images * C * HW
    rng = np.random.default_rng(n + 17)
    lr = np.asarray(lr_table(0.1, "cosine-decay", 0, T, n_lr), dtype=np.float32)
    lo, hi = (-1.0 - 0.1 * np.arange(C)).astype(np.float32), (0.8 + 0.07 * np.arange(C)).astype(np.float32)
    x0 = rng.uniform(-0.5, 0.5, n).astype(np.float32)
    dev = DeviceStep(ccfg, lr, lo, hi, C, HW, x0, max_hist=4)
    chk = OS.StepChecker(OS.StepCfg.from_ccfg(ccfg), lr, lo, hi, C, HW)
    g = (1e-2 * rng.standard_normal(n)).astype(np.float32)
    return dev, chk, g, rng


def _checked(dev, chk, g, gt, obj):
    before, after = dev.step(g, gt, obj)
    chk.check(before, g, gt, obj, after)
    return before, after


def test_hard_sign_of_zero_and_tiny_gradients():
    dev, chk, g, _ = _edge(optimizer="gd", signed="hard")
    g[:6] = [0.0, -0.0, 1e-45, -1e-45, 1e-38, -1e-38]
    before, after = _checked(dev, chk, g, None, dict(match=1.0))
    lr = float(dev.lr[0])
    assert np.array_equal(after["x"][:2], before["x"][:2])                      # sign(0) = 0: no move
    assert np.allclose(after["x"][2:6] - before["x"][2:6], [-lr, lr, -lr, lr], atol=1e-7)
    assert chk.either_sign == 0


@pytest.mark.parametrize("clip", [None, 10.0])
def test_nan_gradient_entry_stays_local(clip):
    dev, chk, g, _ = _edge(optimizer="adam", clip=clip)
    g[7] = np.nan
    before, after = _checked(dev, chk, g, None, dict(match=1.0))
    bad = np.isnan(after["x"])
    if clip is None:
        assert bad.sum() == 1 and bad[7] and np.isnan(after["m"][7]) and np.isnan(after["v"][7])
    else:   # the norm is NaN, `NaN > clip` is false: no clipping, as in torch, and still one pixel
        assert math.isnan(after["grad_norm_sq"]) and bad.sum() == 1 and bad[7]


@pytest.mark.parametrize("optimizer", ["adam", "bert-adam", "momgd"])
def test_schedule_ends(optimizer):
    """it = 0, it = n_lr - 1, it >= n_lr (lr = 0: x fixed -- AdamW's factor is 1 --, moments still move)."""
    dev, chk, g, rng = _edge(optimizer=optimizer, n_lr=3)
    for k in range(5):
        before, after = _checked(dev, chk, (g * (1 + k)).astype(np.float32), None, dict(match=1.0 / (1 + k)))
        if k >= 3:
            assert np.array_equal(after["x"], before["x"]) and not np.array_equal(after["m"], before["m"])
    assert dev.sc["it"] == 5


@pytest.mark.parametrize("optimizer, signed", [("adam", "soft"), ("bert-adam", None), ("momgd", "soft")])
def test_late_in_a_long_trial(optimizer, signed):
    """it = 23 990 .. 23 999 of 24 000: bias corrections ~ 1, soft-sign factor down to 4e-5 (its own rounding matters there)."""
    T = 24_000
    dev, chk, g, rng = _edge(optimizer=optimizer, signed=signed, noise=0.01, T=T, n_lr=T)
    dev.sc["it"] = T - 10
    dev.m = torch.as_tensor((1e-2 * rng.standard_normal(g.size)).astype(np.float32)).to(DEV)
    dev.v = torch.as_tensor((1e-4 * rng.random(g.size)).astype(np.float32)).to(DEV)
    dev.lr = torch.full((T,), 0.01, device=DEV)
    chk.lr_table = np.full(T, np.float32(0.01), dtype=np.float64)
    for k in range(10):
        _checked(dev, chk, (g * rng.standard_normal(g.size)).astype(np.float32) * 100, None, dict(match=1.0))
    print(f"late {optimizer} {signed}: max |error|/bound {chk.ratios}")
    assert dev.sc["it"] == T


def test_box_faces_and_channel_index():
    dev, chk, g, _ = _edge(optimizer="gd", boxed=True, size=(2, 3, 5))
    n = g.size
    ch = (np.arange(n) // 5) % 3
    x = np.where(np.arange(n) % 2 == 0, dev.hi.cpu().numpy()[ch], dev.lo.cpu().numpy()[ch]).astype(np.float32)
    dev.x = torch.as_tensor(x).to(DEV)
    dev.best = dev.x.clone()
    g = np.where(np.arange(n) % 2 == 0, -1.0, 1.0).astype(np.float32)     # pushes every element outward
    before, after = _checked(dev, chk, g, None, dict(match=1.0))
    assert np.array_equal(after["x"], x)
    # and inward moves are kept
    before, after = _checked(dev, chk, -g, None, dict(match=0.5))
    assert np.all(after["x"] != x)


def test_best_so_far_below_equal_above():
    dev, chk, g, _ = _edge(optimizer="adam")
    seen = []
    for phi in (1.0, 1.0, 2.0, 0.5, 0.5, float(np.float32(0.5)) + 1e-12):   # the last one equals 0.5 once rounded to fp32
        before, after = _checked(dev, chk, g, None, dict(match=phi))
        seen.append(np.array_equal(after["best"], after["x"]))
        assert np.array_equal(after["best"], after["x"] if seen[-1] else before["best"])
    assert seen == [True, False, False, True, False, False]
    assert dev.sc["fmin"] == 0.5


@pytest.mark.parametrize("bad", [math.nan, math.inf])
def test_non_finite_objective_applies_the_step_once_then_freezes(bad):
    dev, chk, g, _ = _edge(optimizer="adam", clip=1.0, noise=0.01)
    _checked(dev, chk, g, None, dict(match=1.0))
    before, after = _checked(dev, chk, g, None, dict(match=bad))
    assert after["stopped"] == 1 and after["recorded"] == 1 and after["it"] == 2 and not np.array_equal(after["x"], before["x"])
    frozen_before, frozen = _checked(dev, chk, g, None, dict(match=0.1))
    for key in ("x", "m", "v", "best"):
        assert np.array_equal(frozen[key], after[key])
    assert (frozen["it"], frozen["recorded"], frozen["stopped"], frozen["fmin"]) == (2, 1, 1, after["fmin"])


def test_objective_excluding_the_task_term():
    dev, chk, g, rng = _edge(optimizer="adam", tau=0.3, excludes=True)
    gt = (1e-2 * rng.standard_normal(g.size)).astype(np.float32)
    before, after = _checked(dev, chk, g, gt, dict(match=1.0, task_loss=5.0))
    assert after["last_objective"] == 1.0                                    # the task loss is not in phi ...
    dev2, chk2, g2, _ = _edge(optimizer="adam", tau=0.3, excludes=True)
    _, after2 = _checked(dev2, chk2, g, None, dict(match=1.0, task_loss=5.0))
    assert not np.array_equal(after["x"], after2["x"])                       # ... but its gradient is in the step


def test_full_history_is_not_overrun():
    dev, chk, g, _ = _edge(optimizer="gd")            # max_hist = 4, guard region behind it
    for k in range(7):
        _checked(dev, chk, g, None, dict(match=1.0 + k))
    assert dev.sc["recorded"] == 7
    tail = dev.hist.cpu().numpy()
    assert np.array_equal(tail[:4], np.float32([1, 2, 3, 4])) and np.all(tail[4:] == -7.0)


# ---- through the engine, noise on ---------------------------------------------------------------------------------------------------
def _attack_engine(cfg, case, backend, candidate_shape):
    model, loss_fn, payload, shared, true = case
    attacker = prepare_attack(model, loss_fn, cfg, dict(device=DEV, dtype=torch.float, backend=backend))
    torch.manual_seed(11)
    rec_models, labels, stats, shared2 = attacker.prepare_attack(payload, copy.deepcopy(shared))
    if type(attacker).__name__ == "OptimizationJointAttacker":
        labels = torch.zeros(labels.shape[0], dtype=torch.long)
    eng = attacker._get_engine(rec_models, shared2, labels)
    x0 = torch.randn(candidate_shape, generator=torch.Generator().manual_seed(5)).to(DEV)
    if hasattr(attacker, "_augmentation_plan"):
        plan = attacker._augmentation_plan(x0)
        if plan is not None:
            eng.set_augmentations(plan)
    return attacker, eng, x0


def _read_leaf(eng, joint):
    flat = lambda t: t.detach().cpu().numpy().reshape(-1).copy()  # noqa: E731
    if joint:
        return dict(x=flat(eng.joint_labels(best=False)), m=flat(eng.debug_step_state("label_m")), v=flat(eng.debug_step_state("label_v")),
                    best=flat(eng.joint_labels(best=True)))
    return dict(x=flat(eng.candidate()), m=flat(eng.debug_step_state("m")), v=flat(eng.debug_step_state("v")), best=flat(eng.best()))


def _check_engine_steps(eng, iters, meta, label_leaf=False):
    """Every iteration: read the state, run(1), read what the step read and left, and let the checker replay it in float64."""
    shape = eng.input_shape
    C, HW = shape[1], int(np.prod(shape[2:]))
    mean, std = np.float32(meta.mean), np.float32(meta.std)
    lo, hi = (-mean / std).astype(np.float32), ((np.float32(1) - mean) / std).astype(np.float32)
    cfg = OS.StepCfg.from_ccfg(eng.ccfg)
    table = np.asarray(eng._table, dtype=np.float32)
    checkers = [OS.StepChecker(cfg, table, lo, hi, C, HW)]
    if label_leaf:   # the label logits: no box, their own noise stream
        lcfg = OS.StepCfg.from_ccfg(eng.ccfg)
        lcfg.boxed, lcfg.seed = False, (cfg.seed + 0x9E3779B97F4A7C15) % 2 ** 64
        checkers.append(OS.StepChecker(lcfg, table))
    for k in range(iters):
        st = eng.status()
        befores = [dict(_read_leaf(eng, j), fmin=st["min_objective"], it=k, recorded=st["recorded"], stopped=int(st["stopped"]), trial=eng._trial)
                   for j in range(len(checkers))]
        eng.run(1)
        eng.sync()
        st = eng.status()
        terms = eng.last_terms()
        obj = dict(match=terms["match"], task_loss=terms["task_loss"], tv=terms["total_variation"], norm=terms["norm"], di=terms["deep_inversion"],
                   feat=terms["features"])
        hist = float(eng.history()[-1]) if st["recorded"] > befores[0]["recorded"] else None
        for j, chk in enumerate(checkers):
            grad = eng.debug_step_state("label_grad" if j else "grad").numpy().reshape(-1)
            gt = None
            if j == 0:
                try:
                    gt = eng.debug_step_state("grad_task").numpy().reshape(-1)
                except EngineError:
                    gt = None
            after = dict(_read_leaf(eng, j), fmin=st["min_objective"], it=k + 1, recorded=st["recorded"], stopped=int(st["stopped"]), hist=hist)
            chk.check(befores[j], grad, gt, obj, after)
    return checkers


def _begin(eng, x0, cfg, trial=0, labels=None, n=None):
    opt = cfg.optim
    eng._table = lr_table(opt.step_size, opt.get("step_size_decay"), opt.get("warmup", 0), opt.max_iterations, n)
    eng._trial = trial
    if labels is None:
        eng.begin_trial(x0, eng._table, trial=trial)
    else:
        eng.begin_joint_trial(x0, labels, eng._table, trial=trial)


def _resnet_case():
    return synthetic.make_case("resnet18", "imagenet", batch=2, seed=21, bn_random=True, image_size=64, classes=10)


ENGINE_CASES = {
    "seethroughgradients": ("seethroughgradients", {}, (2, 3, 64, 64)),
    "clip_soft": ("seethroughgradients", {"optim.grad_clip": 0.05, "optim.signed": "soft", "optim.warmup": 2, "objective.task_regularization": 0.1},
                  (2, 3, 64, 64)),
    "centerzoom_view": ("invertinggradients", {"augmentations": {"centerzoom": {"initial_fov": 48, "out_size": 64}},
                                               "differentiable_augmentations": True, "optim.langevin_noise": 0.5,
                                               "objective.task_regularization": 0.1}, (2, 3, 80, 80)),
}


@pytest.mark.parametrize("backend", ["simt", "tc"])
@pytest.mark.parametrize("name", sorted(ENGINE_CASES))
def test_engine_step_with_noise_on(name, backend):
    if name != "seethroughgradients" and backend == "tc":
        pytest.skip("the step does not depend on the GEMM back end; both are run for the shipped preset")
    preset, overrides, shape = ENGINE_CASES[name]
    cfg = get_attack_config(preset, overrides)
    case = _resnet_case()
    attacker, eng, x0 = _attack_engine(cfg, case, backend, shape)
    assert eng.ccfg.langevin_noise > 0 and eng.ccfg.noise_seed != 0
    _begin(eng, x0, cfg, trial=2)
    (chk,) = _check_engine_steps(eng, 10, case[2][0]["metadata"])
    print(f"engine {name} {backend}: max |error|/bound {chk.ratios}, either-sign {chk.either_sign}, clip-ambiguous {chk.clip_ambiguous}")
    eng.close()


def test_engine_joint_step_with_noise_on():
    """AdamW, clip and warm-up as the `tag` preset sets them, on the joint fixture's ConvNet: the label-logit leaf is stepped by the
    same kernels from its own noise stream."""
    fx = load_golden("trial_joint_adam_convnet.pt")
    case = case_from_fixture(fx)
    cfg = cfg_from_fixture(fx)
    tag = get_attack_config("tag").optim
    cfg.optim.update(optimizer=tag.optimizer, grad_clip=tag.grad_clip, warmup=3, step_size_decay=tag.step_size_decay, langevin_noise=0.01)
    attacker, eng, _ = _attack_engine(cfg, case, "simt", tuple(fx["x0"].shape))
    _begin(eng, fx["x0"].to(DEV), cfg, trial=1, labels=fx["l0"].to(DEV))
    checkers = _check_engine_steps(eng, 8, case[2][0]["metadata"], label_leaf=True)
    for which, chk in zip(("data", "labels"), checkers):
        print(f"engine joint {which}: max |error|/bound {chk.ratios}, clip-ambiguous {chk.clip_ambiguous}")
    eng.close()


# ---- every trial its own noise ---------------------------------------------------------------------------------------------------------
def test_trials_draw_their_own_noise():
    cfg = get_attack_config("seethroughgradients", {"optim.langevin_noise": 1.0, "optim.warmup": 0})
    case = _resnet_case()
    attacker, eng, x0 = _attack_engine(cfg, case, "simt", (2, 3, 64, 64))
    runs = {}
    for tag, trial in (("a", 0), ("a2", 0), ("b", 1)):
        _begin(eng, x0, cfg, trial=trial)
        eng.run(1)
        eng.sync()
        first, grad = eng.candidate().cpu(), eng.debug_step_state("grad")
        eng.run(2)
        eng.sync()
        runs[tag] = (first, eng.candidate().cpu(), grad)
    assert torch.equal(runs["a"][0], runs["a2"][0]) and torch.equal(runs["a"][1], runs["a2"][1])       # a trial index replays
    assert not torch.equal(runs["a"][0], runs["b"][0]) and not torch.equal(runs["a"][1], runs["b"][1])
    assert torch.equal(runs["a"][2], runs["b"][2])                                                     # same closure at the same x0
    # the first steps differ by what the two noise fields predict
    meta = case[2][0]["metadata"]
    mean, std = np.float32(meta.mean), np.float32(meta.std)
    lo, hi = -mean / std, (np.float32(1) - mean) / std
    scfg = OS.StepCfg.from_ccfg(eng.ccfg)
    terms = dict(match=1.0)
    pred = [OS.step(OS.new_state(x0.cpu().numpy(), trial=t), runs["a"][2].numpy(), None, scfg, np.float32(eng._table), lo, hi, terms,
                    C=3, HW=64 * 64)["x"] for t in (0, 1)]
    got = (runs["b"][0].double() - runs["a"][0].double()).numpy().reshape(-1)
    assert np.abs(pred[1] - pred[0]).max() > 1e-3
    assert np.abs(got - (pred[1] - pred[0])).max() < 1e-5
    eng.close()


@pytest.mark.parametrize("noise, differ", [(1.0, True), (0.0, False)])
def test_restarts_of_reconstruct_differ_only_through_the_noise(noise, differ):
    model, loss_fn, payload, shared, true = synthetic.make_case("convnet-tiny", "cifar", batch=1, seed=5, bn_random=True)
    cfg = get_attack_config("invertinggradients", {"restarts.num_trials": 2, "optim.max_iterations": 6, "optim.callback": 3,
                                                   "optim.langevin_noise": noise})
    attacker = prepare_attack(model, loss_fn, cfg, dict(device=DEV, dtype=torch.float, backend="simt"))
    seen = []
    run_trial = attacker._run_trial
    attacker._run_trial = lambda *a, **k: seen.append(run_trial(*a, **k).clone()) or seen[-1]
    x0 = torch.randn(1, 3, 32, 32, generator=torch.Generator().manual_seed(2))
    attacker.reconstruct(payload, copy.deepcopy(shared), {}, initial_data=x0)
    assert len(seen) == 2 and torch.equal(seen[0], seen[1]) != differ


# ---- noise off: nothing moves -----------------------------------------------------------------------------------------------------------
def test_without_noise_the_trial_index_changes_nothing():
    model, loss_fn, payload, shared, true = synthetic.make_case("convnet-tiny", "cifar", batch=2, seed=3, bn_random=True)
    cfg = get_attack_config("invertinggradients")
    case = (model, loss_fn, payload, shared, true)
    x0 = torch.randn(2, 3, 32, 32, generator=torch.Generator().manual_seed(1)).to(DEV)
    outs = []
    for use_graph, trial in ((1, 0), (0, 0), (1, 5)):
        attacker, eng, _ = _attack_engine(cfg, case, "simt", (2, 3, 32, 32))
        eng.set_option("use_graph", use_graph)
        eng.begin_trial(x0, lr_table(0.1, "step-lr", 0, 24000, 64), trial=trial)
        eng.run(12)
        eng.sync()
        outs.append((eng.candidate().cpu(), eng.history().clone(), eng.launches_per_iteration()))
        eng.close()
    import hashlib

    print("12-iteration candidate sha256:", hashlib.sha256(outs[0][0].numpy().tobytes()).hexdigest(), "launches per iteration:", outs[0][2])
    for other in outs[1:]:
        assert torch.equal(outs[0][0], other[0]) and torch.equal(outs[0][1], other[1]) and outs[0][2] == other[2] > 0
