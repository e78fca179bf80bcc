"""The float64 restatement of the optimiser step (oracle/optim_step.py) and its checker, without a GPU: the Langevin-noise generator's
statistics, an fp32 emulation of the kernels' arithmetic through the whole case matrix, every tamper point, and agreement with the
fixture-pinned trial restatement (oracle/restate.py)."""
import math

import numpy as np
import pytest
import torch
from scipy import stats

import helpers
import optim_step_cases as K
from oracle import optim_step as OS

N_DRAWS = 1 << 20
KS_P_FLOOR = 1e-3   # a correct generator falls below it once in a thousand seeds; the seed is fixed


# ---- the generator -------------------------------------------------------------------------------------------------------------
def test_philox_known_answer():
    # Random123 known-answer vectors for philox4x32-10
    out = OS.philox4x32_10(np.zeros((1, 4), dtype=np.uint32), (0, 0))[0]
    assert [int(w) for w in out] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    out = OS.philox4x32_10(np.full((1, 4), 0xFFFFFFFF, dtype=np.uint32), (0xFFFFFFFF, 0xFFFFFFFF))[0]
    assert [int(w) for w in out] == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]


def test_streams_are_deterministic_and_distinct():
    idx = np.arange(4096, dtype=np.uint64)
    base = OS.gaussian(7, 0, 0, idx)
    assert np.array_equal(base, OS.gaussian(7, 0, 0, idx))
    for other in (OS.gaussian(8, 0, 0, idx), OS.gaussian(7, 1, 0, idx), OS.gaussian(7, 0, 1, idx), OS.gaussian(7 + (1 << 32), 0, 0, idx),
                  OS.gaussian(7, 0, 0, idx + np.uint64(1 << 32))):
        assert not np.any(other == base) or np.mean(other == base) < 1e-3
        assert abs(np.corrcoef(base, other)[0, 1]) < 5 / math.sqrt(idx.size)


def test_gaussian_statistics():
    idx = np.arange(N_DRAWS, dtype=np.uint64)
    z = OS.gaussian(K.SEED, 3, 11, idx)
    n = z.size
    assert np.all(np.isfinite(z))
    assert np.abs(z).max() <= OS.Z_MAX
    # sampling errors of the first four standardised moments of N(0,1): 1/n, 2/n, 6/n, 24/n
    assert abs(z.mean()) < 5 * math.sqrt(1 / n)
    assert abs(z.var() - 1) < 5 * math.sqrt(2 / n)
    assert abs(stats.skew(z)) < 5 * math.sqrt(6 / n)
    assert abs(stats.kurtosis(z)) < 5 * math.sqrt(24 / n)
    p = stats.kstest(z, "norm").pvalue
    print(f"KS p-value against N(0,1), {n} draws: {p:.4f}")
    assert p > KS_P_FLOOR
    assert abs(np.mean(z[1:] * z[:-1])) < 5 / math.sqrt(n)                       # lag 1 along the element index
    z_next = OS.gaussian(K.SEED, 3, 12, idx)
    assert abs(np.mean(z * z_next)) < 5 / math.sqrt(n)                            # lag 1 along the iteration
    assert abs(np.mean(z * OS.gaussian(K.SEED, 4, 11, idx))) < 5 / math.sqrt(n)   # and along the trial


def test_uniform_grid_edges():
    # the fp32 `(w >> 8) + 0.5`: exact below 2^23, ties-to-even above; never 0, at most 1
    u1, u2 = OS.uniforms(1, 0, 0, np.arange(1 << 16, dtype=np.uint64))
    assert u1.min() >= 2.0 ** -25 and u1.max() <= 1.0 and u2.min() > 0
    assert abs(math.sqrt(-2 * math.log(2.0 ** -25)) - OS.Z_MAX) < 1e-12


# ---- the fp32 emulation through the matrix ----------------------------------------------------------------------------------------
def run_sequence(seq, tamper=None, start=None, steps=None, checker=None):
    chk = checker or OS.StepChecker(seq.cfg, seq.lr, seq.lo, seq.hi, seq.C, seq.HW)
    state = start or K.state32(seq.x0)
    for k in range(steps or seq.steps):
        g, gt, obj = seq.inputs(k)
        after = K.emulate(state, g, gt, seq.ccfg, seq.lr, seq.lo, seq.hi, obj, seq.C, seq.HW, tamper=tamper)
        chk.check(state, g, gt, obj, after)
        state = {k_: v for k_, v in after.items() if k_ not in ("hist", "grad_norm_sq", "last_objective")}
    return chk, state


@pytest.mark.parametrize("case", K.matrix(), ids=K.case_id)
def test_emulation_passes_the_matrix(case):
    for size in K.SMALL_SIZES:
        seq = K.Sequence(case, size)
        chk, state = run_sequence(seq)
        assert state["it"] == K.STEPS and state["recorded"] == K.STEPS
        assert chk.either_sign <= 2, chk.either_sign      # |g| <= a few ulps of itself: vanishingly rare on random data
        assert max(chk.ratios.values()) <= 1.0
        print(f"{K.case_id(case)} {size}: max |error|/bound {chk.ratios}, either-sign {chk.either_sign}, clip-ambiguous {chk.clip_ambiguous}")


# tamper -> (case, buffer on which it must be reported, buffers upstream of it that must stay clean)
TAMPER_CASES = {
    "bias_t": (dict(optimizer="adam"), "x", ("m", "v")),
    "eps_inside": (dict(optimizer="adam-safe"), "x", ("m", "v")),
    "decay_after": (dict(optimizer="bert-adam"), "x", ("m", "v")),
    "mom_init": (dict(optimizer="momgd"), "m", ()),
    "nesterov_old": (dict(optimizer="momgd"), "x", ("m",)),
    "clip_before_noise": (dict(optimizer="adam", clip="active", noise=1.0), "grad_norm", ()),
    "noise_no_lr": (dict(optimizer="adam", noise=1.0), "m", ()),
    "soft_factor": (dict(optimizer="adam", signed="soft"), "m", ()),
    "box_nhwc": (dict(optimizer="gd", boxed=True), "x", ("m", "v")),
    "best_pre": (dict(optimizer="adam"), "best", ("x", "m", "v")),
    "best_le": (dict(optimizer="adam"), "best", ("x", "m", "v")),
    "it_while_stopped": (dict(optimizer="adam"), "it", ("x", "m", "v", "best")),
}


def test_every_tamper_has_a_case():
    assert set(TAMPER_CASES) == set(K.TAMPERS)


@pytest.mark.parametrize("tamper", K.TAMPERS)
def test_tamper_is_reported(tamper):
    over, where, clean = TAMPER_CASES[tamper]
    case = dict(optimizer="adam", signed=None, clip="off", noise=0.0, boxed=False, task="null")
    case.update(over)
    seq = K.Sequence(case, (2, 3, 15 * 13), seed=3)
    start = K.state32(seq.x0)
    if tamper == "mom_init":
        start["m"] = np.full_like(start["x"], 0.5)     # torch's first SGD step sets the buffer to g whatever it held
    if tamper == "box_nhwc":
        start["x"] = np.tile(np.repeat(seq.hi, seq.HW), 2).astype(np.float32)   # on the upper face; the gradient pushes half of it out
    if tamper == "it_while_stopped":
        start["stopped"] = 1
    if tamper == "best_le":
        # an objective equal to fmin must not replace best
        start["fmin"] = OS.objective_value(dict(match=0.75), seq.cfg)
        start["it"] = 5                                 # past the warm-up's first step, which runs at lr = 0
        g, gt, _ = seq.inputs(0)
        obj = dict(match=0.75)
        after = K.emulate(start, g, gt, seq.ccfg, seq.lr, seq.lo, seq.hi, obj, seq.C, seq.HW, tamper=tamper)
        with pytest.raises(OS.StepMismatch) as err:
            OS.StepChecker(seq.cfg, seq.lr, seq.lo, seq.hi, seq.C, seq.HW).check(start, g, gt, obj, after)
    else:
        with pytest.raises(OS.StepMismatch) as err:
            run_sequence(seq, tamper=tamper, start=start, steps=6)
    failed = set(err.value.buffers)
    assert where in failed, (where, str(err.value))
    assert not failed & set(clean), (clean, str(err.value))
    # and the untampered emulation passes from the same start
    run_sequence(K.Sequence(case, (2, 3, 15 * 13), seed=3), start=dict(start), steps=6)


def test_hard_sign_ambiguity_is_counted_as_planted():
    """|g| below its own rounding bound only through the noise term: the element may take either sign, and only that one."""
    case = dict(optimizer="adam", signed="hard", clip="off", noise=1.0, boxed=False, task="null")
    seq = K.Sequence(case, (1, 1, 257))
    state = K.state32(seq.x0)
    state["it"] = 5
    lr = float(seq.lr[5])
    z = OS.gaussian(seq.cfg.seed, 0, 5, np.arange(seq.n, dtype=np.uint64))
    g = np.full(seq.n, 0.5, dtype=np.float32)
    planted = (3, 100, 256)
    for i in planted:
        g[i] = np.float32(-seq.cfg.langevin_noise * lr * z[i])     # cancels the noise to within fp32 rounding
    for forced in (-1.0, 1.0):
        after = K.emulate(state, g, None, seq.ccfg, seq.lr, seq.lo, seq.hi, dict(match=1.0), seq.C, seq.HW)
        # flip the planted elements to the forced sign by redoing their update by hand through the float64 step
        choice = np.full(seq.n, np.nan)
        choice[list(planted)] = forced
        r = OS.step(state, g, None, seq.cfg, seq.lr, seq.lo, seq.hi, dict(match=1.0), sign_choice=choice)
        for key in ("x", "m", "v"):
            after[key][list(planted)] = r[key][list(planted)].astype(np.float32)
        after["best"] = after["x"].copy()
        chk = OS.StepChecker(seq.cfg, seq.lr, seq.lo, seq.hi, seq.C, seq.HW)
        chk.check(state, g, None, dict(match=1.0), after)
        assert chk.either_sign == len(planted)
    # an unambiguous element with the wrong sign is not excused
    after["m"][7] = -after["m"][7]
    with pytest.raises(OS.StepMismatch):
        OS.StepChecker(seq.cfg, seq.lr, seq.lo, seq.hi, seq.C, seq.HW).check(state, g, None, dict(match=1.0), after)


def test_clip_threshold_accepts_either_branch_only_inside_the_band():
    case = dict(optimizer="gd", signed=None, clip="active", noise=0.0, boxed=False, task="null")
    seq = K.Sequence(case, (1, 1, 256))
    g, _, obj = seq.inputs(0)
    norm = math.sqrt(float(np.sum(g.astype(np.float64) ** 2)))
    for clip, expect in ((np.float32(norm), 1), (np.float32(norm * 0.9), 0)):
        ccfg = K.make_ccfg("gd", None, float(clip))
        cfg = OS.StepCfg.from_ccfg(ccfg)
        state = K.state32(seq.x0)
        after = K.emulate(state, g, None, ccfg, seq.lr, seq.lo, seq.hi, obj)
        chk = OS.StepChecker(cfg, seq.lr)
        chk.check(state, g, None, obj, after)
        assert chk.clip_ambiguous == expect


# ---- agreement with the fixture-pinned restatement ----------------------------------------------------------------------------------
@pytest.mark.parametrize("name,noise", [("ig_convnet", 0.5), ("tag_clip_convnet", 0.5), ("l1_sgd_convnet", 0.0)])
def test_step_reproduces_trial_oracle(name, noise):
    fx = helpers.load_golden(f"trial_{name}.pt")
    orc, cfg, _ = helpers.oracle_for_fixture(fx)
    orc.dtype = torch.float64
    orc.model.double()
    orc.g = [g.double() for g in orc.g]
    orc.dm, orc.ds = orc.dm.double(), orc.ds.double()
    opt = cfg.optim
    opt.langevin_noise = noise
    iters = 5
    x0 = fx["x0"].double()
    n, (C, H, W) = x0.numel(), x0.shape[1:]
    noises = [torch.from_numpy(OS.gaussian(9, 2, it, np.arange(n, dtype=np.uint64))).view_as(x0) for it in range(iters)]
    best, hist, trace = orc.run(x0, iterations=iters, record=True, noises=noises if noise > 0 else None)
    from breaching_b200.engine import OPTIMIZERS

    kind, b1, b2, eps, wd, mom, nest = OPTIMIZERS[str(opt.optimizer).lower()]
    scfg = OS.StepCfg(optimizer=("adam", "adamw", "sgd")[kind], beta1=b1, beta2=b2, eps=eps, weight_decay=wd, momentum=mom, nesterov=bool(nest),
                      signed=opt.get("signed"), boxed=bool(opt.get("boxed", False)), max_iterations=int(opt.max_iterations),
                      langevin_noise=noise, grad_clip=opt.get("grad_clip"), seed=9)
    lo, hi = (-orc.dm / orc.ds).flatten().numpy(), ((1 - orc.dm) / orc.ds).flatten().numpy()
    state = OS.new_state(x0.numpy(), trial=2)
    for it, tr in enumerate(trace):
        state = OS.step(state, tr["raw_grad"].numpy(), None, scfg, [t["lr"] for t in trace], lo, hi, dict(match=tr["objective"]), C=C, HW=H * W)
        assert np.abs(state["x"] - tr["candidate"].numpy().reshape(-1)).max() < 1e-12, (name, it)
    assert np.abs(state["best"] - best.numpy().reshape(-1)).max() < 1e-12
    assert state["recorded"] == len(hist) and state["it"] == iters
