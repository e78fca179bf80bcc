"""Cases of the optimiser-step tests (CPU and GPU share them): the pairwise-pruned matrix, seeded inputs, and an fp32 emulation of
the step kernels' arithmetic -- the stand-in for the GPU where there is none, and the thing the tamper points are applied to."""
import itertools
import math

import numpy as np

import helpers  # noqa: F401  (puts the repository root on sys.path)
from breaching_b200.engine import OPTIMIZERS, AttackCfg
from breaching_b200.schedule import lr_table
from oracle import optim_step as OS

T_MAX = 40          # max_iterations of the matrix: the soft-sign factor 1 - it / T stays positive over the 25 steps
N_LR = 20           # shorter than the sequences: the last steps run with it >= n_lr, i.e. lr = 0
STEPS = 25
SIGNS = (None, "hard", "soft")
CLIPS = ("off", "unreached", "active")
NOISES = (0.0, 0.01, 1.0)
TASKS = ("null", "tau0", "tau")
SEED = 0x5EED1234ABCD


def make_ccfg(optimizer="adam", signed=None, clip=None, noise=0.0, boxed=False, tau=0.0, excludes_task=False, T=T_MAX, seed=SEED):
    c = AttackCfg()
    c.optimizer, c.beta1, c.beta2, c.adam_eps, c.weight_decay, c.momentum, c.nesterov = OPTIMIZERS[optimizer]
    c.signed_mode = {None: 0, "hard": 1, "soft": 2}[signed]
    c.boxed, c.max_iterations, c.langevin_noise = int(boxed), T, noise
    c.grad_clip = -1.0 if clip is None else clip
    c.task_regularization, c.objective_excludes_task, c.noise_seed = tau, int(excludes_task), seed
    return c


def matrix():
    """Every (noise, clip, sign) triple once; the optimiser, box and task-gradient axes cycle underneath so that every value of every
    axis and every (optimiser, sign) pair appears."""
    names = list(OPTIMIZERS)
    cases = []
    for s, sign in enumerate(SIGNS):
        for k, (noise, clip) in enumerate(itertools.product(NOISES, CLIPS)):
            cases.append(dict(optimizer=names[(k + s) % len(names)], signed=sign, clip=clip, noise=noise, boxed=bool((k + s) % 2),
                              task=TASKS[(k + 2 * s) % 3]))
    pairs = {(c["optimizer"], c["signed"]) for c in cases}
    assert pairs == set(itertools.product(names, SIGNS))
    for axis, values in (("boxed", (False, True)), ("task", TASKS)):
        assert {c[axis] for c in cases} == set(values)
    return cases


def case_id(c):
    return f"{c['optimizer']}-{c['signed']}-clip_{c['clip']}-noise{c['noise']}-{'box' if c['boxed'] else 'free'}-task_{c['task']}"


# (images, C, HW): one element; around one block; odd HW; the label leaf of the joint path; an embedding-space candidate
SMALL_SIZES = [(1, 1, 1), (1, 1, 255), (1, 1, 256), (1, 1, 257), (2, 3, 15 * 13), (40, 1, 1), (2, 96, 1)]
BIG_SIZE = (8, 3, 224 * 224)   # more elements than one grid pass: grid-stride loop, multi-block norm fold


class Sequence:
    """Seeded inputs of one case at one size: x0, per-step gradients and objective pieces, box, schedule."""

    def __init__(self, case, size, seed=0, steps=STEPS):
        self.case, self.size, self.steps = case, size, steps
        images, self.C, self.HW = size
        self.n = images * self.C * self.HW
        self.rng = np.random.default_rng(seed + 1000 * self.n)
        rng = self.rng
        self.x0 = rng.standard_normal(self.n).astype(np.float32)
        self.gscale = 1e-2
        typical = self.gscale * math.sqrt(self.n)
        clip = {"off": None, "unreached": 1e6, "active": 0.25 * typical}[case["clip"]]
        tau = 0.3 if case["task"] == "tau" else 0.0
        self.ccfg = make_ccfg(case["optimizer"], case["signed"], clip, case["noise"], case["boxed"], tau)
        self.cfg = OS.StepCfg.from_ccfg(self.ccfg)
        self.lr = np.asarray(lr_table(0.1, "cosine-decay", 4, T_MAX, N_LR), dtype=np.float32)
        self.lo = (-1.0 - 0.1 * np.arange(self.C)).astype(np.float32)     # different per channel: a wrong channel index shows
        self.hi = (0.8 + 0.07 * np.arange(self.C)).astype(np.float32)

    def inputs(self, k):
        rng = self.rng
        g = (self.gscale * rng.standard_normal(self.n)).astype(np.float32)
        gt = None if self.case["task"] == "null" else (self.gscale * rng.standard_normal(self.n)).astype(np.float32)
        obj = dict(match=float(2.0 / (1 + k) + 0.3 * rng.random()), task_loss=float(1.0 + rng.random()), tv=float(0.1 * rng.random()))
        return g, gt, obj


def state32(x0, trial=0):
    x = np.asarray(x0, dtype=np.float32).reshape(-1).copy()
    return dict(x=x, m=np.zeros_like(x), v=np.zeros_like(x), best=x.copy(), fmin=math.inf, it=0, recorded=0, stopped=0, trial=trial)


# ---- fp32 emulation of grad_norm_kernel / pixel_step_kernel / commit_kernel ------------------------------------------------------
f32 = np.float32


def _fma(a, b, c):
    return (np.asarray(a, dtype=np.float64) * np.asarray(b, dtype=np.float64) + np.asarray(c, dtype=np.float64)).astype(f32)


def gaussian32(seed, trial, it, idx):
    """The kernel's Box-Muller in fp32: log and cospi taken in float64 and rounded (within their 1 ulp), the rest fp32 operations."""
    u1, u2 = OS.uniforms(seed, trial, it, idx)
    r = np.sqrt((f32(-2.0) * np.log(u1).astype(f32)).astype(f32)).astype(f32)
    return (r * np.cos(2.0 * np.pi * u2).astype(f32)).astype(f32)


TAMPERS = ("bias_t", "eps_inside", "decay_after", "mom_init", "nesterov_old", "clip_before_noise", "noise_no_lr", "soft_factor",
           "box_nhwc", "best_pre", "best_le", "it_while_stopped")


def emulate(state, grad, grad_task, ccfg, lr_tab, lo, hi, objective, C=1, HW=1, tamper=None):
    """One step in the kernels' operation order on fp32 numpy arrays; ``tamper`` plants one of :data:`TAMPERS`."""
    cfg = OS.StepCfg.from_ccfg(ccfg)
    out = dict(state)
    out["hist"], out["grad_norm_sq"] = None, None
    if state["stopped"]:
        if tamper == "it_while_stopped":
            out["it"] = state["it"] + 1
        return out
    it = state["it"]
    n = state["x"].size
    lr = f32(lr_tab[it]) if it < len(lr_tab) else f32(0)
    tau, noise = f32(cfg.task_regularization), f32(cfg.langevin_noise)

    def raw(with_noise=True):
        g = np.asarray(grad, dtype=f32).copy()
        if grad_task is not None and tau != 0:
            g = _fma(tau, grad_task, g)
        if noise > 0 and with_noise:
            coef = noise if tamper == "noise_no_lr" else f32(noise * lr)
            g = _fma(coef, gaussian32(cfg.seed, state["trial"], it, np.arange(n, dtype=np.uint64)), g)
        return g

    g = raw()
    mul = f32(1)
    if cfg.grad_clip is not None:
        gn = raw(with_noise=tamper != "clip_before_noise")
        sq = float(np.sum(gn.astype(np.float64) ** 2))
        out["grad_norm_sq"] = sq
        nrm = f32(math.sqrt(sq)) if sq == sq else f32(np.nan)
        if nrm > f32(cfg.grad_clip):
            mul = f32(f32(cfg.grad_clip) / f32(nrm + f32(1e-6)))
    g = (g * mul).astype(f32)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        if cfg.signed == "hard":
            g = np.where(g > 0, f32(1), np.where(g < 0, f32(-1), g)).astype(f32)
        elif cfg.signed == "soft":
            soft = f32(1) - f32(f32(it + (1 if tamper == "soft_factor" else 0)) / f32(cfg.max_iterations))
            g = (np.tanh((g * soft).astype(f32).astype(np.float64)).astype(f32) / soft).astype(f32)
        x, m, v = (np.asarray(state[k], dtype=f32).copy() for k in ("x", "m", "v"))
        x_pre = x.copy()
        if cfg.optimizer == "sgd":
            d = g
            if cfg.momentum != 0:
                mom = f32(cfg.momentum)
                m_old = m.copy()
                m = g.copy() if (it == 0 and tamper != "mom_init") else _fma(mom, m, g)
                d = _fma(mom, m_old if tamper == "nesterov_old" else m, g) if cfg.nesterov else m
            x = _fma(-lr, d, x)
        else:
            t = float(it if tamper == "bias_t" else it + 1)
            bc1 = 1.0 - float(f32(cfg.beta1)) ** t
            bc2s = math.sqrt(1.0 - float(f32(cfg.beta2)) ** t)
            step_size = f32(float(lr) / bc1) if bc1 != 0 else f32(np.inf)
            decay = f32(1.0 - float(lr) * cfg.weight_decay)
            if cfg.optimizer == "adamw" and tamper != "decay_after":
                x = (x * decay).astype(f32)
            b1, b2 = f32(cfg.beta1), f32(cfg.beta2)
            m = _fma(f32(1) - b1, (g - m).astype(f32), m)
            v = _fma(f32(1) - b2, (g * g).astype(f32), (v * b2).astype(f32))
            if tamper == "eps_inside":
                denom = (np.sqrt((v + f32(cfg.eps)).astype(f32)) / f32(bc2s)).astype(f32)
            else:
                denom = ((np.sqrt(v) / f32(bc2s)).astype(f32) + f32(cfg.eps)).astype(f32)
            x = _fma(-step_size, (m / denom).astype(f32), x)
            if cfg.optimizer == "adamw" and tamper == "decay_after":
                x = (x * decay).astype(f32)
        if cfg.boxed:
            idx = np.arange(n)
            ch = idx % C if tamper == "box_nhwc" else (idx // HW) % C
            x = np.where(np.isnan(x), x, np.maximum(np.minimum(x, np.asarray(hi, dtype=f32)[ch]), np.asarray(lo, dtype=f32)[ch])).astype(f32)
    phi = OS.objective_value(objective, cfg)
    fmin32 = f32(state["fmin"])
    improved = bool(f32(phi) <= fmin32) if tamper == "best_le" else bool(f32(phi) < fmin32)
    out.update(x=x, m=m, v=v, last_objective=phi)
    if improved:
        out["best"] = (x_pre if tamper == "best_pre" else x).copy()
    if f32(phi) < fmin32:
        out["fmin"] = phi
    if math.isfinite(phi):
        out["hist"] = phi
        out["recorded"] = state["recorded"] + 1
    else:
        out["stopped"] = 1
    out["it"] = it + 1
    return out
