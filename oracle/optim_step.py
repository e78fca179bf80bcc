"""Float64 restatement of the tail of one iteration -- gradient post-processing, optimiser update, box projection, best-so-far and the
trial bookkeeping (optimization_based_attack.py:112-135,166-184; torch.optim.Adam / AdamW / SGD) -- on flat buffers, the counter-based
generator of the Langevin noise in numpy integer arithmetic, and a local checker with per-element bounds for the fp32 kernels
(``grad_norm_kernel``, ``pixel_step_kernel``, ``commit_kernel`` of csrc/objective.cu).

The generator
-------------
Philox4x32-10 with key = the 64-bit seed and counter = (element low, element high, iteration, trial).  Output words 0 and 1 give the
uniforms ``((w >> 8) + 0.5) / 2^24`` and Box-Muller gives ``sqrt(-2 ln u1) cos(2 pi u2)``.  The kernel forms ``(w >> 8) + 0.5`` in
fp32: exact below 2^23, rounded to even above (the upper half of the unit interval sits on a 23-bit grid, and the single value
``w >> 8 == 2^24 - 1`` gives u1 = 1 and a draw of exactly 0).  :func:`uniforms` restates that rounding; everything after it is float64.
u1 >= 2^-25, so ``|z| <= sqrt(50 ln 2) < 5.8871`` (:data:`Z_MAX`); u1 <= 1, so no draw is non-finite.

Bounds
------
``U = 2^-24`` is the unit roundoff of fp32: one correctly rounded operation (+, *, /, fma, sqrtf and / under nvcc's default
``-prec-sqrt=true -prec-div=true``) returns its exact result times ``1 + d``, ``|d| <= U``.  The CUDA programming guide's table of
maximum ulp errors gives logf 1, cospif 1 and tanhf 2 ulp; one ulp is at most ``2 U`` relative.  The checker feeds the float64 step the
kernel's own inputs of that step and pushes an absolute error bound ``E`` through the same chain of operations, first order in U:

* z:      ln 2U -> sqrt U + U, cos 2U, product U: ``|dz| <= 6 U |z|``; the checker uses ``Z_ULPS = 8``.
* raw g:  one fma for the task term (``U |g|``), one for the noise: the coefficient ``fl(noise * lr)`` (U) times z (8 U) plus the fma
          (``U |g|``): ``E += 9 U |c z| + U |g|``.
* clip:   the squares are summed in double, so ``| |g_k| - |g_64| | <= |E|_2``; the fp32 cast of the root and of ``norm + 1e-6`` and the
          division add ``3 U``.  The multiplier is continuous at ``norm == clip`` (up to 1e-6 / clip), so inside that band either
          branch is accepted (``clip_ambiguous``).
* sign:   hard -- exact unless ``|g_64| <= E``; such an element may come out as -1, 0 or +1, and the step is accepted if one of the
          three explains x, m and v of that element together; they are counted (``either_sign``).  soft -- the factor
          ``s = 1 - it / T`` carries ``U (it / T + s)`` absolute, which is *not* small relative to s late in a trial; tanh is
          1-Lipschitz with slope ``1 - tanh^2`` at the near end of the interval, tanhf adds ``4 U |tanh|``, the division U.
* update: every fma / product / quotient adds U of its result; ``fl(1 - beta)`` U; sqrt halves a relative error (and
          ``|sqrt a - sqrt b| <= sqrt |a - b|`` near 0); the bias corrections and ``1 - lr * weight_decay`` are formed in double and
          cast once (U each).  The formulas are spelled out in :meth:`StepChecker._bounds`.
* box:    min / max are exact and 1-Lipschitz.
* exact:  ``best`` (bitwise the kernel's own new x, or untouched), ``fmin``, ``it``, ``recorded``, ``stopped``, the history entry and
          ``last_objective``: phi is the same double sum rounded once to fp32, compared as ``float32(phi) < float32(fmin)``.

``SLACK = 2`` multiplies every bound: second-order terms and the few places where the first-order count is not tight.  The tests print
the largest observed ``|error| / bound``.
"""
import math
from dataclasses import dataclass
from typing import Optional

import numpy as np

U = 2.0 ** -24
SLACK = 2.0
Z_ULPS = 8.0
Z_MAX = math.sqrt(50.0 * math.log(2.0))

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_LO = np.uint64(0xFFFFFFFF)


def philox4x32_10(counter, key):
    """``counter``: uint32 array [..., 4]; ``key``: (k0, k1).  Returns the four output words, uint32 [..., 4]."""
    c = [np.asarray(counter[..., j], dtype=np.uint64) for j in range(4)]
    k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = _M0 * c[0], _M1 * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ np.uint64(k0), p1 & _LO, (p0 >> np.uint64(32)) ^ c[3] ^ np.uint64(k1), p0 & _LO]
        k0, k1 = (k0 + _W0) & 0xFFFFFFFF, (k1 + _W1) & 0xFFFFFFFF
    return np.stack(c, axis=-1).astype(np.uint32)


def _words(seed, trial, it, idx):
    idx = np.asarray(idx, dtype=np.uint64)
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    ctr = np.empty(idx.shape + (4,), dtype=np.uint32)
    ctr[..., 0] = (idx & _LO).astype(np.uint32)
    ctr[..., 1] = (idx >> np.uint64(32)).astype(np.uint32)
    ctr[..., 2] = np.uint32(int(it) & 0xFFFFFFFF)
    ctr[..., 3] = np.uint32(int(trial) & 0xFFFFFFFF)
    return philox4x32_10(ctr, (seed & 0xFFFFFFFF, seed >> 32))


def uniforms(seed, trial, it, idx):
    """(u1, u2) as float64, on the grid the kernel's fp32 ``(w >> 8) + 0.5`` lands on."""
    w = _words(seed, trial, it, idx)
    half = np.float32(0.5)
    u = [((w[..., j] >> np.uint32(8)).astype(np.float32) + half).astype(np.float64) * 2.0 ** -24 for j in (0, 1)]
    return u[0], u[1]


def gaussian(seed, trial, it, idx):
    """The N(0,1) draw of element ``idx`` in iteration ``it`` of trial ``trial`` (float64)."""
    u1, u2 = uniforms(seed, trial, it, idx)
    return np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)


# -----------------------------------------------------------------------------------------------------------------------------------
@dataclass
class StepCfg:
    optimizer: str = "adam"            # "adam" | "adamw" | "sgd"
    beta1: float = 0.9
    beta2: float = 0.999
    eps: float = 1e-8
    weight_decay: float = 0.0
    momentum: float = 0.0
    nesterov: bool = False
    signed: Optional[str] = None       # None | "hard" | "soft"
    boxed: bool = False
    max_iterations: int = 1
    langevin_noise: float = 0.0
    grad_clip: Optional[float] = None
    task_regularization: float = 0.0
    objective_excludes_task: bool = False
    seed: int = 0

    @classmethod
    def from_ccfg(cls, c):
        """From the engine's ``AttackCfg`` (any object with its fields): the fp32 values the kernels receive, widened."""
        return cls(optimizer=("adam", "adamw", "sgd")[c.optimizer], beta1=float(c.beta1), beta2=float(c.beta2), eps=float(c.adam_eps),
                   weight_decay=float(c.weight_decay), momentum=float(c.momentum), nesterov=bool(c.nesterov),
                   signed=(None, "hard", "soft")[c.signed_mode], boxed=bool(c.boxed), max_iterations=int(c.max_iterations),
                   langevin_noise=float(c.langevin_noise), grad_clip=None if c.grad_clip < 0 else float(c.grad_clip),
                   task_regularization=float(c.task_regularization), objective_excludes_task=bool(c.objective_excludes_task),
                   seed=int(c.noise_seed))


PIECES = ("match", "tv", "norm", "di", "feat")


def objective_value(objective, cfg):
    """phi as the kernels form it: the double sum of the pieces, the task loss times task_regularization unless the objective
    excludes it, rounded once to fp32."""
    phi = 0.0
    for key in PIECES:
        phi = phi + float(objective.get(key, 0.0))
    tau = 0.0 if cfg.objective_excludes_task else cfg.task_regularization
    if tau != 0.0:
        phi = phi + tau * float(objective.get("task_loss", 0.0))
    with np.errstate(over="ignore"):
        return float(np.float32(phi))


def new_state(x0, trial=0):
    x = np.asarray(x0, dtype=np.float64).reshape(-1).copy()
    return dict(x=x, m=np.zeros_like(x), v=np.zeros_like(x), best=x.copy(), fmin=math.inf, it=0, recorded=0, stopped=0, trial=trial)


def step(state, grad, grad_task, cfg, lr_table, lo, hi, objective, noise=None, C=1, HW=1, sign_choice=None, clip_branch=None):
    """One iteration's tail in float64.  ``state``: dict(x, m, v, best, fmin, it, recorded, stopped, trial) on flat arrays;
    ``objective``: dict of the pieces of phi (match, task_loss, tv, norm, di, feat) of the evaluation *before* this step.
    ``noise``: the N(0,1) field (default: :func:`gaussian` of (cfg.seed, trial, it)).  ``sign_choice`` (array, NaN = no override)
    forces the post-sign gradient of single elements and ``clip_branch`` (bool) the clip decision: the checker's either-way cases.
    Returns the new state plus ``hist`` (the history entry or None), ``grad_norm_sq``, ``last_objective`` and ``aux`` (intermediates)."""
    out = dict(state)
    out["hist"], out["grad_norm_sq"], out["aux"] = None, None, None
    out["last_objective"] = state.get("last_objective")
    if state["stopped"]:
        return out
    it, n_lr = int(state["it"]), len(lr_table)
    x, m, v = (np.asarray(state[k], dtype=np.float64) for k in ("x", "m", "v"))
    n = x.size
    lr = float(lr_table[it]) if it < n_lr else 0.0
    T = cfg.max_iterations
    # closure tail (:166-184)
    g = np.asarray(grad, dtype=np.float64).reshape(-1).copy()
    aux = dict(lr=lr, g0=g.copy())
    if grad_task is not None and cfg.task_regularization != 0.0:
        g = g + cfg.task_regularization * np.asarray(grad_task, dtype=np.float64).reshape(-1)
    aux["g1"] = g.copy()
    z = None
    if cfg.langevin_noise > 0:
        z = gaussian(cfg.seed, state.get("trial", 0), it, np.arange(n, dtype=np.uint64)) if noise is None else np.asarray(noise, dtype=np.float64).reshape(-1)
        g = g + cfg.langevin_noise * lr * z
    aux["z"], aux["g2"] = z, g.copy()
    mul, norm = 1.0, None
    if cfg.grad_clip is not None:
        norm = math.sqrt(float(np.sum(g * g)))
        out["grad_norm_sq"] = norm * norm
        clipped = (norm > cfg.grad_clip) if clip_branch is None else bool(clip_branch)   # NaN norm: no clip, like torch
        if clipped:
            mul = cfg.grad_clip / (norm + 1e-6)
        g = g * mul
    aux["norm"], aux["mul"], aux["g3"] = norm, mul, g.copy()
    soft = None
    if cfg.signed == "hard":
        g = np.sign(g)          # keeps 0 and NaN
    elif cfg.signed == "soft":
        soft = 1.0 - it / T
        with np.errstate(divide="ignore", invalid="ignore"):
            g = np.tanh(g * soft) / soft
    if sign_choice is not None:
        g = np.where(np.isnan(sign_choice), g, sign_choice)
    aux["soft"], aux["g"] = soft, g.copy()
    # optimiser (torch.optim.SGD / Adam / AdamW, single tensor, no amsgrad / maximize)
    t = it + 1
    if cfg.optimizer == "sgd":
        d = g
        if cfg.momentum != 0.0:
            m = g.copy() if it == 0 else cfg.momentum * m + g
            d = g + cfg.momentum * m if cfg.nesterov else m
        xn = x - lr * d
        aux.update(d=d)
    else:
        x1 = x * (1.0 - lr * cfg.weight_decay) if cfg.optimizer == "adamw" else x
        m = m + (1.0 - cfg.beta1) * (g - m)
        v = cfg.beta2 * v + (1.0 - cfg.beta2) * g * g
        bc1, bc2 = 1.0 - cfg.beta1 ** t, 1.0 - cfg.beta2 ** t
        with np.errstate(invalid="ignore", divide="ignore"):
            denom = np.sqrt(v) / math.sqrt(bc2) + cfg.eps
            ratio = m / denom
        xn = x1 - (lr / bc1) * ratio
        aux.update(x1=x1, bc1=bc1, bc2s=math.sqrt(bc2), denom=denom, ratio=ratio, step=lr / bc1)
    if cfg.boxed:   # :117-118, per channel of an [images, C, HW] candidate
        ch = (np.arange(n) // HW) % C
        lo_, hi_ = np.asarray(lo, dtype=np.float64)[ch], np.asarray(hi, dtype=np.float64)[ch]
        xn = np.where(np.isnan(xn), xn, np.maximum(np.minimum(xn, hi_), lo_))   # torch.min / max propagate NaN
    # best-so-far on the pre-step objective with the post-step candidate (:119-121), history, stop (:131-135)
    phi = objective_value(objective, cfg)
    improved = bool(np.float32(phi) < np.float32(state["fmin"]))
    aux["improved"] = improved
    out.update(x=xn, m=m, v=v, aux=aux, last_objective=phi)
    if improved:
        out["best"], out["fmin"] = xn.copy(), phi
    if math.isfinite(phi):
        out["hist"] = phi
        out["recorded"] = state["recorded"] + 1
    else:
        out["stopped"] = 1
    out["it"] = it + 1
    return out


# -----------------------------------------------------------------------------------------------------------------------------------
class StepMismatch(AssertionError):
    """``buffers``: the names of the outputs that disagree."""

    def __init__(self, failures, where=""):
        super().__init__(where + "; ".join(failures))
        self.buffers = [f.split(":")[0] for f in failures]


class StepChecker:
    """Local check of one step: ``check(before, grad, grad_task, objective, after)`` runs :func:`step` on the kernel's own ``before``
    state and inputs and compares every output.  ``before`` / ``after``: dicts as :func:`new_state` (arrays of any float dtype);
    ``after`` also carries ``hist`` (the history entry written, or None), ``grad_norm_sq`` and ``last_objective`` when available.
    Collects ``ratios`` (largest |error| / bound per buffer), ``either_sign`` and ``clip_ambiguous`` over all calls."""

    def __init__(self, cfg, lr_table, lo=None, hi=None, C=1, HW=1):
        self.cfg, self.lr_table, self.lo, self.hi, self.C, self.HW = cfg, np.asarray(lr_table, dtype=np.float64), lo, hi, C, HW
        self.ratios = {}
        self.either_sign = 0
        self.clip_ambiguous = 0
        self.steps = 0

    # error bounds of the kernel's x, m, v around the float64 step `r`, given the bound E3 of the pre-sign gradient
    def _bounds(self, before, r, E3):
        cfg, a = self.cfg, r["aux"]
        lr, g = a["lr"], a["g"]
        x, m0, v0 = (np.asarray(before[k], dtype=np.float64) for k in ("x", "m", "v"))
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            if cfg.signed == "hard":
                E4 = np.zeros_like(g)
            elif cfg.signed == "soft":
                s = a["soft"]
                q = 1.0 - s
                Es = U * (abs(q) + abs(s))
                arg = a["g3"] * s
                Ea = E3 * abs(s) + np.abs(a["g3"]) * Es + U * np.abs(arg)
                th = np.tanh(arg)
                slope = 1.0 - np.tanh(np.maximum(np.abs(arg) - Ea, 0.0)) ** 2
                Eth = slope * Ea + 4 * U * np.abs(th)
                E4 = Eth / abs(s) + np.abs(g) * Es / abs(s) + U * np.abs(g)
            else:
                E4 = E3
            if cfg.optimizer == "sgd":
                Em, Ev = np.zeros_like(g), np.zeros_like(g)
                Ed = E4
                if cfg.momentum != 0.0:
                    Em = E4 + U * np.abs(r["m"])
                    Ed = cfg.momentum * Em + E4 + U * np.abs(a["d"]) if cfg.nesterov else Em
                Ex = lr * Ed + U * np.abs(r["x"]) + U * np.abs(lr * a["d"])
            else:
                b1, b2 = cfg.beta1, cfg.beta2
                Ex1 = 2 * U * np.abs(a["x1"]) if cfg.optimizer == "adamw" else 0.0
                Em = (1 - b1) * (E4 + 2 * U * np.abs(g - m0)) + U * np.abs(r["m"])
                Ev = (1 - b2) * (2 * np.abs(g) * E4 + E4 * E4 + 2 * U * g * g) + U * b2 * np.abs(v0) + U * np.abs(r["v"])
                root = np.sqrt(r["v"])
                Esq = np.minimum(np.where(root > 0, Ev / (2 * np.maximum(root, 1e-300)), np.inf), np.sqrt(Ev)) + U * root
                Eden = Esq / a["bc2s"] + 2 * U * root / a["bc2s"] + U * a["denom"]
                Er = Em / a["denom"] + np.abs(a["ratio"]) * Eden / a["denom"] + U * np.abs(a["ratio"])
                Ex = Ex1 + a["step"] * Er + 2 * U * a["step"] * np.abs(a["ratio"]) + U * np.abs(r["x"]) + U * np.abs(a["x1"])
        tiny = 1e-45   # one fp32 denormal: results that underflow
        return dict(x=SLACK * Ex + tiny, m=SLACK * Em + tiny, v=SLACK * Ev + tiny)

    def _raw_bound(self, r):
        cfg, a = self.cfg, r["aux"]
        E = np.zeros_like(a["g0"])
        if not np.array_equal(a["g1"], a["g0"], equal_nan=True):
            E = E + U * np.abs(a["g1"])
        if a["z"] is not None:
            cz = cfg.langevin_noise * a["lr"] * a["z"]
            E = E + (Z_ULPS + 1) * U * np.abs(cz) + U * np.abs(a["g2"])
        return E

    @staticmethod
    def _within(got, want, bound):
        got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
        nan_g, nan_w = np.isnan(got), np.isnan(want)
        with np.errstate(invalid="ignore"):
            err = np.abs(got - want)
            ratio = np.where(nan_g | nan_w, np.where(nan_g == nan_w, 0.0, np.inf), np.where(got == want, 0.0, err / bound))
        return ratio

    def check(self, before, grad, grad_task, objective, after, noise=None):
        cfg = self.cfg
        self.steps += 1
        fail = []
        r = step(before, grad, grad_task, cfg, self.lr_table, self.lo, self.hi, objective, noise=noise, C=self.C, HW=self.HW)
        exact = ["fmin", "it", "recorded", "stopped"]
        if before["stopped"]:
            for key in ("x", "m", "v", "best"):
                if not np.array_equal(np.asarray(after[key]), np.asarray(before[key]), equal_nan=True):
                    fail.append(f"{key}: changed although the trial is stopped")
            for key in exact:
                if after[key] != before[key]:
                    fail.append(f"{key}: {after[key]} != {before[key]} although the trial is stopped")
            if after.get("hist") is not None:
                fail.append("hist: written although the trial is stopped")
            if fail:
                raise StepMismatch(fail)
            return r
        for key in exact + ["last_objective", "hist"]:
            if key in after:
                got, want = after[key], r[key]
                same = (got is None and want is None) or (got is not None and want is not None and
                                                          (got == want or (isinstance(got, float) and math.isnan(got) and math.isnan(want))))
                if not same:
                    fail.append(f"{key}: kernel {got} != float64 step {want}")
        # best: bitwise the kernel's own new x, or untouched
        ref_best = after["x"] if r["aux"]["improved"] else before["best"]
        if not np.array_equal(np.asarray(after["best"]), np.asarray(ref_best), equal_nan=True):
            fail.append("best: not the post-step candidate" if r["aux"]["improved"] else "best: changed without an improvement")
        E2 = self._raw_bound(r)
        variants = [(r, E2, False)]
        if cfg.grad_clip is not None:
            norm = r["aux"]["norm"]
            with np.errstate(invalid="ignore"):
                En = SLACK * (float(np.sqrt(np.nansum(E2 * E2))) + 4 * U * norm) if math.isfinite(norm) else 0.0
            if after.get("grad_norm_sq") is not None:
                got = math.sqrt(after["grad_norm_sq"]) if after["grad_norm_sq"] >= 0 else math.nan
                ok = (math.isnan(got) and math.isnan(norm)) or abs(got - norm) <= En + 1e-300
                self._note("grad_norm", 0.0 if (got == norm or (math.isnan(got) and math.isnan(norm))) else abs(got - norm) / (En + 1e-300))
                if not ok:
                    fail.append(f"grad_norm: kernel {got!r} vs {norm!r}, bound {En:.3e}")
            Emul = r["aux"]["mul"] * (En / norm + 3 * U) if math.isfinite(norm) and norm > 0 else 0.0
            variants = [(r, E2 * r["aux"]["mul"] + np.abs(r["aux"]["g3"]) * (Emul + U), False)]
            if math.isfinite(norm) and abs(norm - cfg.grad_clip) <= En + 4 * U * cfg.grad_clip:
                self.clip_ambiguous += 1
                r2 = step(before, grad, grad_task, cfg, self.lr_table, self.lo, self.hi, objective, noise=noise, C=self.C, HW=self.HW,
                          clip_branch=not (norm > cfg.grad_clip))
                variants.append((r2, E2 * r2["aux"]["mul"] + np.abs(r2["aux"]["g3"]) * (Emul + U + 1e-6 / cfg.grad_clip), True))
        best_fail, best_ratios, best_either = None, None, 0
        for rv, E3, _ in variants:
            ok_el, ratios, either = self._elements(before, grad, grad_task, objective, after, rv, E3, noise)
            vfail = [f"{key}: {int((~(ratios[key] <= 1.0)).sum())} element(s) outside the bound, worst |error|/bound = {np.nanmax(ratios[key]):.3g} "
                     f"at {int(np.nanargmax(ratios[key]))}" for key in ("x", "m", "v") if not np.all(ratios[key] <= 1.0)]
            if best_fail is None or len(vfail) < len(best_fail):
                best_fail, best_ratios, best_either = vfail, ratios, either
            if not vfail:
                break
        self.either_sign += best_either
        for key in ("x", "m", "v"):
            finite = best_ratios[key][np.isfinite(best_ratios[key])]
            self._note(key, float(finite.max()) if finite.size else 0.0)
        fail += best_fail
        if fail:
            raise StepMismatch(fail, f"step it={before['it']}: ")
        return r

    def _note(self, key, ratio):
        self.ratios[key] = max(self.ratios.get(key, 0.0), ratio)

    def _elements(self, before, grad, grad_task, objective, after, r, E3, noise):
        """Per-element |error| / bound of x, m, v against step result ``r``; under hard sign an element with ``|g| <= E`` is also
        tried with each of -1, 0, +1 and takes the choice that explains x, m and v together best."""
        cfg = self.cfg
        bounds = self._bounds(before, r, E3)
        ratios = {key: self._within(after[key], r[key], bounds[key]) for key in ("x", "m", "v")}
        either = 0
        if cfg.signed == "hard":
            with np.errstate(invalid="ignore"):
                amb = np.abs(r["aux"]["g3"]) <= SLACK * E3
                amb &= (E3 > 0)
            either = int(amb.sum())
            if either:
                worst = np.maximum(np.maximum(ratios["x"], ratios["m"]), ratios["v"])
                for s in (-1.0, 0.0, 1.0):
                    choice = np.where(amb, s, np.nan)
                    ra = step(before, grad, grad_task, cfg, self.lr_table, self.lo, self.hi, objective, noise=noise, C=self.C, HW=self.HW,
                              sign_choice=choice, clip_branch=(r["aux"]["mul"] != 1.0) if cfg.grad_clip is not None else None)
                    ba = self._bounds(before, ra, E3)
                    alt = {key: self._within(after[key], ra[key], ba[key]) for key in ("x", "m", "v")}
                    alt_worst = np.maximum(np.maximum(alt["x"], alt["m"]), alt["v"])
                    take = amb & (alt_worst < worst)
                    for key in ("x", "m", "v"):
                        ratios[key] = np.where(take, alt[key], ratios[key])
                    worst = np.where(take, alt_worst, worst)
        ok = (ratios["x"] <= 1.0) & (ratios["m"] <= 1.0) & (ratios["v"] <= 1.0)
        return ok, ratios, either
