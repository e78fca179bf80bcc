"""L-BFGS trials on the device (reference: ``optimizer_lookup`` -> ``torch.optim.LBFGS(params, lr=step_size)``,
attacks/auxiliaries/common.py:18; used by the ``beyondinfering`` / ``wei`` / ``deepleakage`` presets).

The reference hands the closure of ``_compute_objective`` (optimization_based_attack.py:146-189) to torch's L-BFGS with
its defaults -- 20 inner iterations and at most 25 closure evaluations per ``step``, history of 100 curvature pairs, no line
search, ``tolerance_grad=1e-7``, ``tolerance_change=1e-9`` -- and the optimiser state persists over the outer iterations of
``_run_trial``.

Trials with one engine, no augmentations and no Langevin noise run on the device (``Engine.begin_lbfgs_trial``, csrc/lbfgs.cu):
one captured graph per ``optimizer.step``, its inner loop a conditional WHILE node, the direction the two-loop recursion
re-associated over Gram matrices of the ring, every scalar and early exit on the device.  The constants below are the ones it
is given.  ``DeviceLBFGS`` is the host loop for the remaining cases (several model queries, augmentations, Langevin noise,
token models) and the reference the device path is tested against: every closure evaluation is one pass of the CUDA engine
(``Engine.objective_and_gradient``), the direction update the classic two-loop recursion over a ring of curvature pairs held in
two ``[history, n]`` device buffers, driven from Python with a few host reductions per inner iteration.
"""
import math

import torch

MAX_ITER, MAX_EVAL, HISTORY = 20, 25, 100          # torch.optim.LBFGS defaults (max_eval = max_iter * 5 // 4)
TOL_GRAD, TOL_CHANGE, CURVATURE_MIN = 1e-7, 1e-9, 1e-10


class DeviceLBFGS:
    """State of one L-BFGS optimiser over a flat device vector ``x`` (updated in place)."""

    def __init__(self, x):
        self.x = x
        n = x.numel()
        self.Y = torch.empty((HISTORY, n), device=x.device, dtype=x.dtype)   # gradient differences y_k
        self.S = torch.empty((HISTORY, n), device=x.device, dtype=x.dtype)   # steps s_k
        self.rho = [0.0] * HISTORY
        self.first, self.count = 0, 0      # ring: oldest slot, number of valid pairs
        self.total_iters = 0               # inner iterations over the optimiser's lifetime
        self.func_evals = 0
        self.d = None                      # last search direction
        self.t = None                      # last step length
        self.h_diag = 1.0
        self.prev_grad = None
        self.prev_loss = None

    def _slots(self):
        return [(self.first + k) % HISTORY for k in range(self.count)]   # oldest -> newest

    def _push(self, y, s, ys):
        if self.count == HISTORY:          # drop the oldest pair
            slot = self.first
            self.first = (self.first + 1) % HISTORY
        else:
            slot = (self.first + self.count) % HISTORY
            self.count += 1
        self.Y[slot].copy_(y)
        self.S[slot].copy_(s)
        self.rho[slot] = 1.0 / ys

    def _direction(self, grad):
        """-H grad by the two-loop recursion, newest pair first on the way down, oldest first on the way up."""
        q = grad.neg()
        slots = self._slots()
        alpha = {}
        for slot in reversed(slots):
            alpha[slot] = float(self.S[slot].dot(q)) * self.rho[slot]
            q.add_(self.Y[slot], alpha=-alpha[slot])
        r = q.mul_(self.h_diag)
        for slot in slots:
            beta = float(self.Y[slot].dot(r)) * self.rho[slot]
            r.add_(self.S[slot], alpha=alpha[slot] - beta)
        return r

    def step(self, closure, lr):
        """One ``optimizer.step(closure)``: returns the loss of the first closure evaluation (what the reference records)."""
        first_loss, grad = closure()
        loss = first_loss
        evals = 1
        self.func_evals += 1
        if float(grad.abs().max()) <= TOL_GRAD:
            return first_loss
        inner = 0
        while inner < MAX_ITER:
            inner += 1
            self.total_iters += 1
            if self.total_iters == 1:
                self.d = grad.neg()
                self.first, self.count, self.h_diag = 0, 0, 1.0
            else:
                y = grad - self.prev_grad
                s = self.d * self.t
                ys = float(y.dot(s))
                if ys > CURVATURE_MIN:
                    self._push(y, s, ys)
                    self.h_diag = ys / float(y.dot(y))
                self.d = self._direction(grad)
            if self.prev_grad is None:
                self.prev_grad = grad.clone()
            else:
                self.prev_grad.copy_(grad)
            self.prev_loss = loss
            self.t = min(1.0, 1.0 / float(grad.abs().sum())) * lr if self.total_iters == 1 else lr
            gtd = float(grad.dot(self.d))
            if gtd > -TOL_CHANGE:
                break
            self.x.add_(self.d, alpha=self.t)          # fixed step, no line search
            evaluated = 0
            converged = False
            if inner != MAX_ITER:                      # the reference does not re-evaluate after the last inner iteration
                loss, grad = closure()
                converged = float(grad.abs().max()) <= TOL_GRAD
                evaluated = 1
            evals += evaluated
            self.func_evals += evaluated
            if inner == MAX_ITER or evals >= MAX_EVAL or converged:
                break
            if float(self.d.abs().max()) * abs(self.t) <= TOL_CHANGE:
                break
            if abs(loss - self.prev_loss) < TOL_CHANGE:
                break
        return first_loss


def postprocess_gradient(grad, cfg_optim, iteration, lr, generator=None):
    """The closure's in-place gradient edits (optimization_based_attack.py:166-184): Langevin noise, norm clipping,
    soft / hard sign -- applied to the engine's raw d(objective)/d(candidate)."""
    from ..config import cfg_get

    noise = float(cfg_get(cfg_optim, "langevin_noise", 0.0) or 0.0)
    if noise > 0:
        grad = grad + noise * lr * torch.randn(grad.shape, device=grad.device, dtype=grad.dtype, generator=generator)
    clip = cfg_get(cfg_optim, "grad_clip")
    if clip is not None:
        norm = grad.norm()
        if float(norm) > clip:
            grad = grad * (clip / (norm + 1e-6))
    signed = cfg_get(cfg_optim, "signed")
    if signed == "soft":
        scaling = 1 - iteration / cfg_optim.max_iterations
        grad = (grad * scaling).tanh() / scaling
    elif signed == "hard":
        grad = grad.sign()
    return grad


def run_trial(engine, candidate, cfg, lr_of_iteration, lo, hi, dryrun=False, log_fn=None, iterations=None):
    """``_run_trial`` (optimization_based_attack.py:90-143) with the L-BFGS optimiser.  Returns (best candidate, history)."""
    from ..config import cfg_get

    opt = cfg.optim
    x = candidate.detach().clone().contiguous()
    flat = x.view(-1)
    name = str(opt.optimizer).lower()
    if name == "l-bfgs":
        optimizer = DeviceLBFGS(flat)
    else:  # multi-query attacks with the first-order optimisers: same host-driven loop, torch.optim update rules
        from .host_optim import LeafOptimizer

        optimizer = LeafOptimizer([flat], name)
    best = x.clone()
    fmin = float("inf")
    history = []
    total = 1 if dryrun else int(opt.max_iterations if iterations is None else iterations)
    for it in range(total):
        lr = float(lr_of_iteration[it])

        def closure():
            val, grad = engine.objective_and_gradient(x)
            return float(val), postprocess_gradient(grad, opt, it, lr).reshape(-1)

        if name == "l-bfgs":
            value = optimizer.step(closure, lr)
        else:
            value, grad = closure()
            optimizer.step([grad], lr)
        if cfg_get(opt, "boxed", False):
            torch.max(torch.min(x, hi, out=x), lo, out=x)   # :117-118
        if value < fmin:                                     # :119-121 (objective before the step, candidate after it)
            fmin = value
            best.copy_(x)
        if log_fn is not None:
            log_fn(it, value)
        if not math.isfinite(value):                         # :131-133
            break
        history.append(value)
    return best, history
