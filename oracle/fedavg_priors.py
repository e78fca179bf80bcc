"""FedAvg (multi-step) evaluations with the priors of the last local step.  TEST INFRASTRUCTURE ONLY.

Extends the float64 restatement of the engine's multi-step evaluation (``program_interp.MultiStepInterpreter``) and its
layer-local checker (``sweep_check.MultiStepChecker``) by task-loss regularisation and DeepInversion.

Semantics.  With 0-indexed steps (step k on slice x_k at weights W_k, ``W_{k+1} = W_k - lr G_k``, ``u_K = dh/dD``, last = K - 1)
the objective is ``Phi = h(D) + tau L(x_last, W_last) + R_DI(x_last, W_last) + TV / norm (x)``: tau is the objective's
``task_regularization`` (the reference returns the last local step's loss, objectives.py:71-72) and R_DI the DeepInversion value
of the BN-input statistics of the last step's forward (regularizers.py:222-227; the hooks act on the functional copy, so the last
forward of the iteration wins, SURVEY.md section 8(c)).

Derivation of the seeds.  Both terms depend on x_last directly and on W_last, so ``dPhi/dx_last`` gains ``tau dL/dx_last +
dR/dx_last`` and the adjoint gains ``tau G_last + dR/dW_last``: ``u_last = u_K - lr H_last u_K + tau G_last + dR/dW_last``.  The
tangent-backward sweep of step last is linear in its seeds, and a seed s entering at the logits (or at a BN input) propagates
through the rest of that sweep as a plain backward at W_last: it adds ``J_x^T s`` to the step's input gradient and ``J_W^T s``
to its tangent parameter gradients (the ``a . d_T`` source of the dual wgrad, the bias sums and the BN tangents).  Seeding
``-tau/lr (p - y)/N`` at the logits and ``-1/lr dR/dz`` at every BN input z therefore gives, through the unchanged glue,
``-lr TB_last = ... + tau dL/dx_last + dR/dx_last`` for the candidate and ``u_last = u_K - lr TG_last`` with exactly the prior
terms above.  With K = 1 only the candidate term exists.

Bounds (``PriorMultiStepChecker``, added to those of ``sweep_check``).  Only step last's relations change:

  * its logits seed is the cross-entropy tangent plus ``c (p - y) / N``, ``c = -tau / lr`` (lr the engine's fp32 value).  The extra
    term is one fp32 product of the softmax difference and ``c / N``; its rounding errors (p from ``expf`` of ``z - max z``, the
    difference, the products) are bounded like the cross-entropy seed, ``(16 + 2 |z - max z|) 2^-24 |c| (p + y) / N``, which is
    added to that bound;
  * every BN input receives the DeepInversion adjoint of the single-step relation with the layer multiplier scaled by -1/lr: the
    adjoint and its composite bound are linear in the multiplier, so the bound scales by 1/lr (the fp32 rounding of the factor,
    ``2^-24`` relative, lies inside the composite constant);
  * no seed may appear at any other step: those steps keep the single-step relations without priors.

The TG, U and final-assembly relations stay as they are: they recompute each result from the stored tangent deltas and tangent
parameter gradients, which carry the seeds, so ``u_last = u_K - lr TG_last`` includes ``tau G_last + dR/dW_last`` with the same
one-rounding bound.
"""
import torch

from oracle import program_interp as PI
from oracle import sweep_check as SC


def tangent_backward_seeded(it, V, inject=None, want_G=False, task_seed=0.0):
    """``ProgramInterpreter.tangent_backward`` of a vision program with ``task_seed`` c: ``c (p - y) / N`` added to the logits
    seed (the task-loss term of the last local step)."""
    n = it.p.shape[0]
    zdot = it.ta[it.prog.logits].view(n, -1)
    p = it.p
    seed = (p * zdot - p * (p * zdot).sum(dim=1, keepdim=True)) / n
    if task_seed != 0:
        seed = seed + task_seed * (p - it.onehot) / n
    d, TG, _ = it._reverse(seed, V=V, d_prev=it.d_B, inject=inject, want_G=want_G)
    it.d_T, it.inject = d, inject or {}
    if want_G:
        it.TG = TG
        return d[0], TG
    return d[0]


class PriorMultiStepInterpreter(PI.MultiStepInterpreter):
    """``MultiStepInterpreter`` with ``obj["task_regularization"]`` and ``obj["di"]`` on the last local step (module docstring).

    Besides the tamper points of the base class: "SEED" (``stored`` = the prior seeds ``(task coefficient, {tensor id: adjoint})``
    step k's tangent backward receives, None for none; ``contribution`` = the seeds of step last) and "DI" (at step last:
    ``stored`` = the index of the step whose forward statistics the DeepInversion prior reads); the hook returns what is used."""

    def run(self, x, labels, g, obj):
        lr, K = self.lr, len(labels)
        x = x.to(self.dtype)
        dps, N = self.prog.tensors[0].N, x.shape[0]
        self.steps, self.offsets, seen = [], [], 0
        W = [p.detach().to(self.dtype) for p in self.model.parameters()]
        self.W, self.D = [W], [[torch.zeros_like(w) for w in W]]
        for k in range(K):
            it = PI.ProgramInterpreter(self.model, self.prog, self.dtype)
            it.P, it.tamper = self.W[k], self._hook(k)
            self.offsets.append(seen)
            it.forward(x[seen:seen + dps], labels[k])
            seen = (seen + dps) % N
            G = it.backward()
            self.W.append(self._glue(k, "W", None, [w - lr * gk for w, gk in zip(self.W[k], G)], G))
            self.D.append([d - lr * gk for d, gk in zip(self.D[k], G)])
            self.steps.append(it)
        gg = [t.to(self.dtype) for t in g]
        kw = {k_: obj[k_] for k_ in ("tag_scale", "scale_scheme") if k_ in obj}
        val, u = PI.objective_direction(obj["kind"], self.D[K], gg, scale=obj.get("scale", 1.0), **kw)
        self.V = u
        last = K - 1
        tau, di = float(obj.get("task_regularization", 0.0) or 0.0), obj.get("di")
        self.seeds = None
        if tau != 0 or di is not None:
            if lr == 0:
                raise ValueError("the prior terms of a multi-step evaluation are seeded with -1/lr: lr must be nonzero")
            inject = None
            if di is not None:
                src = self._glue(last, "DI", None, last, None)
                dval, adj = self.steps[src].deep_inversion(di["scale"], di.get("first_bn_multiplier", 10))
                val = val + dval
                inject = {t: -a / lr for t, a in adj.items()}
            if tau != 0:
                val = val + tau * self.steps[last].loss
            self.seeds = (-tau / lr, inject)
        grad = torch.zeros_like(x)
        for k in reversed(range(K)):
            it, o = self.steps[k], self.offsets[k]
            it.U = u
            seeds = self._glue(k, "SEED", None, self.seeds if k == last else None, self.seeds)
            task_seed, inject = seeds if seeds is not None else (0.0, None)
            it.tangent_forward(u)
            if k > 0:
                it.gx, TG = tangent_backward_seeded(it, u, inject=inject, want_G=True, task_seed=task_seed)
            else:
                it.gx = tangent_backward_seeded(it, u, inject=inject, task_seed=task_seed)
            term = -lr * it.gx
            grad[o:o + dps] = self._glue(k, "GX", o, grad[o:o + dps] + term, term)
            if k > 0:
                u = self._glue(k, "U", None, [a - lr * b for a, b in zip(u, TG)], TG)
        pv, gp = PI.image_prior(x, obj)
        return val + pv, grad + gp


class PriorStepSource(SC.InterpreterStepSource):
    """Step k of a ``PriorMultiStepInterpreter`` run: the DeepInversion seeds are stored with the tangent deltas, as in the engine."""

    def tensor(self, which, tid):
        if which == "tangent_delta" and tid != 0:
            return self.it.d_T[tid] + self.it.inject.get(tid, 0)
        return super().tensor(which, tid)


class SeededSweepChecker(SC.SweepChecker):
    """``SweepChecker`` whose tangent-backward logits seed includes the task-loss seed ``task_seed (p - y) / N`` (vision
    programs; bound in the module docstring)."""

    def __init__(self, *args, task_seed=0.0, **kw):
        super().__init__(*args, **kw)
        self.task_seed = task_seed

    def tangent_backward(self):
        prog = self.prog
        z = self.T("val", prog.logits).flatten(1)
        zd = self.T("tangent", prog.logits).flatten(1)
        n = z.shape[0]
        p = torch.softmax(z, dim=1)
        ref = (p * zd - p * (p * zd).sum(dim=1, keepdim=True)) / n
        rng = (z - z.max(dim=1, keepdim=True).values).abs()
        mag = (p * zd.abs() + p * (p * zd.abs()).sum(dim=1, keepdim=True)) / n
        c = self.task_seed
        if c != 0:
            onehot = self._targets(n)
            ref = ref + c * (p - onehot) / n
            mag = mag + abs(c) * (p + onehot) / n
        y = self.T("tangent_delta", prog.logits).flatten(1)
        self._cmp(len(prog.ops) - 1, "TB", f"tangent_delta[t{prog.logits}] (cross-entropy + task-loss seed)", y, ref,
                  (16 + 2 * rng) * SC.U * mag + self._rounded(y, ref))
        contrib = self._check_deltas("TB", self._reverse("TB"))
        # the step's input gradient: the candidate-fed op's contribution (the priors of the whole candidate act in the final assembly)
        parts = contrib.get(0, [])
        ref = sum(p_[1] for p_ in parts)
        mag = sum(p_[3] for p_ in parts)
        bound = sum(p_[2] for p_ in parts) + 2 * SC.U * mag
        self._cmp(self.first_consumer[0], "TB", "tangent_delta[t0] (candidate gradient)", self.T("tangent_delta", 0), ref, bound)


class PriorMultiStepChecker(SC.MultiStepChecker):
    """``MultiStepChecker`` for evaluations with task-loss regularisation / DeepInversion on the last local step: that step's
    tangent backward is checked with its seeds (task seed ``-tau/lr``, DeepInversion multiplier scaled by ``-1/lr``), every other
    step without any (module docstring)."""

    def _objective_of(self, k):
        o = dict(self.obj)
        o.update(tv=None, norm=None, di=None, features=None, orthogonality=None, task_regularization=0.0)
        task_seed = 0.0
        if k == self.K - 1:
            lr = self.glue.lr
            tau = float(self.obj.get("task_regularization", 0.0) or 0.0)
            di = self.obj.get("di")
            if tau != 0:
                task_seed = -tau / lr
            if di is not None:
                o["di"] = dict(di, scale=-di["scale"] / lr)
        return o, task_seed

    def check(self, raise_on_failure=True):
        n = len(self.g)
        self.steps = []
        for k in range(self.K):
            W = [w.double() for w in self.glue.W[k]]
            o, task_seed = self._objective_of(k)
            chk = SeededSweepChecker(self.prog, W, self.bn, self.g, self.labels[k], o, self.src[k], task_seed=task_seed)
            chk.forward()
            chk.backward()
            chk.tangent_forward()
            chk.tangent_backward()
            if k > 0:
                chk.tangent_G()
            self.off_grid.update({(k, i) for i in chk.off_grid})
            self._absorb(chk, k)
            self.steps.append(chk)
        self.glue_relations(n)
        if raise_on_failure and self.findings:
            raise SC.SweepCheckError("\n".join(repr(f) for f in self.findings[:20]))
        return self.findings

