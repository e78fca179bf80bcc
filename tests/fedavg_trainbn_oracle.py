"""FedAvg (multi-step) evaluations of train-mode BatchNorm networks.  TEST INFRASTRUCTURE ONLY.

Without BN buffers from the server or the user, every local step normalises with its own batch statistics (the reference's
``UserMultiStep`` trains in train mode, cases/users.py:345-353, and ``_grad_fn_multi_step`` runs every step so,
objectives.py:48-72).  The float64 restatement of the multi-step evaluation (``oracle.fedavg_priors.PriorMultiStepInterpreter``)
and its layer-local checker (``PriorMultiStepChecker``) already carry the train-mode rules of every sweep; what a multi-step
evaluation adds is the tangent of the gamma / beta gradients in the Hessian-vector product of steps k > 0 (sweep "TG").

Rule.  With du the ReLU-masked delta of the op's output, xh the normalised input, m(.) the per-channel mean over (N, H, W) and
inv = 1 / sigma of the batch, ``G_gamma = sum du xh`` and ``G_beta = sum du``.  Along the direction, du becomes du' (the masked
tangent delta) and xh becomes ``xh' = inv (x' - m(x') - xh m(xh x'))`` (the tangent-forward rule), so

    TG_gamma = sum (du' xh + du xh'),     TG_beta = sum du'.

These are the undivided sums whose means the tangent backward of the op needs anyway (its ``m(du')`` and ``m(du' xh + du xh')``).

Bound.  The engine forms both sums over P = N H W pixels in fp32, TG_gamma from two products per pixel: ``(2P + 4) 2^-23`` times
the sum of the magnitudes, plus twice the composite constant of the fp32 batch statistics (``SweepChecker._bn_train``) for the
error of xh and of the means inside xh'.  TG_beta is a plain sum, ``(P + 4) 2^-23 sum |du'|``.  The magnitude of xh in these
bounds, and in the sweep-B gamma relation of a train-mode op, is ``|x inv| + |mean inv|`` (``_bn_param_grads``).

The base classes are used unchanged: each multi-step run swaps in the subclasses below for its steps (``_steps_use``).
"""
import contextlib
import copy
import dataclasses

from breaching_b200 import compiler as C
from oracle import fedavg_priors as FP
from oracle import program_interp as PI
from oracle import sweep_check as SC


def _train_bn(op):
    return op.kind == C.OP_BNACT and op.has_bn and op.bn_train


@contextlib.contextmanager
def _steps_use(module, name, cls):
    """While active, ``module.<name>`` (the class a multi-step run instantiates for each step) is ``cls``."""
    base = getattr(module, name)
    setattr(module, name, cls)
    try:
        yield
    finally:
        setattr(module, name, base)


class TrainBnInterpreter(PI.ProgramInterpreter):
    """``ProgramInterpreter`` with the tangent parameter gradients of train-mode BN (module docstring)."""

    def _tangent_param_grads(self, i, op, dout, d_prev, put):
        if not _train_bn(op):
            return super()._tangent_param_grads(i, op, dout, d_prev, put)
        mask = (self.a[op.tout] > 0).to(self.dtype) if op.relu else 1.0
        duT, duB = dout * mask, self.du_B[i]
        put(op.gamma, (duT * self.aux[i] + duB * self.taux[i]).sum(dim=(0, 2, 3)))
        put(op.beta, duT.sum(dim=(0, 2, 3)))


class TrainBnMultiStepInterpreter(FP.PriorMultiStepInterpreter):
    """``PriorMultiStepInterpreter`` whose steps are ``TrainBnInterpreter`` s."""

    def run(self, x, labels, g, obj):
        with _steps_use(PI, "ProgramInterpreter", TrainBnInterpreter):
            return super().run(x, labels, g, obj)


class TrainBnSweepChecker(FP.SeededSweepChecker):
    """``SeededSweepChecker`` whose sweep TG also checks the gamma / beta tangents of train-mode BN (bound in the module
    docstring); every other relation is the base class's."""

    def tangent_G(self):
        prog = self.prog
        train = [i for i, op in enumerate(prog.ops) if _train_bn(op)]
        # the base relations of every other op: the train-mode BN ops are hidden from its loop
        view = copy.copy(prog)
        view.ops = [dataclasses.replace(op, has_bn=False) if i in train else op for i, op in enumerate(prog.ops)]
        self.prog = view
        try:
            super().tangent_G()
        finally:
            self.prog = prog
        m, A = self._m, (lambda t: t.abs())
        for i in train:
            op = prog.ops[i]
            x, dT = self.T("val", op.tin), self.T("tangent_delta", op.tout)
            mask = (self.T("val", op.tout) > 0).double() if op.relu else 1.0
            duT, duB = dT * mask, self.T("delta", op.tout) * mask
            mean, _, inv, xh, c = self._bn_train(op, x)
            xd = self._tangent_in(op)
            xhd = inv * (xd - m(xd) - xh * m(xh * xd))
            xhm = A(x * inv) + A(mean * inv)
            xhdm = inv * (A(xd) + m(A(xd)) + A(xh) * m(A(xh * xd)))
            Pch = x.shape[0] * x.shape[2] * x.shape[3]
            s = (A(duT) * xhm + A(duB) * xhdm).sum(dim=(0, 2, 3))
            self._cmp(i, "TG", f"TG[{op.gamma}] (train-mode BN gamma tangent)", self.Pm("TG", op.gamma),
                      (duT * xh + duB * xhd).sum(dim=(0, 2, 3)), ((2 * Pch + 4) * SC.U2 + 2 * c.view(-1)) * s)
            self._cmp(i, "TG", f"TG[{op.beta}] (train-mode BN beta tangent)", self.Pm("TG", op.beta), duT.sum(dim=(0, 2, 3)),
                      (Pch + 4) * SC.U2 * A(duT).sum(dim=(0, 2, 3)))

    def _bn_param_grads(self, i, op, du, xh, xhm):
        """The sweep-B gamma / beta relation of the base class, with the magnitude of xh taken as ``|x inv| + |mean inv|`` for a
        train-mode op.  The kernels form xh as ``x inv + nrm`` (nrm = -mean inv) from the fp32 batch statistics, so its error
        scales with the two terms of that sum, not with |xh|: where a channel's values sit close to their mean (a handful of
        pixels per channel, ResNet-18's last stage at one image per step) |xh| is far smaller than either term."""
        if op.bn_train:
            x = self.T("val", op.tin)
            mean, _, inv, _, _ = self._bn_train(op, x)
            xhm = (x * inv).abs() + (mean * inv).abs()
        super()._bn_param_grads(i, op, du, xh, xhm)


class TrainBnMultiStepChecker(FP.PriorMultiStepChecker):
    """``PriorMultiStepChecker`` whose steps are checked by ``TrainBnSweepChecker`` s."""

    def check(self, raise_on_failure=True):
        with _steps_use(FP, "SeededSweepChecker", TrainBnSweepChecker):
            return super().check(raise_on_failure)
