"""``MultiScaleOptimizationAttacker`` on the sm_90a engine (SURVEY section 8 f-4).

Reference: ``attacks/multiscale_optimization_attack.py:18-122`` -- the candidate is optimised on a pyramid of resolutions; every
stage starts from the bilinearly up-sampled result of the previous one (optionally pasted into the centre of a fresh
initialisation, ``resize: focus``), runs a full optimisation with a fresh optimiser / schedule, and the last stage's best
candidate, resized to the data shape, is the trial's result.  (The reference class cannot be called as shipped: its ``_run_trial``
signature no longer matches the caller in ``optimization_based_attack.py:72``, SURVEY section 8f; the stage logic below follows
its body.)

On the engine one stage = one trial of a layer program compiled for that resolution (the model must accept variable input sizes,
e.g. ResNets with adaptive pooling -- otherwise the compiler refuses, as the reference's forward pass would); the resizes run in
``bre_resize_bilinear`` (``F.interpolate(mode="bilinear", align_corners=False)`` semantics).  Each stage's program is compiled at
the view shape of that stage's candidate: with ``augmentations: {zoom: {out_size: H}}`` every stage runs the model at H.
"""
import logging

import torch

from ..config import cfg_get
from ..engine import resize_bilinear
from . import host
from .optimization_attack import OptimizationBasedAttacker

log = logging.getLogger(__name__)


def scale_pyramid(kind, num_stages, full):
    """multiscale_optimization_attack.py:31-41."""
    if kind == "linear":
        increment = full // num_stages
        return list(range(increment, full + 1, increment))
    if kind == "log":
        return [int(round(full / (2 ** i))) for i in range(num_stages - 1, -1, -1)]
    if kind == "trivial":
        return [full] * num_stages
    raise ValueError(f"Invalid scale pyramid {kind}.")


class MultiScaleOptimizationAttacker(OptimizationBasedAttacker):
    def _get_engine(self, rec_models, shared_data, labels, index=0, cfg=None, data_shape=None, primary=True, **kw):
        if primary and index == 0:
            self._stage_context = (rec_models, shared_data, labels)
            for eng in getattr(self, "_stage_engines", {}).values():
                eng.close()
            self._stage_engines = {}
        return super()._get_engine(rec_models, shared_data, labels, index, cfg, data_shape, primary, **kw)

    def _stage_engine(self, scale):
        C, H, W = self.data_shape
        if scale == H:
            return self._engine
        if scale not in self._stage_engines:
            rec_models, shared_data, labels = self._stage_context
            if len(rec_models) != 1:
                raise NotImplementedError("multi-scale attacks with several model queries are not implemented by the engine")
            self._stage_engines[scale] = self._get_engine(rec_models, shared_data, labels, data_shape=(C, scale, scale), primary=False)
        return self._stage_engines[scale]

    def _run_trial(self, engine, candidate, stats, trial, dryrun=False):
        C, H, W = self.data_shape
        if H != W:
            raise ValueError("multi-scale attacks need square images")  # reference :27 asserts
        stages = int(self.cfg.num_stages)
        pyramid = scale_pyramid(cfg_get(self.cfg, "scale_pyramid", "linear"), stages, H)
        n = candidate.shape[0]
        # lowest-scale initialisation, then the full-size placeholder the reference also draws (:46-47)
        current = host.initialize_data(self.cfg.init, [n, C, pyramid[0], pyramid[0]], self.dm, self.ds, self.setup)
        best = host.initialize_data(self.cfg.init, [n, C, H, W], self.dm, self.ds, self.setup)
        for stage, scale in enumerate(pyramid):
            log.info(f"| Now solving stage {stage + 1}/{stages} with scale {scale}:")
            if cfg_get(self.cfg, "resize", "upsampling") == "focus":      # :54-60: paste into the centre of a fresh init
                p = scale // 2
                background = host.initialize_data(self.cfg.init, [n, C, scale, scale], self.dm, self.ds, self.setup)
                cx = (scale - p) // 2
                background[:, :, cx:cx + p, cx:cx + p] = resize_bilinear(current, p)
                current = background
            else:
                current = resize_bilinear(current, scale)
            try:
                stage_engine = self._stage_engine(scale)
            except ValueError as err:    # e.g. a focus window larger than this stage's candidate
                raise ValueError(f"stage {stage + 1}/{stages} (scale {scale}): {err}") from err
            stage_best = super()._run_trial(stage_engine, current, stats, trial, dryrun)
            current = stage_best
            best = resize_bilinear(stage_best, H)                           # :66
            if dryrun:
                break
        return best.detach()
