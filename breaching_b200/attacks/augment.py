"""Candidate augmentations for the engine (SURVEY section 8 f-4): the reference's ``cfg.attack.augmentations`` block
(``attacks/auxiliaries/augmentations.py``, wired in at ``optimization_based_attack.py:42-48,149-153``) translated into the linear view
pipeline of ``csrc/augment.cu``.

Supported, in config order: ``discrete_shift`` (``Jitter``), ``flip`` (``Flip``), ``colorjitter`` (``ColorJitter``; constants drawn
once per attacker like the module's ``shuffled`` flag) and ``continuous_shift`` (``RandomTransform``: bilinear, ``align=True``,
``padding`` ``circular`` / ``zeros``; must come after the shift / flip steps).  The shape-changing or non-linear ones (``zoom``,
``focus``, ``centerzoom``, ``median``, ``antialias``) raise ``NotImplementedError``.
"""
from dataclasses import dataclass, field
from typing import List, Optional, Tuple

import torch

from ..config import cfg_get

SHIFT, FLIP = 1, 2
_UNSUPPORTED = ("zoom", "focus", "centerzoom", "median", "antialias")


@dataclass
class AugmentationPlan:
    steps: List[Tuple[int, float]] = field(default_factory=list)   # (kind, lim | p) in config order
    continuous_shift: Optional[float] = None                        # RandomTransform.shift (pixels) or None
    circular: bool = False
    colour_scale: Optional[torch.Tensor] = None                     # [N, C]: composite of the colorjitter steps, out = in * scale + shift
    colour_shift: Optional[torch.Tensor] = None
    differentiable: bool = False
    seed: int = 0


def build_plan(cfg_attack, batch, channels, setup):
    """``None`` when no augmentations are configured."""
    aug = cfg_get(cfg_attack, "augmentations")
    if aug is None or len(list(aug.keys())) == 0:
        return None
    plan = AugmentationPlan(differentiable=bool(cfg_get(cfg_attack, "differentiable_augmentations", False)))
    scale = torch.ones(batch, channels, device=setup["device"])
    shift = torch.zeros(batch, channels, device=setup["device"])
    any_colour = False
    for key in aug.keys():
        opts = dict(aug[key]) if aug[key] is not None else {}
        if key == "discrete_shift":                        # Jitter(lim=32)
            if plan.continuous_shift is not None:
                raise NotImplementedError("discrete_shift after continuous_shift is not implemented by the engine")
            plan.steps.append((SHIFT, float(opts.get("lim", 32))))
        elif key == "flip":                                # Flip(p=0.5)
            if plan.continuous_shift is not None:
                raise NotImplementedError("flip after continuous_shift is not implemented by the engine")
            plan.steps.append((FLIP, float(opts.get("p", 0.5))))
        elif key == "colorjitter":                         # ColorJitter(mean=0.0, std=1.0): (img - mean) / std, drawn once (:77-83)
            if channels != 3:
                raise ValueError("colorjitter draws constants for 3 colour channels")
            mean_p, std_p = float(opts.get("mean", 0.0)), float(opts.get("std", 1.0))
            m = (torch.rand((batch, 3, 1, 1), **setup) - 0.5) * 2 * mean_p
            sd = ((torch.rand((batch, 3, 1, 1), **setup) - 0.5) * 2 * std_p).exp()
            m, sd = m.view(batch, 3), sd.view(batch, 3)
            scale, shift = scale / sd, (shift - m) / sd
            any_colour = True
        elif key == "continuous_shift":                    # RandomTransform(shift=8, padding="reflection", ...)
            if plan.continuous_shift is not None:
                raise NotImplementedError("two continuous_shift steps are not implemented by the engine")
            if opts.get("fliplr", False) or opts.get("flipud", False) or opts.get("mode", "bilinear") != "bilinear":
                raise NotImplementedError("continuous_shift: only bilinear sampling without grid flips is implemented")
            padding = opts.get("padding", "reflection")
            if padding not in ("circular", "zeros"):
                raise NotImplementedError(f"continuous_shift padding {padding} is not implemented by the engine (circular / zeros)")
            plan.continuous_shift, plan.circular = float(opts.get("shift", 8)), padding == "circular"
        elif key in _UNSUPPORTED:
            raise NotImplementedError(f"augmentation {key} is not implemented by the engine")
        else:
            raise KeyError(key)
    if len(plan.steps) > 4:
        raise NotImplementedError("at most four shift / flip steps")
    if any_colour:
        plan.colour_scale, plan.colour_shift = scale, shift
    plan.seed = int(torch.randint(0, 2 ** 31 - 1, (1,)).item())
    return plan
