"""Candidate augmentations for the engine (SURVEY section 8 f-4): the reference's ``cfg.attack.augmentations`` block
(``attacks/auxiliaries/augmentations.py``, wired in at ``optimization_based_attack.py:42-48,149-162``) translated into the linear view
pipeline of ``csrc/augment.cu``.

Supported, in config order: ``discrete_shift`` (``Jitter``), ``flip`` (``Flip``), ``colorjitter`` (``ColorJitter``; constants drawn
once per attacker like the module's ``shuffled`` flag) and ``continuous_shift`` (``RandomTransform``: ``align=True`` as the module forces,
``mode`` bilinear / nearest / bicubic, ``padding`` reflection (the module's default) / border / zeros / circular, ``fliplr`` /
``flipud`` grid flips drawn per image), and the shape-changing ``zoom`` (``Zoom``),
``centerzoom`` (``CenterZoom``), ``focus`` (``Focus``, its window corner drawn on the device every evaluation) and ``antialias``
(``AntiAlias``).  A config with only the first four kinds is one pipeline of shape-keeping steps (``AugmentationPlan.steps`` and the
colour / continuous-shift fields).  With any of the others the view is an ordered list of ``Stage`` s: each maximal run of the
shape-keeping kinds is one ``PIXEL`` stage, each zoom / centerzoom / focus a ``RESAMPLE`` stage and each antialias a ``BLUR`` stage.
The device applies a stage's continuous shift after its shift / flip steps, so a ``discrete_shift`` or ``flip`` after a
``continuous_shift`` opens a new ``PIXEL`` stage; a config of the shape-keeping kinds in such an order is a list of ``PIXEL`` stages.
The model then runs on the view's shape (``view_shape``), which may differ from the candidate's; the reference's objective and every
regulariser see the view (``:161-162``), and the gradient is pulled back onto the candidate.  A stage that changes the shape needs
``differentiable_augmentations: True`` (the reference's non-differentiable mode would replace the candidate by its view and shrink or
grow it every iteration); shape-keeping stages (antialias of odd width at stride 1) also run in the non-differentiable mode.
``median`` (a non-linear order statistic) raises ``NotImplementedError``.
"""
from dataclasses import dataclass, field, replace
from typing import List, Optional, Tuple

import torch

from ..config import cfg_get

SHIFT, FLIP = 1, 2
PIXEL, RESAMPLE, BLUR = "pixel", "resample", "blur"
_PIXEL_KINDS = ("discrete_shift", "flip", "colorjitter", "continuous_shift")
_GRID_KINDS = ("discrete_shift", "flip", "continuous_shift")       # what a continuous shift must come after within one stage
CS_MODES = {"bilinear": 0, "nearest": 1, "bicubic": 2}              # grid_sample mode / padding_mode -> bre_augment_view_ex codes
CS_PADDINGS = {"zeros": 0, "border": 1, "reflection": 2}
_VIEW_KINDS = ("zoom", "centerzoom", "focus", "antialias")
_UNSUPPORTED = ("median",)
MAX_STAGES = 8


@dataclass
class Stage:
    kind: str                                                        # PIXEL / RESAMPLE / BLUR
    in_hw: Tuple[int, int]
    out_hw: Tuple[int, int]
    steps: List[Tuple[int, float]] = field(default_factory=list)     # PIXEL: as AugmentationPlan
    continuous_shift: Optional[float] = None
    circular: bool = False
    colour_scale: Optional[torch.Tensor] = None
    colour_shift: Optional[torch.Tensor] = None
    cs_mode: str = "bilinear"                                        # PIXEL: continuous_shift sampling, as AugmentationPlan
    cs_padding: str = "zeros"
    fliplr: bool = False
    flipud: bool = False
    corner: Tuple[int, int] = (0, 0)                                 # RESAMPLE: window corner (row, column) and size
    window: Tuple[int, int] = (0, 0)
    focus_std: Optional[float] = None                                # RESAMPLE (focus): corner drawn per evaluation
    width: int = 0                                                   # BLUR
    stride: int = 1


@dataclass
class AugmentationPlan:
    steps: List[Tuple[int, float]] = field(default_factory=list)   # (kind, lim | p) in config order
    continuous_shift: Optional[float] = None                        # RandomTransform.shift (pixels) or None
    circular: bool = False
    colour_scale: Optional[torch.Tensor] = None                     # [N, C]: composite of the colorjitter steps, out = in * scale + shift
    colour_shift: Optional[torch.Tensor] = None
    differentiable: bool = False
    seed: int = 0
    stages: List[Stage] = field(default_factory=list)               # empty: the fields above are the whole (shape-keeping) view
    candidate_shape: Optional[Tuple[int, int, int, int]] = None     # with stages: [N, C, H, W] of the candidate
    cs_mode: str = "bilinear"                                       # grid_sample mode of the continuous shift
    cs_padding: str = "zeros"                                       # its padding_mode ("circular": zeros after the wrap, circular=True)
    fliplr: bool = False                                            # RandomTransform's grid flips
    flipud: bool = False


def _opts(aug, key):
    return dict(aug[key]) if aug[key] is not None else {}


def _geometry(key, opts, C, H, W):
    """Draw-free shape map of one shape-changing key: (Stage without PIXEL fields)."""
    if key == "zoom":                                   # Zoom(out_size=224) :34-40
        out = int(opts.get("out_size", 224))
        return Stage(RESAMPLE, (H, W), (out, out), corner=(0, 0), window=(H, W))
    if key == "centerzoom":                             # CenterZoom(initial_fov=32, out_size=224) :43-55
        fov, out = int(opts.get("initial_fov", 32)), int(opts.get("out_size", 224))
        if fov > H or fov > W or fov < 1:
            raise ValueError(f"centerzoom: a {fov} x {fov} field of view does not fit a {H} x {W} input")
        return Stage(RESAMPLE, (H, W), (out, out), corner=((H - fov) // 2, (W - fov) // 2), window=(fov, fov))
    if key == "focus":                                  # Focus(size=224, std=1.0) :20-31
        size, std = int(opts.get("size", 224)), float(opts.get("std", 1.0))
        if size > H or size > W or size < 1:
            raise ValueError(f"focus: a {size} x {size} window does not fit a {H} x {W} input")
        return Stage(RESAMPLE, (H, W), (size, size), window=(size, size), focus_std=std)
    if key == "antialias":                              # AntiAlias(channels=3, width=5, stride=1) :198-226
        channels, width, stride = int(opts.get("channels", 3)), opts.get("width", 5), int(opts.get("stride", 1))
        if channels != C:
            raise ValueError(f"antialias: a filter for {channels} channels cannot filter {C}")
        if int(width) != width or not 1 <= int(width) <= 7:
            raise ValueError(f"antialias: width {width} is not in the filter bank (1..7)")
        width = int(width)
        if stride < 1:
            raise ValueError("antialias: stride must be positive")
        pad = width // 2
        out = ((H + 2 * pad - width) // stride + 1, (W + 2 * pad - width) // stride + 1)
        if out[0] < 1 or out[1] < 1:
            raise ValueError(f"antialias: width {width} leaves no output on a {H} x {W} input")
        return Stage(BLUR, (H, W), out, width=width, stride=stride)
    raise KeyError(key)


def _stage_starts(aug):
    """The keys that open a PIXEL stage: a shape-keeping kind at the start or after a shape-changing one, and a discrete_shift, flip or
    continuous_shift after a continuous_shift of the same stage."""
    starts, in_run, shifted = set(), False, False
    for key in aug.keys():
        if key in _VIEW_KINDS:
            in_run = False
        elif key in _PIXEL_KINDS:
            if not in_run or (shifted and key in _GRID_KINDS):
                starts.add(key)
                in_run, shifted = True, False
            shifted = shifted or key == "continuous_shift"
    return starts


def _needs_stages(aug):
    return any(k in _VIEW_KINDS for k in aug.keys()) or len(_stage_starts(aug)) > 1


def has_view_stages(cfg_attack):
    """Does the config contain a shape-changing kind (zoom, centerzoom, focus, antialias)?  Draws nothing."""
    aug = cfg_get(cfg_attack, "augmentations")
    return aug is not None and any(k in _VIEW_KINDS for k in aug.keys())


def view_shape(cfg_attack, candidate_shape):
    """The shape [N, C, H, W] the model sees for a candidate of ``candidate_shape`` (the candidate's own shape without
    shape-changing kinds).  Consumes no random numbers; raises the refusals of ``build_plan`` that depend on shapes."""
    N, C, H, W = (int(s) for s in candidate_shape)
    if not has_view_stages(cfg_attack):
        return (N, C, H, W)
    aug = cfg_get(cfg_attack, "augmentations")
    stages = []
    for key in aug.keys():
        if key in _VIEW_KINDS:
            stages.append(_geometry(key, _opts(aug, key), C, H, W))
            H, W = stages[-1].out_hw
    _check_differentiable(cfg_attack, stages)
    return (N, C, H, W)


def _check_differentiable(cfg_attack, stages):
    if any(st.in_hw != st.out_hw for st in stages) and not bool(cfg_get(cfg_attack, "differentiable_augmentations", False)):
        raise ValueError("shape-changing augmentations (zoom, centerzoom, focus, antialias) need differentiable_augmentations: True: "
                         "the non-differentiable mode replaces the candidate by its view, which changes its shape every iteration")


def build_plan(cfg_attack, batch, channels, setup, spatial=None):
    """``None`` when no augmentations are configured.  ``spatial`` = (H, W) of the candidate, needed when the config contains a
    shape-changing kind.  Random numbers are drawn in config order (the colorjitter constants), then the Philox seed."""
    aug = cfg_get(cfg_attack, "augmentations")
    if aug is None or len(list(aug.keys())) == 0:
        return None
    plan = AugmentationPlan(differentiable=bool(cfg_get(cfg_attack, "differentiable_augmentations", False)))
    staged = _needs_stages(aug)
    starts = _stage_starts(aug)
    if staged:
        if spatial is None:
            raise ValueError("shape-changing augmentations and shift / flip steps after a continuous_shift need the candidate's spatial shape")
        view_shape(cfg_attack, (batch, channels, *spatial))       # shape refusals before anything is drawn
        H, W = int(spatial[0]), int(spatial[1])
    scale = torch.ones(batch, channels, device=setup["device"])
    shift = torch.zeros(batch, channels, device=setup["device"])
    any_colour = False
    run = None                                          # the PIXEL stage being filled (staged plans)

    def close_run():
        nonlocal run
        if run is not None:
            if len(run.steps) > 4:
                raise NotImplementedError("at most four shift / flip steps")
            plan.stages.append(run)
        run = None

    for key in aug.keys():
        opts = _opts(aug, key)
        if key in _PIXEL_KINDS and staged and (run is None or key in starts):
            close_run()
            run = Stage(PIXEL, (H, W), (H, W))
        target = run if staged and key in _PIXEL_KINDS else plan
        if key == "discrete_shift":                        # Jitter(lim=32)
            target.steps.append((SHIFT, float(opts.get("lim", 32))))
        elif key == "flip":                                # Flip(p=0.5)
            target.steps.append((FLIP, float(opts.get("p", 0.5))))
        elif key == "colorjitter":                         # ColorJitter(mean=0.0, std=1.0): (img - mean) / std, drawn once (:77-83)
            if channels != 3:
                raise ValueError("colorjitter draws constants for 3 colour channels")
            mean_p, std_p = float(opts.get("mean", 0.0)), float(opts.get("std", 1.0))
            m = (torch.rand((batch, 3, 1, 1), **setup) - 0.5) * 2 * mean_p
            sd = ((torch.rand((batch, 3, 1, 1), **setup) - 0.5) * 2 * std_p).exp()
            m, sd = m.view(batch, 3), sd.view(batch, 3)
            if staged:
                s0 = run.colour_scale if run.colour_scale is not None else torch.ones_like(scale)
                h0 = run.colour_shift if run.colour_shift is not None else torch.zeros_like(shift)
                run.colour_scale, run.colour_shift = s0 / sd, (h0 - m) / sd
            else:
                scale, shift = scale / sd, (shift - m) / sd
                any_colour = True
        elif key == "continuous_shift":                    # RandomTransform(shift=8, fliplr=False, flipud=False, mode="bilinear", padding="reflection")
            mode, padding = opts.get("mode", "bilinear"), opts.get("padding", "reflection")
            if mode not in CS_MODES:                       # the errors of F.grid_sample
                raise ValueError(f"continuous_shift: mode must be one of bilinear, nearest, bicubic, got {mode!r}")
            if padding not in (*CS_PADDINGS, "circular"):
                raise ValueError(f"continuous_shift: padding must be one of zeros, border, reflection, circular, got {padding!r}")
            target.continuous_shift, target.circular = float(opts.get("shift", 8)), padding == "circular"
            target.cs_mode, target.cs_padding = mode, "zeros" if padding == "circular" else padding
            target.fliplr, target.flipud = bool(opts.get("fliplr", False)), bool(opts.get("flipud", False))
        elif key in _VIEW_KINDS:
            close_run()
            st = _geometry(key, opts, channels, H, W)
            plan.stages.append(st)
            H, W = st.out_hw
        elif key in _UNSUPPORTED:
            raise NotImplementedError(f"augmentation {key} is not implemented by the engine")
        else:
            raise KeyError(key)
    close_run()
    if len(plan.steps) > 4:
        raise NotImplementedError("at most four shift / flip steps")
    if len(plan.stages) > MAX_STAGES:
        raise NotImplementedError(f"at most {MAX_STAGES} augmentation stages (a run of shift / flip / colour steps counts once)")
    if any_colour:
        plan.colour_scale, plan.colour_shift = scale, shift
    if staged:
        plan.candidate_shape = (int(batch), int(channels), int(spatial[0]), int(spatial[1]))
    plan.seed = int(torch.randint(0, 2 ** 31 - 1, (1,)).item())
    return plan


def with_spatial(plan, cfg_attack, spatial):
    """``plan`` (with stages) for a candidate of another spatial shape (H, W): the same colour constants and seed, the stage geometry
    of the new shape.  Draws nothing; raises the shape refusals of ``view_shape``."""
    N, C = plan.candidate_shape[:2]
    H, W = int(spatial[0]), int(spatial[1])
    view_shape(cfg_attack, (N, C, H, W))
    aug = cfg_get(cfg_attack, "augmentations")
    runs = iter([st for st in plan.stages if st.kind == PIXEL])
    starts = _stage_starts(aug)
    stages = []
    for key in aug.keys():
        if key in _VIEW_KINDS:
            stages.append(_geometry(key, _opts(aug, key), C, H, W))
            H, W = stages[-1].out_hw
        elif key in starts:                                # the next PIXEL stage, at this point's shape
            stages.append(replace(next(runs), in_hw=(H, W), out_hw=(H, W)))
    return replace(plan, stages=stages, candidate_shape=(N, C, int(spatial[0]), int(spatial[1])))
