"""ctypes binding of ``libbreaching_b200.so`` (C ABI in ``include/breaching_b200.h``).

PyTorch is used here only as plumbing: it owns the tensors whose ``data_ptr()`` is handed to the library.
There is no fallback: if the shared library is missing or a call fails, an exception is raised.
"""
import ctypes
import os

import torch

from . import compiler as C

_LIB = None
LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib", "libbreaching_b200.so")


class EngineError(RuntimeError):
    pass


class TensorDesc(ctypes.Structure):
    _fields_ = [("N", ctypes.c_int32), ("C", ctypes.c_int32), ("H", ctypes.c_int32), ("W", ctypes.c_int32)]


class ParamDesc(ctypes.Structure):
    _fields_ = [("numel", ctypes.c_int64), ("perm", ctypes.c_int32), ("d0", ctypes.c_int32), ("d1", ctypes.c_int32),
                ("d2", ctypes.c_int32)]


class OpDesc(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in
                ("kind", "tin", "tout", "res", "R", "S", "stride", "pad", "w", "b", "has_bn", "relu", "gamma", "beta",
                 "bn_buffer")] + [("eps", ctypes.c_float), ("acc_in", ctypes.c_int32), ("acc_res", ctypes.c_int32),
                                  ("bn_train", ctypes.c_int32)]


class AugStage(ctypes.Structure):   # bre_aug_stage
    _fields_ = [("kind", ctypes.c_int32), ("n_steps", ctypes.c_int32), ("kinds", ctypes.c_int32 * 4), ("params", ctypes.c_float * 4),
                ("cs_enabled", ctypes.c_int32), ("cs_circular", ctypes.c_int32), ("cs_shift", ctypes.c_float),
                ("cj_scale", ctypes.c_void_p), ("cj_shift", ctypes.c_void_p)] + \
               [(n, ctypes.c_int32) for n in ("y0", "x0", "wh", "ww", "Ho", "Wo", "focus")] + \
               [("focus_std", ctypes.c_float), ("width", ctypes.c_int32), ("stride", ctypes.c_int32)]


class AugStageEx(ctypes.Structure):   # bre_aug_stage_ex
    _fields_ = [("stage", AugStage)] + [(n, ctypes.c_int32) for n in ("cs_mode", "cs_padding", "cs_fliplr", "cs_flipud")]


class StepScalars(ctypes.Structure):   # bre_step_scalars
    _fields_ = [(n, ctypes.c_double) for n in ("match", "task_loss", "tv", "norm", "di", "feat", "fmin")] + \
               [(n, ctypes.c_int32) for n in ("it", "recorded", "stopped", "trial")] + \
               [("grad_norm_sq", ctypes.c_double), ("last_objective", ctypes.c_double)]


class LbfgsConsts(ctypes.Structure):   # bre_lbfgs_consts
    _fields_ = [(n, ctypes.c_int32) for n in ("max_iter", "max_eval", "history", "reserved")] + \
               [(n, ctypes.c_double) for n in ("tol_grad", "tol_change", "curvature_min")]


class LbfgsScalars(ctypes.Structure):   # bre_lbfgs_scalars
    _fields_ = [(n, ctypes.c_double) for n in ("h_diag", "t", "loss", "prev_loss", "first_loss", "gtd", "d_max", "g_max", "g_abs_sum", "ys")] + \
               [("first_terms", ctypes.c_double * 6)] + \
               [(n, ctypes.c_int32) for n in ("first", "count", "total_iters", "inner", "evals", "func_evals", "brk", "converged", "pushed",
                                              "reserved")]


def lbfgs_consts():
    """torch.optim.LBFGS's defaults as the C struct (their one definition is breaching_b200/attacks/lbfgs.py)."""
    from .attacks import lbfgs

    return LbfgsConsts(lbfgs.MAX_ITER, lbfgs.MAX_EVAL, lbfgs.HISTORY, 0, lbfgs.TOL_GRAD, lbfgs.TOL_CHANGE, lbfgs.CURVATURE_MIN)


class AttackCfg(ctypes.Structure):
    _fields_ = [
        ("objective", ctypes.c_int32),
        ("obj_scale", ctypes.c_float), ("task_regularization", ctypes.c_float), ("tag_scale", ctypes.c_float),
        ("mask_value", ctypes.c_float), ("angular_fudge", ctypes.c_float),
        ("optimizer", ctypes.c_int32),
        ("beta1", ctypes.c_float), ("beta2", ctypes.c_float), ("adam_eps", ctypes.c_float),
        ("weight_decay", ctypes.c_float), ("momentum", ctypes.c_float),
        ("nesterov", ctypes.c_int32), ("signed_mode", ctypes.c_int32), ("boxed", ctypes.c_int32),
        ("max_iterations", ctypes.c_int32),
        ("langevin_noise", ctypes.c_float), ("grad_clip", ctypes.c_float),
        ("noise_seed", ctypes.c_uint64),
        ("tv_scale", ctypes.c_float), ("tv_inner_exp", ctypes.c_float), ("tv_outer_exp", ctypes.c_float),
        ("tv_eps", ctypes.c_float), ("tv_double_opponents", ctypes.c_int32),
        ("norm_scale", ctypes.c_float), ("norm_p", ctypes.c_float),
        ("di_scale", ctypes.c_float), ("di_first_bn_multiplier", ctypes.c_float),
        ("feat_scale", ctypes.c_float),
        ("orthogonality", ctypes.c_int32),
        ("objective_excludes_task", ctypes.c_int32),
    ]


OBJECTIVES = {  # reference objectives.py:496-506
    "euclidean": 0, "cosine-similarity": 1, "l1": 2, "tag-euclidean": 3, "angular": 4,
    "fast-cosine-similarity": 5, "masked-cosine-similarity": 6,
}
# Pearlmutter* (objectives.py:279-365, 468-493) approximate d/dx <grad_W L, v> -- v = d(objective)/dG, *without* the scale --
# by finite differences of grad_x L along W + eps v ("forward" / "backward" / "central"); the engine's tangent sweeps compute
# that directional derivative exactly, i.e. the eps -> 0 limit of all three, at no extra cost.  (The reference versions are
# broken under torch >= 2: `candidate.grad +=` on a None gradient, SURVEY section 8c.)
PEARLMUTTER = {"pearlmutter-loss": "euclidean", "pearlmutter-cosine": "cosine-similarity"}
OPTIMIZERS = {  # reference common.py:6-17 -> (kind, beta1, beta2, eps, weight_decay, momentum, nesterov)
    "adam": (0, 0.9, 0.999, 1e-8, 0.0, 0.0, 0),
    "adam-safe": (0, 0.5, 0.99, 1e-4, 0.0, 0.0, 0),
    "bert-adam": (1, 0.9, 0.999, 1e-6, 0.01, 0.0, 0),
    "momgd": (2, 0.0, 0.0, 0.0, 0.0, 0.9, 1),
    "gd": (2, 0.0, 0.0, 0.0, 0.0, 0.0, 0),
}

EXPORTS = [
    "bre_engine_create", "bre_engine_destroy", "bre_engine_load_model", "bre_engine_load_targets",
    "bre_engine_load_feature_targets", "bre_engine_set_local_steps", "bre_engine_begin_trial", "bre_engine_run", "bre_engine_run_timed", "bre_engine_sync",
    "bre_engine_status", "bre_engine_read_history", "bre_engine_get_best", "bre_engine_get_candidate",
    "bre_engine_score", "bre_engine_objective_and_gradient", "bre_engine_last_terms", "bre_engine_debug_param",
    "bre_engine_debug_step_param", "bre_engine_debug_tensor", "bre_engine_debug_op", "bre_engine_launches_per_iteration", "bre_engine_set_option", "bre_match_reduce",
    "bre_total_variation", "bre_conv_gemm", "bre_last_error", "bre_version",
    "bre_engine_load_soft_labels", "bre_engine_label_gradient", "bre_engine_set_labels",
    "bre_token_layernorm", "bre_token_attention", "bre_token_match", "bre_token_attention_ex", "bre_token_attention_plan",
    "bre_engine_load_constant",
    "bre_engine_param_gradients", "bre_engine_bn_batch_stats", "bre_engine_forward", "bre_image_mse",
    "bre_engine_begin_joint_trial", "bre_engine_get_joint_labels", "bre_resize_bilinear",
    "bre_engine_set_augmentations", "bre_engine_last_augmentation", "bre_augment_view",
    "bre_engine_set_augmentation_stages", "bre_engine_augmentation_draws", "bre_augment_resample", "bre_augment_blur",
    "bre_engine_set_augmentations_ex", "bre_engine_set_augmentation_stages_ex", "bre_augment_view_ex", "bre_engine_augmentation_flips",
    "bre_engine_set_trial_index", "bre_engine_debug_step_state", "bre_optimizer_step", "bre_langevin_noise",
    "bre_debug_last_gemm_plan", "bre_gemm_plan", "bre_debug_row_plan", "bre_row_op",
    "bre_engine_begin_lbfgs_trial", "bre_engine_lbfgs_counters", "bre_lbfgs_direction",
]


def load_library(path=None):
    """Load the shared library (no compute is triggered; works without a GPU)."""
    global _LIB
    if _LIB is not None and path is None:
        return _LIB
    path = path or LIB_PATH
    if not os.path.exists(path):
        raise EngineError(
            f"{path} not found: build it with `python -m breaching_b200.build` (there is no CPU/eager fallback)"
        )
    lib = ctypes.CDLL(path)
    lib.bre_last_error.restype = ctypes.c_char_p
    lib.bre_version.restype = ctypes.c_char_p
    lib.bre_engine_destroy.restype = None
    vp, i32, i64, f32 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_float
    P = ctypes.POINTER
    lib.bre_engine_create.argtypes = [P(TensorDesc), i32, P(OpDesc), i32, P(ParamDesc), i32, i32, P(AttackCfg), i32, P(vp)]
    lib.bre_engine_destroy.argtypes = [vp]
    lib.bre_engine_load_model.argtypes = [vp, P(vp), i32, P(vp), P(vp), i32]
    lib.bre_engine_load_targets.argtypes = [vp, P(vp), i32, vp, vp, i32, vp, vp, i32]
    lib.bre_engine_load_feature_targets.argtypes = [vp, vp, i64]
    lib.bre_engine_set_local_steps.argtypes = [vp, i32, i32, f32, vp]
    lib.bre_engine_load_soft_labels.argtypes = [vp, vp, i64]
    lib.bre_engine_label_gradient.argtypes = [vp, vp]
    lib.bre_engine_set_labels.argtypes = [vp, vp, i32]
    lib.bre_engine_begin_trial.argtypes = [vp, vp, vp, i32]
    lib.bre_engine_run.argtypes = [vp, i32]
    lib.bre_engine_sync.argtypes = [vp]
    lib.bre_engine_run_timed.argtypes = [vp, i32, P(ctypes.c_float)]
    lib.bre_engine_status.argtypes = [vp, P(i32), P(i32), P(ctypes.c_double), P(ctypes.c_double)]
    lib.bre_engine_read_history.argtypes = [vp, vp, i32]
    lib.bre_engine_get_best.argtypes = [vp, vp]
    lib.bre_engine_get_candidate.argtypes = [vp, vp]
    lib.bre_engine_score.argtypes = [vp, vp, i32, P(ctypes.c_double)]
    lib.bre_engine_objective_and_gradient.argtypes = [vp, vp, P(ctypes.c_double), vp]
    lib.bre_engine_last_terms.argtypes = [vp, P(ctypes.c_double)]
    lib.bre_engine_debug_param.argtypes = [vp, i32, i32, vp]
    lib.bre_engine_debug_step_param.argtypes = [vp, i32, i32, i32, vp]
    lib.bre_engine_debug_tensor.argtypes = [vp, i32, i32, vp]
    lib.bre_engine_debug_op.argtypes = [vp, i32, P(i32)]
    lib.bre_engine_launches_per_iteration.argtypes = [vp, P(i32)]
    lib.bre_engine_set_option.argtypes = [vp, ctypes.c_char_p, i64]
    lib.bre_match_reduce.argtypes = [vp, vp, vp, i64, f32, P(ctypes.c_double), vp]
    lib.bre_total_variation.argtypes = [vp, vp, i32, i32, i32, f32, f32, f32, f32, i32, i32, P(ctypes.c_double), vp]
    lib.bre_conv_gemm.argtypes = [i32, i32, vp, vp, vp, vp, vp] + [i32] * 9 + [vp]
    lib.bre_token_layernorm.argtypes = [i32, vp, vp, vp, vp, vp, vp, vp, vp, f32, i32, i32, vp, vp, vp, vp, i32, vp]
    lib.bre_token_attention.argtypes = [i32, vp, vp, vp, vp, i32, i32, i32, i32, vp, vp, vp, i32, vp]
    lib.bre_token_attention_ex.argtypes = [i32, vp, vp, vp, vp, i32, i32, i32, i32, vp, vp, vp, i32, vp, i32]
    lib.bre_token_attention_plan.argtypes = [i32, i32, i32, P(i32)]
    lib.bre_engine_load_constant.argtypes = [vp, i32, vp, i64]
    lib.bre_token_match.argtypes = [vp, vp, vp, i32, i32, i32, vp, vp]
    lib.bre_engine_begin_joint_trial.argtypes = [vp, vp, vp, i64, vp, i32]
    lib.bre_engine_get_joint_labels.argtypes = [vp, i32, vp]
    lib.bre_engine_param_gradients.argtypes = [vp, vp, vp, i32, P(vp), i32, P(ctypes.c_double)]
    lib.bre_engine_bn_batch_stats.argtypes = [vp, i32, vp, vp]
    lib.bre_engine_forward.argtypes = [vp, vp, vp]
    lib.bre_engine_set_augmentations.argtypes = [vp, i32, P(i32), P(f32), i32, f32, i32, vp, vp, i32, ctypes.c_uint64]
    lib.bre_engine_last_augmentation.argtypes = [vp, P(i32), P(i32), P(f32), P(f32)]
    lib.bre_augment_view.argtypes = [vp, vp, i32, i32, i32, i32, i32, P(i32), P(i32), P(i32), f32, i32, P(f32), P(f32), vp, vp, i32, vp, vp]
    lib.bre_engine_set_augmentation_stages.argtypes = [vp, i32, P(AugStage), i32, i32, i32, i32, i32, ctypes.c_uint64]
    lib.bre_engine_augmentation_draws.argtypes = [vp, P(i32), P(i32), P(i32), P(f32), P(f32)]
    lib.bre_augment_resample.argtypes = [vp, vp] + [i32] * 11 + [vp]
    lib.bre_engine_set_augmentations_ex.argtypes = [vp, i32, P(i32), P(f32), i32, f32, i32, i32, i32, i32, i32, vp, vp, i32, ctypes.c_uint64]
    lib.bre_engine_set_augmentation_stages_ex.argtypes = [vp, i32, P(AugStageEx), i32, i32, i32, i32, i32, ctypes.c_uint64]
    lib.bre_augment_view_ex.argtypes = [vp, vp, i32, i32, i32, i32, i32, P(i32), P(i32), P(i32), f32, i32, i32, i32, P(f32), P(f32), P(i32), P(i32),
                                        vp, vp, i32, vp, vp]
    lib.bre_engine_augmentation_flips.argtypes = [vp, P(i32), P(i32), P(i32)]
    lib.bre_augment_blur.argtypes = [vp, vp] + [i32] * 7 + [vp]
    lib.bre_resize_bilinear.argtypes = [vp, vp, i32, i32, i32, i32, i32, i32, vp]
    lib.bre_image_mse.argtypes = [vp, vp, i32, i32, i32, vp, vp, i32, P(ctypes.c_double), vp]
    lib.bre_engine_set_trial_index.argtypes = [vp, i32]
    lib.bre_engine_debug_step_state.argtypes = [vp, i32, vp]
    lib.bre_optimizer_step.argtypes = [vp] * 7 + [i32, vp, vp, i64, i32, i32, P(AttackCfg), vp, i32, P(StepScalars), vp]
    lib.bre_langevin_noise.argtypes = [ctypes.c_uint64, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint64, i64, vp, vp]
    lib.bre_debug_last_gemm_plan.argtypes = [P(i32)]
    lib.bre_gemm_plan.argtypes = [i32] * 12 + [P(i32)]
    lib.bre_debug_row_plan.argtypes = [i32, P(i32), P(i32)]
    lib.bre_row_op.argtypes = [i32, vp, vp, vp, vp, i32, i32, i32, i32, f32, i32, vp, vp, vp, vp]
    lib.bre_engine_begin_lbfgs_trial.argtypes = [vp, vp, vp, i64, vp, i32, P(LbfgsConsts)]
    lib.bre_engine_lbfgs_counters.argtypes = [vp, P(i32)]
    lib.bre_lbfgs_direction.argtypes = [vp, vp, vp, vp, vp, vp, vp, i64, P(LbfgsConsts), vp]
    for name in EXPORTS:
        if name not in ("bre_last_error", "bre_version", "bre_engine_destroy"):
            getattr(lib, name).restype = ctypes.c_int
    _LIB = lib
    return lib


def _check(lib, rc, what):
    if rc != 0:
        raise EngineError(f"{what} failed ({rc}): {lib.bre_last_error().decode()}")


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _f32c(t, device=None):
    t = t.detach()
    if device is not None:
        t = t.to(device)
    return t.to(torch.float32).contiguous()


def make_cfg(cfg_attack, noise_seed=0):
    """Flatten the reference-style attack config into the C struct (values as the reference reads them,
    attacks/optimization_based_attack.py:29-38, :166-184; regularizers.py constructors)."""
    from .config import cfg_get

    c = AttackCfg()
    obj = cfg_attack["objective"]
    kind = obj["type"]
    if kind in PEARLMUTTER:
        impl = cfg_get(obj, "implementation", "forward")
        if impl not in ("forward", "backward", "central"):
            # "upwind" mixes one-sided differences by the sign of dL/dx reduced over the batch axis (objectives.py:440-461): it has
            # no eps -> 0 limit that a directional derivative expresses
            raise EngineError(f"{kind}: finite-difference implementation '{impl}' is not implemented by the engine")
        if cfg_get(obj, "level_gradients", False):
            raise EngineError(f"{kind}: level_gradients is not implemented by the engine")
        kind = PEARLMUTTER[kind]
        c.objective_excludes_task = 1
    if kind not in OBJECTIVES:
        raise ValueError(f"Unknown objective type {kind} given.")
    c.objective = OBJECTIVES[kind]
    c.obj_scale = float(cfg_get(obj, "scale", 1.0))
    c.task_regularization = float(cfg_get(obj, "task_regularization", 0.0) or 0.0)
    c.tag_scale = float(cfg_get(obj, "tag_scale", 0.1))
    c.mask_value = 1e-6  # objectives.py:227 hard-codes 1e-6
    c.angular_fudge = 1e-7  # objectives.py:208
    opt = cfg_attack["optim"]
    name = str(opt["optimizer"]).lower()
    if name not in OPTIMIZERS and name != "l-bfgs":
        raise ValueError(f"Invalid optimizer {opt['optimizer']} given.")
    # L-BFGS trials (Engine.begin_lbfgs_trial, or the host loop of attacks/lbfgs.py) use the step kernel only to post-process the
    # gradient; its optimiser fields are unused then
    c.optimizer, c.beta1, c.beta2, c.adam_eps, c.weight_decay, c.momentum, c.nesterov = OPTIMIZERS["gd" if name == "l-bfgs" else name]
    signed = cfg_get(opt, "signed")
    c.signed_mode = {"hard": 1, "soft": 2}.get(signed, 0) if isinstance(signed, str) else 0
    c.boxed = int(bool(cfg_get(opt, "boxed", False)))
    c.max_iterations = int(opt["max_iterations"])
    c.langevin_noise = float(cfg_get(opt, "langevin_noise", 0.0) or 0.0)
    clip = cfg_get(opt, "grad_clip")
    c.grad_clip = -1.0 if clip is None else float(clip)
    c.noise_seed = int(noise_seed) & 0xFFFFFFFFFFFFFFFF
    c.tv_eps, c.tv_inner_exp, c.tv_outer_exp, c.norm_p, c.di_first_bn_multiplier = 1e-8, 1.0, 1.0, 2.0, 10.0
    reg = cfg_get(cfg_attack, "regularization")
    if reg is not None:
        for key in reg.keys():
            r = reg[key]
            if not r["scale"] > 0:
                continue
            if key == "total_variation":
                c.tv_scale = float(r["scale"])
                c.tv_inner_exp = float(cfg_get(r, "inner_exp", 1))
                c.tv_outer_exp = float(cfg_get(r, "outer_exp", 1))
                c.tv_eps = float(cfg_get(r, "eps", 1e-8))
                c.tv_double_opponents = int(bool(cfg_get(r, "double_opponents", False)))
            elif key == "norm":
                c.norm_scale = float(r["scale"])
                c.norm_p = float(cfg_get(r, "pnorm", 2.0))
            elif key == "deep_inversion":
                c.di_scale = float(r["scale"])
                c.di_first_bn_multiplier = float(cfg_get(r, "first_bn_multiplier", 10))
            elif key == "features":
                c.feat_scale = float(r["scale"])
            elif key == "orthogonality":
                c.orthogonality = 1  # regularizers.py:169-178 never multiplies by its scale
            else:
                raise KeyError(key)
    return c


def _check_prior_layers(prog, c):
    """The reference's DeepInversion prior weights the first *registered* BatchNorm2d by ``first_bn_multiplier`` and its features
    prior reads the input of the last *registered* Linear (regularizers.py); the engine applies them to the first BN op and the
    last Linear op that run.  Where the two orders pick different layers the engine would optimise another objective than the
    reference, so the prior is refused, naming both layers."""
    ops = prog.ops
    bn = [i for i, op in enumerate(ops) if op.kind == C.OP_BNACT and op.has_bn]
    lin = [i for i, op in enumerate(ops) if op.kind == C.OP_LINEAR]
    if c.di_scale > 0 and c.di_first_bn_multiplier != 1.0 and bn and prog.di_first_op != bn[0]:
        raise EngineError(f"deep_inversion: BatchNorm '{ops[prog.di_first_op].bn_module}' is registered first but "
                          f"'{ops[bn[0]].bn_module}' runs first; first_bn_multiplier belongs to the first registered one: register "
                          f"the BatchNorm layers in the order forward() runs them")
    if c.feat_scale > 0 and lin and prog.feature_op != lin[-1]:
        raise EngineError(f"features: Linear '{ops[prog.feature_op].module}' is registered last but '{ops[lin[-1]].module}' runs "
                          f"last; the prior reads the input of the last registered one: register the Linear layers in the order "
                          f"forward() runs them")


class Engine:
    """One engine = one model replica + one trial state on one GPU."""

    def __init__(self, model, input_shape, cfg_attack, device, noise_seed=0, backend=None, program=None):
        """``backend``: "tc" (TF32 tensor-core GEMMs, default; shapes it does not cover run on the fp32 SIMT
        kernels) or "simt" (fp32 CUDA-core GEMMs everywhere: bit-faithful fp32 products).  Default from
        ``BRE_GEMM_BACKEND``."""
        self.lib = load_library()
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise EngineError("the engine runs on CUDA devices only (no CPU fallback)")
        self.model = model
        # ``program``: an already lowered layer program (compiler.compile_transformer for token-sequence models, whose
        # candidate is the embedding sequence [batch, seq_len, d]); default: lower the vision model with torch.fx
        self.prog = program if program is not None else C.compile_model(model, input_shape)
        self.input_shape = tuple(int(s) for s in input_shape)
        self.ccfg = make_cfg(cfg_attack, noise_seed)
        prog = self.prog
        if program is None:
            _check_prior_layers(prog, self.ccfg)
        tens = (TensorDesc * len(prog.tensors))(*[TensorDesc(t.N, t.C, t.H, t.W) for t in prog.tensors])
        pds = []
        for p in prog.params:
            if p.perm == C.PERM_OIHW_TO_OHWI:
                pds.append(ParamDesc(p.numel, 1, p.shape[0], p.shape[1], p.shape[2] * p.shape[3]))
            elif p.perm == C.PERM_LINEAR_CHW_TO_HWC:
                pds.append(ParamDesc(p.numel, 1, p.shape[0], p.perm_c, p.perm_hw))
            else:   # plain layout; d0 carries the reserved element count when a zero tail is wanted (padded vocabulary)
                pds.append(ParamDesc(p.numel, 0, int(getattr(p, "alloc_numel", 0) or 0), 0, 0))
        self._bn_modules = []
        ops = []
        mods = C.bn_modules(model, prog) if program is None else [None] * len(prog.ops)
        for op, mod in zip(prog.ops, mods):
            bn_idx = -1
            if mod is not None:
                bn_idx = len(self._bn_modules)
                self._bn_modules.append(mod)
            ops.append(OpDesc(op.kind, op.tin, op.tout, op.res, op.R, op.S, op.stride, op.pad, op.w, op.b, int(op.has_bn),
                              int(op.relu), op.gamma, op.beta, bn_idx, float(op.eps), int(op.acc_in), int(op.acc_res),
                              int(getattr(op, "bn_train", False))))
        self._keep = (tens, (OpDesc * len(ops))(*ops), (ParamDesc * len(pds))(*pds))
        handle = ctypes.c_void_p()
        dev_index = self.device.index if self.device.index is not None else torch.cuda.current_device()
        rc = self.lib.bre_engine_create(self._keep[0], len(prog.tensors), self._keep[1], len(ops), self._keep[2], len(pds),
                                        prog.logits, ctypes.byref(self.ccfg), dev_index, ctypes.byref(handle))
        _check(self.lib, rc, "bre_engine_create")
        self.h = handle
        backend = backend or os.environ.get("BRE_GEMM_BACKEND", "tc")
        if backend not in ("tc", "simt"):
            raise ValueError(f"unknown GEMM backend {backend}")
        self.backend = backend
        self.set_option("gemm_backend", 1 if backend == "tc" else 0)
        valid = getattr(prog, "logits_valid", 0)
        if valid and valid != prog.tensors[prog.logits].C:
            self.set_option("logits_valid", valid)
        self.numel = 1
        for s in self.input_shape:
            self.numel *= s

    def close(self):
        if getattr(self, "h", None):
            self.lib.bre_engine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass

    # ---------------------------------------------------------------------------------------------
    def _ptr_array(self, tensors):
        arr = (ctypes.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])
        return arr

    def load_model(self, params=None, buffers_from=None):
        """``params``: list of tensors in ``model.parameters()`` order (default: the model's own)."""
        params = [_f32c(p) for p in (params if params is not None else self.model.parameters())]
        mods = self._bn_modules
        # train-mode BN (no buffers anywhere, base_attack.py:192-197) has no running statistics: placeholders, never read
        means = [_f32c(m.running_mean) if m.running_mean is not None else torch.zeros(m.num_features) for m in mods]
        vars_ = [_f32c(m.running_var) if m.running_var is not None else torch.ones(m.num_features) for m in mods]
        torch.cuda.synchronize(self.device) if any(p.is_cuda for p in params) else None
        pa, ma, va = self._ptr_array(params), self._ptr_array(means), self._ptr_array(vars_)
        rc = self.lib.bre_engine_load_model(self.h, pa, len(params), ma, va, len(mods))
        _check(self.lib, rc, "bre_engine_load_model")
        for i, op in enumerate(self.prog.ops):   # constant tables of the program (the fixed positional encoding)
            if op.kind == C.OP_POSCONST:
                table = _f32c(op.table)
                rc = self.lib.bre_engine_load_constant(self.h, i, _ptr(table), table.numel())
                _check(self.lib, rc, "bre_engine_load_constant")

    def load_targets(self, gradients, labels, mean=None, std=None, tensor_weights=None):
        grads = [_f32c(g) for g in gradients]
        labels = labels.detach().to(torch.int64).contiguous()
        if any(g.is_cuda for g in grads) or labels.is_cuda:
            torch.cuda.synchronize(self.device)
        tw = None if tensor_weights is None else _f32c(tensor_weights).cpu()
        mean_t = None if mean is None else torch.as_tensor(mean, dtype=torch.float32).flatten().contiguous().cpu()
        std_t = None if std is None else torch.as_tensor(std, dtype=torch.float32).flatten().contiguous().cpu()
        ga = self._ptr_array(grads)
        rc = self.lib.bre_engine_load_targets(self.h, ga, len(grads), _ptr(tw), _ptr(labels), labels.numel(), _ptr(mean_t),
                                              _ptr(std_t), 0 if mean_t is None else mean_t.numel())
        _check(self.lib, rc, "bre_engine_load_targets")

    def load_feature_targets(self, measured):
        """``measured``: [N, F] in torch (flatten) feature order; permuted here if the head sees a spatial map."""
        lin = [op for op in self.prog.ops if op.kind == C.OP_LINEAR][-1]
        ti = self.prog.tensors[lin.tin]
        m = _f32c(measured)
        if ti.H * ti.W > 1:
            m = m.view(ti.N, ti.C, ti.H * ti.W).permute(0, 2, 1).contiguous()
        if m.is_cuda:
            torch.cuda.synchronize(self.device)
        _check(self.lib, self.lib.bre_engine_load_feature_targets(self.h, _ptr(m), m.numel()), "bre_engine_load_feature_targets")

    def set_local_steps(self, total_images, steps, lr, labels_per_step):
        """FedAvg: ``labels_per_step`` = list of ``steps`` LongTensors of length ``data_per_step`` (the program batch).

        Supported with the matching objectives, TV / norm / orthogonality on the whole candidate, and ``task_regularization`` and
        DeepInversion on the last local step (its task loss, the BN-input statistics of its forward; both need ``lr != 0``).
        Train-mode BN (no BN buffers shared) normalises every local step with its own batch statistics.  The feature prior (its
        target is the input feature of no forward pass once the update spans several steps) and a train-mode BN layer that would
        normalise one value per channel (``data_per_step * H * W == 1``; torch refuses that training step too) raise
        ``EngineError``."""
        labels = torch.cat([l.detach().to(torch.int64).flatten().cpu() for l in labels_per_step]).contiguous()
        if labels.numel() != steps * self.input_shape[0]:
            raise EngineError("labels_per_step must hold data_per_step labels for every local step")
        _check(self.lib, self.lib.bre_engine_set_local_steps(self.h, int(total_images), int(steps), float(lr), _ptr(labels)),
               "bre_engine_set_local_steps")
        self.input_shape = (int(total_images), *self.input_shape[1:])
        self.numel = 1
        for s_ in self.input_shape:
            self.numel *= s_

    def set_trial_index(self, trial):
        """Global index of the trials begun from now on: each index draws its own Langevin noise field from the engine's seed."""
        _check(self.lib, self.lib.bre_engine_set_trial_index(self.h, int(trial)), "bre_engine_set_trial_index")

    def begin_trial(self, candidate, lr_table, trial=0):
        self.set_trial_index(trial)
        cand = _f32c(candidate)
        if cand.numel() != self.numel:
            raise EngineError(f"candidate has {cand.numel()} elements, engine expects {self.numel}")
        lr = torch.as_tensor(lr_table, dtype=torch.float32).contiguous().cpu()
        if cand.is_cuda:
            torch.cuda.synchronize(self.device)
        _check(self.lib, self.lib.bre_engine_begin_trial(self.h, _ptr(cand), _ptr(lr), lr.numel()), "bre_engine_begin_trial")

    def begin_joint_trial(self, candidate, label_logits, lr_table, trial=0):
        """Joint data + label optimisation on the device: ``label_logits`` [N, classes] (token models: [batch, seq, vocab])."""
        self.set_trial_index(trial)
        cand, ell = _f32c(candidate, self.device), _f32c(label_logits, self.device)
        if cand.numel() != self.numel:
            raise EngineError(f"candidate has {cand.numel()} elements, engine expects {self.numel}")
        lr = torch.as_tensor(lr_table, dtype=torch.float32).contiguous().cpu()
        torch.cuda.synchronize(self.device)
        self._label_shape = tuple(label_logits.shape)
        _check(self.lib, self.lib.bre_engine_begin_joint_trial(self.h, _ptr(cand), _ptr(ell), ell.numel(), _ptr(lr), lr.numel()),
               "bre_engine_begin_joint_trial")

    def begin_lbfgs_trial(self, candidate, lr_table, label_logits=None, trial=0):
        """L-BFGS trial on the device (torch.optim.LBFGS with the defaults of attacks/lbfgs.py): each ``run`` iteration is one
        ``optimizer.step`` with its inner loop inside the captured graph.  ``label_logits`` [N, classes]: the label leaf of a joint
        trial, optimised as one flat vector after the candidate."""
        self.set_trial_index(trial)
        cand = _f32c(candidate, self.device)
        if cand.numel() != self.numel:
            raise EngineError(f"candidate has {cand.numel()} elements, engine expects {self.numel}")
        ell = None if label_logits is None else _f32c(label_logits, self.device)
        lr = torch.as_tensor(lr_table, dtype=torch.float32).contiguous().cpu()
        torch.cuda.synchronize(self.device)
        if ell is not None:
            self._label_shape = tuple(label_logits.shape)
        consts = lbfgs_consts()
        _check(self.lib, self.lib.bre_engine_begin_lbfgs_trial(self.h, _ptr(cand), _ptr(ell), 0 if ell is None else ell.numel(), _ptr(lr),
                                                               lr.numel(), ctypes.byref(consts)), "bre_engine_begin_lbfgs_trial")

    def lbfgs_counters(self):
        """dict(inner_iterations, closures, pairs, first_slot) of the running L-BFGS trial (one host sync)."""
        out = (ctypes.c_int32 * 4)()
        _check(self.lib, self.lib.bre_engine_lbfgs_counters(self.h, out), "bre_engine_lbfgs_counters")
        return dict(zip(("inner_iterations", "closures", "pairs", "first_slot"), list(out)))

    def joint_labels(self, best=True):
        out = torch.empty(self._label_shape, dtype=torch.float32, device=self.device)
        _check(self.lib, self.lib.bre_engine_get_joint_labels(self.h, int(bool(best)), _ptr(out)), "bre_engine_get_joint_labels")
        return out

    def set_augmentations(self, plan):
        """``plan`` (attacks/augment.py ``AugmentationPlan``) or ``None`` to switch augmentations off.  A plan with ``stages`` (it
        contains a resample or blur stage) runs the model on the view's shape, which must be this engine's program shape; the
        candidate then has the plan's candidate shape and ``input_shape`` / ``numel`` follow it."""
        if plan is not None and plan.stages:
            return self._set_augmentation_stages(plan)
        from .attacks import augment as A

        if plan is None:
            _check(self.lib, self.lib.bre_engine_set_augmentations(self.h, 0, None, None, 0, 0.0, 0, None, None, 0, 0), "bre_engine_set_augmentations")
            self._candidate_shape(None)
            return
        n = len(plan.steps)
        kinds = (ctypes.c_int32 * max(n, 1))(*[k for k, _ in plan.steps])
        params = (ctypes.c_float * max(n, 1))(*[float(p) for _, p in plan.steps])
        scale = None if plan.colour_scale is None else _f32c(plan.colour_scale, self.device)
        shift = None if plan.colour_shift is None else _f32c(plan.colour_shift, self.device)
        torch.cuda.synchronize(self.device)
        self._aug_keep = (scale, shift)
        _check(self.lib, self.lib.bre_engine_set_augmentations_ex(self.h, n, kinds, params, int(plan.continuous_shift is not None),
                                                                  float(plan.continuous_shift or 0.0), int(plan.circular), A.CS_MODES[plan.cs_mode],
                                                                  A.CS_PADDINGS[plan.cs_padding], int(plan.fliplr), int(plan.flipud), _ptr(scale),
                                                                  _ptr(shift), int(plan.differentiable), int(plan.seed) & 0xFFFFFFFFFFFFFFFF),
               "bre_engine_set_augmentations_ex")
        self._candidate_shape(None)

    def _candidate_shape(self, shape):
        """Candidate shape of a stage plan (``None``: back to the shape the engine was built for)."""
        if shape is None:
            shape, self._built_shape = getattr(self, "_built_shape", None) or self.input_shape, None
        elif getattr(self, "_built_shape", None) is None:
            self._built_shape = self.input_shape
        self.input_shape = tuple(int(s) for s in shape)
        self.numel = 1
        for s_ in self.input_shape:
            self.numel *= s_

    def _set_augmentation_stages(self, plan):
        from .attacks import augment as A

        arr = (AugStageEx * len(plan.stages))()
        keep = []
        for st, ex in zip(plan.stages, arr):
            cs = ex.stage
            cs.Ho, cs.Wo = st.out_hw
            if st.kind == A.PIXEL:
                ex.cs_mode, ex.cs_padding = A.CS_MODES[st.cs_mode], A.CS_PADDINGS[st.cs_padding]
                ex.cs_fliplr, ex.cs_flipud = int(st.fliplr), int(st.flipud)
                cs.kind, cs.n_steps = 0, len(st.steps)
                for i, (k, p) in enumerate(st.steps):
                    cs.kinds[i], cs.params[i] = int(k), float(p)
                cs.cs_enabled, cs.cs_shift, cs.cs_circular = int(st.continuous_shift is not None), float(st.continuous_shift or 0.0), int(st.circular)
                if st.colour_scale is not None:
                    sc, sh = _f32c(st.colour_scale, self.device), _f32c(st.colour_shift, self.device)
                    keep += [sc, sh]
                    cs.cj_scale, cs.cj_shift = sc.data_ptr(), sh.data_ptr()
            elif st.kind == A.RESAMPLE:
                cs.kind = 1
                (cs.y0, cs.x0), (cs.wh, cs.ww) = st.corner, st.window
                cs.focus, cs.focus_std = int(st.focus_std is not None), float(st.focus_std or 0.0)
            else:
                cs.kind, cs.width, cs.stride = 2, int(st.width), int(st.stride)
        torch.cuda.synchronize(self.device)
        self._aug_keep = tuple(keep)
        N, Cc, H, W = plan.candidate_shape
        _check(self.lib, self.lib.bre_engine_set_augmentation_stages_ex(self.h, len(plan.stages), arr, N, Cc, H, W, int(plan.differentiable),
                                                                        int(plan.seed) & 0xFFFFFFFFFFFFFFFF), "bre_engine_set_augmentation_stages_ex")
        self._candidate_shape(plan.candidate_shape)

    def last_augmentation(self):
        o1, o2 = (ctypes.c_int32 * 4)(), (ctypes.c_int32 * 4)()
        sx, sy = (ctypes.c_float * 64)(), (ctypes.c_float * 64)()
        _check(self.lib, self.lib.bre_engine_last_augmentation(self.h, o1, o2, sx, sy), "bre_engine_last_augmentation")
        n = self.input_shape[0]
        return list(o1), list(o2), list(sx)[:n], list(sy)[:n]

    def augmentation_draws(self):
        """Every stage's draws of the last evaluation: list of dicts (o1, o2: 4 offsets; sx, sy: per image; a focus stage's window
        corner is (o1[0], o2[0]) = (row, column))."""
        n_st = ctypes.c_int32()
        o1, o2 = (ctypes.c_int32 * 32)(), (ctypes.c_int32 * 32)()
        sx, sy = (ctypes.c_float * 512)(), (ctypes.c_float * 512)()
        _check(self.lib, self.lib.bre_engine_augmentation_draws(self.h, ctypes.byref(n_st), o1, o2, sx, sy), "bre_engine_augmentation_draws")
        n = self.input_shape[0]
        return [dict(o1=list(o1[4 * k:4 * k + 4]), o2=list(o2[4 * k:4 * k + 4]), sx=list(sx[64 * k:64 * k + n]), sy=list(sy[64 * k:64 * k + n]))
                for k in range(n_st.value)]

    def augmentation_flips(self):
        """The continuous shift's grid flips of the last evaluation, per stage: list of dicts (fliplr, flipud: 0 / 1 per image)."""
        n_st = ctypes.c_int32()
        lr, ud = (ctypes.c_int32 * 512)(), (ctypes.c_int32 * 512)()
        _check(self.lib, self.lib.bre_engine_augmentation_flips(self.h, ctypes.byref(n_st), lr, ud), "bre_engine_augmentation_flips")
        n = self.input_shape[0]
        return [dict(fliplr=list(lr[64 * k:64 * k + n]), flipud=list(ud[64 * k:64 * k + n])) for k in range(n_st.value)]

    def run(self, n_iters):
        _check(self.lib, self.lib.bre_engine_run(self.h, int(n_iters)), "bre_engine_run")

    def run_timed(self, n_iters):
        """Run ``n_iters`` iterations and return the device time in milliseconds (CUDA events on the engine stream)."""
        ms = ctypes.c_float()
        _check(self.lib, self.lib.bre_engine_run_timed(self.h, int(n_iters), ctypes.byref(ms)), "bre_engine_run_timed")
        return ms.value

    def sync(self):
        _check(self.lib, self.lib.bre_engine_sync(self.h), "bre_engine_sync")

    def status(self):
        rec, stop = ctypes.c_int32(), ctypes.c_int32()
        fmin, tl = ctypes.c_double(), ctypes.c_double()
        _check(self.lib, self.lib.bre_engine_status(self.h, ctypes.byref(rec), ctypes.byref(stop), ctypes.byref(fmin), ctypes.byref(tl)),
               "bre_engine_status")
        return dict(recorded=rec.value, stopped=bool(stop.value), min_objective=fmin.value, task_loss=tl.value)

    def history(self, n=None):
        n = self.status()["recorded"] if n is None else n
        out = torch.empty(max(n, 1), dtype=torch.float32)
        _check(self.lib, self.lib.bre_engine_read_history(self.h, _ptr(out), n), "bre_engine_read_history")
        return out[:n]

    def best(self, device=None):
        out = torch.empty(self.input_shape, dtype=torch.float32, device=device or self.device)
        torch.cuda.synchronize(self.device)
        _check(self.lib, self.lib.bre_engine_get_best(self.h, _ptr(out)), "bre_engine_get_best")
        return out

    def candidate(self, device=None):
        out = torch.empty(self.input_shape, dtype=torch.float32, device=device or self.device)
        torch.cuda.synchronize(self.device)
        _check(self.lib, self.lib.bre_engine_get_candidate(self.h, _ptr(out)), "bre_engine_get_candidate")
        return out

    def score(self, candidate, scoring):
        cand = _f32c(candidate)
        if cand.is_cuda:
            torch.cuda.synchronize(self.device)
        out = ctypes.c_double()
        _check(self.lib, self.lib.bre_engine_score(self.h, _ptr(cand), OBJECTIVES[scoring], ctypes.byref(out)), "bre_engine_score")
        return out.value

    def objective_and_gradient(self, candidate):
        """(objective, d objective / d candidate) of one evaluation without an optimiser step.  With the option
        ``debug_multistep_stop`` set the evaluation stops part-way and neither return value is meaningful."""
        cand = _f32c(candidate)
        if cand.is_cuda:
            torch.cuda.synchronize(self.device)
        grad = torch.empty(self.input_shape, dtype=torch.float32, device=self.device)
        torch.cuda.synchronize(self.device)
        val = ctypes.c_double()
        _check(self.lib, self.lib.bre_engine_objective_and_gradient(self.h, _ptr(cand), ctypes.byref(val), _ptr(grad)),
               "bre_engine_objective_and_gradient")
        return val.value, grad

    def last_terms(self):
        arr = (ctypes.c_double * 6)()
        _check(self.lib, self.lib.bre_engine_last_terms(self.h, arr), "bre_engine_last_terms")
        return dict(zip(("match", "task_loss", "total_variation", "norm", "deep_inversion", "features"), list(arr)))

    # ---- joint data / label optimisation (optimization_with_label_attack.py) --------------------------------
    def load_soft_labels(self, probabilities):
        """Class probabilities [N, classes] as the targets of the task loss (``None`` -> back to index labels)."""
        if probabilities is None:
            _check(self.lib, self.lib.bre_engine_load_soft_labels(self.h, None, 0), "bre_engine_load_soft_labels")
            return
        q = _f32c(probabilities, self.device)
        _check(self.lib, self.lib.bre_engine_load_soft_labels(self.h, _ptr(q), q.numel()), "bre_engine_load_soft_labels")

    def label_gradient(self, shape):
        """d(objective)/d(probabilities) of the last ``objective_and_gradient`` call."""
        out = torch.empty(shape, dtype=torch.float32, device=self.device)
        _check(self.lib, self.lib.bre_engine_label_gradient(self.h, _ptr(out)), "bre_engine_label_gradient")
        return out

    def set_labels(self, labels):
        lab = labels.detach().to(device=self.device, dtype=torch.int64).contiguous()
        _check(self.lib, self.lib.bre_engine_set_labels(self.h, _ptr(lab), lab.numel()), "bre_engine_set_labels")

    # ---- the steps either side of the hot path (SURVEY section 8 f-2 / f-3) -----------------------------------------------
    def param_gradients(self, data, labels):
        """Gradient of the mean task loss w.r.t. every parameter at ``data`` (cases/users.py:148-156): list of device tensors in
        ``model.parameters()`` order and torch layout, and the loss value."""
        x = _f32c(data, self.device)
        lab = labels.detach().to(device=self.device, dtype=torch.int64).contiguous()
        outs = [torch.empty(p.shape, dtype=torch.float32, device=self.device) for p in self.prog.params]
        torch.cuda.synchronize(self.device)
        loss = ctypes.c_double()
        _check(self.lib, self.lib.bre_engine_param_gradients(self.h, _ptr(x), _ptr(lab), lab.numel(), self._ptr_array(outs), len(outs),
                                                             ctypes.byref(loss)), "bre_engine_param_gradients")
        return outs, loss.value

    def bn_batch_stats(self):
        """(mean, biased variance) per train-mode BN layer of the last forward."""
        out = []
        for j, mod in enumerate(self._bn_modules):
            m = torch.empty(mod.num_features, dtype=torch.float32, device=self.device)
            v = torch.empty_like(m)
            _check(self.lib, self.lib.bre_engine_bn_batch_stats(self.h, j, _ptr(m), _ptr(v)), "bre_engine_bn_batch_stats")
            out.append((m, v))
        return out

    def forward(self, data):
        x = _f32c(data, self.device)
        lt = self.prog.tensors[self.prog.logits]
        out = torch.empty((lt.N, lt.C), dtype=torch.float32, device=self.device)
        torch.cuda.synchronize(self.device)
        _check(self.lib, self.lib.bre_engine_forward(self.h, _ptr(x), _ptr(out)), "bre_engine_forward")
        return out

    def debug_param(self, which, index):
        p = self.prog.params[index]
        out = torch.empty(p.shape, dtype=torch.float32)
        # "v_operand" / "W_operand": what the GEMMs read (the TF32 shadow for tensor-core layers; "v" is stale for those)
        code = {"G": 0, "v": 1, "W": 2, "g": 3, "v_operand": 4, "W_operand": 5}[which]
        _check(self.lib, self.lib.bre_engine_debug_param(self.h, code, index, _ptr(out)), "bre_engine_debug_param")
        return out

    def debug_step_param(self, which, step, index):
        """Multi-step engines: "W" = W_step, "W_operand" = W_step as the GEMMs read it, "D" = the accumulated W_K - W_0 (``step``
        ignored); which of them are valid at which ``debug_multistep_stop`` is listed in include/breaching_b200.h."""
        p = self.prog.params[index]
        out = torch.empty(p.shape, dtype=torch.float32)
        code = {"W": 0, "W_operand": 1, "D": 2}[which]
        _check(self.lib, self.lib.bre_engine_debug_step_param(self.h, code, int(step), index, _ptr(out)), "bre_engine_debug_step_param")
        return out

    def debug_tensor(self, which, tid):
        t = self.prog.tensors[tid]
        out = torch.empty((t.N, t.C, t.H, t.W), dtype=torch.float32)
        code = {"val": 0, "delta": 1, "tangent": 2, "tangent_delta": 3}[which]
        _check(self.lib, self.lib.bre_engine_debug_tensor(self.h, code, tid, _ptr(out)), "bre_engine_debug_tensor")
        return out

    def debug_step_state(self, which):
        """What the optimiser step of the last iteration read and left: "grad" (candidate gradient before noise / clip / sign),
        "grad_task" (raises when the step reads no separate task gradient), "m", "v"; "label_grad" / "label_m" / "label_v" for the
        label-logit leaf of a joint trial, and "soft_q": the soft targets softmax(label logits) the last joint iteration evaluated."""
        code = {"grad": 0, "grad_task": 1, "m": 2, "v": 3, "label_grad": 4, "label_m": 5, "label_v": 6, "soft_q": 7}[which]
        out = torch.empty(self._label_shape if code >= 4 else self.input_shape, dtype=torch.float32)
        _check(self.lib, self.lib.bre_engine_debug_step_state(self.h, code, _ptr(out)), "bre_engine_debug_step_state")
        return out

    def debug_op(self, index):
        """What the engine did with op ``index`` in the last sweeps: dict(fused, tangent_in_unwritten, stem_columns)."""
        out = ctypes.c_int32()
        _check(self.lib, self.lib.bre_engine_debug_op(self.h, int(index), ctypes.byref(out)), "bre_engine_debug_op")
        f = out.value
        return dict(fused=bool(f & 1), tangent_in_unwritten=bool(f & 2), stem_columns=bool(f & 4))

    def launches_per_iteration(self):
        out = ctypes.c_int32()
        _check(self.lib, self.lib.bre_engine_launches_per_iteration(self.h, ctypes.byref(out)), "bre_engine_launches_per_iteration")
        return out.value

    def set_option(self, name, value):
        _check(self.lib, self.lib.bre_engine_set_option(self.h, name.encode(), int(value)), "bre_engine_set_option")


# ---- stand-alone kernels ---------------------------------------------------------------------------
def match_reduce(G, g, chunk_weights=None, mask_value=-1.0, readback=True):
    lib = load_library()
    assert G.is_cuda and g.is_cuda and G.dtype == torch.float32 and G.is_contiguous() and g.is_contiguous()
    out = (ctypes.c_double * 5)()
    stream = torch.cuda.current_stream(G.device).cuda_stream
    with torch.cuda.device(G.device):
        rc = lib.bre_match_reduce(_ptr(G), _ptr(g), _ptr(chunk_weights), G.numel(), float(mask_value),
                                  out if readback else None, ctypes.c_void_p(stream))
    _check(lib, rc, "bre_match_reduce")
    return list(out) if readback else None


def optimizer_step(x, m, v, best, grad, ccfg, lr_table, history, scalars, grad_task=None, lo=None, hi=None, C=1, HW=1):
    """One optimiser step + bookkeeping of the engine's iteration on caller-owned CUDA tensors (updated in place): the kernels
    ``Engine.run`` launches after the sweeps.  ``ccfg``: ``AttackCfg``; ``lr_table`` / ``history`` / ``lo`` / ``hi``: CUDA fp32;
    ``scalars``: dict(it, fmin, match, task_loss, tv, norm, di, feat, recorded, stopped, trial), missing entries 0 (fmin: +inf).
    Returns the dict after the step, with ``grad_norm_sq`` and ``last_objective``."""
    lib = load_library()
    for t in (x, m, v, best, grad, lr_table, history, grad_task, lo, hi):
        assert t is None or (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous())
    io = StepScalars()
    io.fmin = float("inf")
    for key, val in scalars.items():
        setattr(io, key, val)
    stream = torch.cuda.current_stream(x.device).cuda_stream
    with torch.cuda.device(x.device):
        rc = lib.bre_optimizer_step(_ptr(x), _ptr(m), _ptr(v), _ptr(best), _ptr(grad), _ptr(grad_task), _ptr(lr_table), lr_table.numel(),
                                    _ptr(lo), _ptr(hi), x.numel(), int(C), int(HW), ctypes.byref(ccfg), _ptr(history), history.numel(),
                                    ctypes.byref(io), ctypes.c_void_p(stream))
    _check(lib, rc, "bre_optimizer_step")
    return {name: getattr(io, name) for name, _ in StepScalars._fields_}


def lbfgs_direction(S, Y, gram, state, g, prev_g, d, consts=None):
    """One inner iteration's direction through the engine's L-BFGS kernels on caller-owned CUDA tensors (updated in place; see
    ``bre_lbfgs_direction``): S, Y [history + 1, n] fp32 rings, ``gram`` fp64 [2 (h+1)^2 + 3 (h+1)], ``state`` a CUDA uint8 tensor
    holding one ``LbfgsScalars``, g / prev_g / d [n] fp32.  Returns the state after the call as an ``LbfgsScalars``."""
    lib = load_library()
    consts = consts or lbfgs_consts()
    R = consts.history + 1
    n = g.numel()
    for t in (S, Y, g, prev_g, d):
        assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()
    assert S.numel() == R * n and Y.numel() == R * n and prev_g.numel() == n and d.numel() == n
    assert gram.is_cuda and gram.dtype == torch.float64 and gram.numel() == 2 * R * R + 3 * R
    assert state.is_cuda and state.dtype == torch.uint8 and state.numel() == ctypes.sizeof(LbfgsScalars)
    stream = torch.cuda.current_stream(g.device).cuda_stream
    with torch.cuda.device(g.device):
        rc = lib.bre_lbfgs_direction(_ptr(S), _ptr(Y), _ptr(gram), _ptr(state), _ptr(g), _ptr(prev_g), _ptr(d), n, ctypes.byref(consts),
                                     ctypes.c_void_p(stream))
    _check(lib, rc, "bre_lbfgs_direction")
    return LbfgsScalars.from_buffer_copy(bytes(state.cpu().numpy().tobytes()))


def lbfgs_state(scalars=None, device="cuda"):
    """A device ``LbfgsScalars`` block (CUDA uint8 tensor) holding ``scalars`` (default: a fresh optimiser, h_diag = 1)."""
    if scalars is None:
        scalars = LbfgsScalars()
        scalars.h_diag = 1.0
    raw = bytes(bytearray(scalars))
    return torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(device)


def langevin_noise(seed, trial, it, n, first=0, device="cuda"):
    """The N(0,1) draws the step kernels use for elements ``first .. first + n`` in iteration ``it`` of trial ``trial``."""
    lib = load_library()
    out = torch.empty(int(n), dtype=torch.float32, device=device)
    stream = torch.cuda.current_stream(out.device).cuda_stream
    with torch.cuda.device(out.device):
        rc = lib.bre_langevin_noise(int(seed) & 0xFFFFFFFFFFFFFFFF, int(trial), int(it), int(first), out.numel(), _ptr(out), ctypes.c_void_p(stream))
    _check(lib, rc, "bre_langevin_noise")
    return out


def total_variation(x, scale=0.1, inner_exp=1.0, outer_exp=1.0, eps=1e-8, double_opponents=False, grad=None):
    lib = load_library()
    assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous() and x.shape[1] == 3
    accumulate = grad is not None
    grad = torch.empty_like(x) if grad is None else grad
    val = ctypes.c_double()
    stream = torch.cuda.current_stream(x.device).cuda_stream
    with torch.cuda.device(x.device):
        rc = lib.bre_total_variation(_ptr(x), _ptr(grad), x.shape[0], x.shape[2], x.shape[3], scale, inner_exp, outer_exp,
                                     eps, int(double_opponents), int(accumulate), ctypes.byref(val), ctypes.c_void_p(stream))
    _check(lib, rc, "bre_total_variation")
    return val.value, grad


def augment_view(x, steps=(), offsets=(), continuous_shift=None, circular=True, uniforms=None, colour_scale=None, colour_shift=None,
                 transpose=False, mode="bilinear", padding="zeros", flips=None):
    """Stand-alone augmentation view (or its transpose) with explicit draws: ``steps`` = [(kind, param)], ``offsets`` = [(o1, o2)] per
    step (roll offsets; flip: (flag, 0)), ``uniforms`` = (sx, sy) lists per image for the continuous shift, sampled with grid_sample's
    ``mode`` and ``padding`` (zeros / border / reflection; ``circular`` wraps the grid first and needs zeros); ``flips`` = (fliplr,
    flipud) lists of 0 / 1 per image: that image's x / y grid coordinate is negated."""
    from .attacks.augment import CS_MODES, CS_PADDINGS

    if mode not in CS_MODES or padding not in CS_PADDINGS:
        raise ValueError(f"continuous_shift: unknown mode {mode!r} or padding {padding!r}")
    lib = load_library()
    x = _f32c(x).clone()
    N, C, H, W = x.shape
    out = torch.empty_like(x)
    n = len(steps)
    kinds = (ctypes.c_int32 * max(n, 1))(*[k for k, _ in steps])
    o1 = (ctypes.c_int32 * max(n, 1))(*[int(a) for a, _ in offsets])
    o2 = (ctypes.c_int32 * max(n, 1))(*[int(b) for _, b in offsets])
    sx = sy = lr = ud = None
    if continuous_shift is not None:
        sx, sy = (ctypes.c_float * N)(*[float(v) for v in uniforms[0]]), (ctypes.c_float * N)(*[float(v) for v in uniforms[1]])
        if flips is not None:
            lr, ud = (ctypes.c_int32 * N)(*[int(v) for v in flips[0]]), (ctypes.c_int32 * N)(*[int(v) for v in flips[1]])
    scratch = torch.empty_like(x)
    cs, csh = (None if colour_scale is None else _f32c(colour_scale, x.device)), (None if colour_shift is None else _f32c(colour_shift, x.device))
    stream = torch.cuda.current_stream(x.device).cuda_stream
    with torch.cuda.device(x.device):
        torch.cuda.synchronize(x.device)
        rc = lib.bre_augment_view_ex(_ptr(x), _ptr(out), N, C, H, W, n, kinds, o1, o2, float(continuous_shift or 0.0), int(circular),
                                     CS_MODES[mode], CS_PADDINGS[padding], sx, sy, lr, ud, _ptr(cs), _ptr(csh), int(transpose), _ptr(scratch),
                                     ctypes.c_void_p(stream))
    _check(lib, rc, "bre_augment_view_ex")
    return out


def augment_resample(x, corner, window, out_hw, transpose=False, in_hw=None):
    """Stand-alone RESAMPLE stage: the window ``corner`` = (y0, x0), ``window`` = (wh, ww) of x [N, C, H, W] resized bilinearly to
    ``out_hw``.  ``transpose``: x is the gradient at the view [N, C, Ho, Wo], pulled back to [N, C, *in_hw]."""
    lib = load_library()
    x = _f32c(x)
    N, C = x.shape[:2]
    Hi, Wi = (x.shape[2], x.shape[3]) if not transpose else in_hw
    out = torch.empty((N, C, *(in_hw if transpose else out_hw)), dtype=torch.float32, device=x.device)
    stream = torch.cuda.current_stream(x.device).cuda_stream
    with torch.cuda.device(x.device):
        rc = lib.bre_augment_resample(_ptr(x), _ptr(out), N, C, Hi, Wi, int(corner[0]), int(corner[1]), int(window[0]), int(window[1]),
                                      int(out_hw[0]), int(out_hw[1]), int(bool(transpose)), ctypes.c_void_p(stream))
    _check(lib, rc, "bre_augment_resample")
    return out


def augment_blur(x, width, stride=1, transpose=False, in_hw=None):
    """Stand-alone BLUR stage (antialias); ``transpose``: x is the gradient at the view, pulled back to [N, C, *in_hw]."""
    lib = load_library()
    x = _f32c(x)
    N, C = x.shape[:2]
    Hi, Wi = (x.shape[2], x.shape[3]) if not transpose else in_hw
    pad = width // 2
    Ho, Wo = (Hi + 2 * pad - width) // stride + 1, (Wi + 2 * pad - width) // stride + 1
    out = torch.empty((N, C, *((Hi, Wi) if transpose else (Ho, Wo))), dtype=torch.float32, device=x.device)
    stream = torch.cuda.current_stream(x.device).cuda_stream
    with torch.cuda.device(x.device):
        rc = lib.bre_augment_blur(_ptr(x), _ptr(out), N, C, Hi, Wi, int(width), int(stride), int(bool(transpose)), ctypes.c_void_p(stream))
    _check(lib, rc, "bre_augment_blur")
    return out


def resize_bilinear(x, size):
    """``F.interpolate(x, size=size, mode="bilinear", align_corners=False)`` for an NCHW fp32 batch on the device."""
    lib = load_library()
    assert x.is_cuda and x.dim() == 4
    x = _f32c(x)
    Ho, Wo = (int(size), int(size)) if not isinstance(size, (tuple, list)) else (int(size[0]), int(size[1]))
    out = torch.empty((x.shape[0], x.shape[1], Ho, Wo), dtype=torch.float32, device=x.device)
    stream = torch.cuda.current_stream(x.device).cuda_stream
    with torch.cuda.device(x.device):
        rc = lib.bre_resize_bilinear(_ptr(x), _ptr(out), x.shape[0], x.shape[1], x.shape[2], x.shape[3], Ho, Wo, ctypes.c_void_p(stream))
    _check(lib, rc, "bre_resize_bilinear")
    return out


def image_mse(rec, ref, mean=None, std=None, clamp=True):
    """Per-example MSE of the de-normalised, [0, 1]-clamped batches (analysis/analysis.py:228-242) -> list of floats."""
    lib = load_library()
    assert rec.is_cuda and rec.shape == ref.shape and rec.dim() == 4
    rec, ref = _f32c(rec), _f32c(ref, rec.device)
    N, C, H, W = rec.shape
    mean_a = std_a = None
    if mean is not None:
        mean_a = (ctypes.c_float * C)(*[float(v) for v in torch.as_tensor(mean).flatten().tolist()])
        std_a = (ctypes.c_float * C)(*[float(v) for v in torch.as_tensor(std).flatten().tolist()])
    out = (ctypes.c_double * N)()
    stream = torch.cuda.current_stream(rec.device).cuda_stream
    with torch.cuda.device(rec.device):
        rc = lib.bre_image_mse(_ptr(rec), _ptr(ref), N, C, H * W, mean_a, std_a, int(bool(clamp)), out, ctypes.c_void_p(stream))
    _check(lib, rc, "bre_image_mse")
    return list(out)


def conv_gemm(mode, a, w, out, N, H, W, Ci, Co, R, S, stride, pad, a2=None, w2=None, backend=0):
    """mode: 0 fprop / 1 dgrad / 2 wgrad on NHWC / OHWI device tensors (see the header)."""
    lib = load_library()
    stream = torch.cuda.current_stream(a.device).cuda_stream
    with torch.cuda.device(a.device):
        rc = lib.bre_conv_gemm(mode, backend, _ptr(a), _ptr(w), _ptr(a2), _ptr(w2), _ptr(out), N, H, W, Ci, Co, R, S, stride,
                               pad, ctypes.c_void_p(stream))
    _check(lib, rc, "bre_conv_gemm")
    return out


GEMM_FAMILIES = {-1: None, 0: "igemm_simt", 1: "dgrad_small_ci", 2: "linear_small", 3: "linear_tall", 4: "tc"}
GEMM_PRODUCERS = {0: None, 1: "tma", 2: "cp.async", 3: "classes"}


def _plan_dict(buf):
    v = list(buf)
    return dict(family=GEMM_FAMILIES[v[0]], mode=v[1], nsrc=v[2], tile_rows=v[3], tile_width=v[4], splits=v[5], stages=v[6],
                producer=GEMM_PRODUCERS[v[7]], total_kblocks=v[8], kblocks_per_split=v[9], vec=v[10])


def last_gemm_plan():
    """The launch plan of the last GEMM issued by this host thread (bre_debug_last_gemm_plan): kernel family, mode, nsrc, tile rows /
    width, split-K factor, ring depth, operand producer, k-blocks in all and per split, and the SIMT vector-loader flags."""
    lib = load_library()
    buf = (ctypes.c_int32 * 11)()
    _check(lib, lib.bre_debug_last_gemm_plan(buf), "bre_debug_last_gemm_plan")
    return _plan_dict(buf)


def gemm_plan(mode, backend, N, H, W, Ci, Co, R, S, stride, pad, nsrc=1):
    """The launch plan conv_gemm would run for this contraction (bre_gemm_plan), in the form of last_gemm_plan(); family None where
    backend 1 does not cover the shape.  Nothing is allocated or launched."""
    lib = load_library()
    buf = (ctypes.c_int32 * 11)()
    _check(lib, lib.bre_gemm_plan(mode, backend, N, H, W, Ci, Co, R, S, stride, pad, nsrc, buf), "bre_gemm_plan")
    return _plan_dict(buf)


def row_plan(C):
    """The plan of the cluster row kernels for rows of ``C`` elements: (CTAs per row, True when each CTA's segment is cached in
    registers, False when it is streamed)."""
    lib = load_library()
    cs, fits = ctypes.c_int32(), ctypes.c_int32()
    _check(lib, lib.bre_debug_row_plan(int(C), ctypes.byref(cs), ctypes.byref(fits)), "bre_debug_row_plan")
    return cs.value, bool(fits.value)


ROW_OPS = {"softmax": 0, "softmax_chain": 1, "token_ce_fwd": 2, "token_ce_tan_bwd": 3, "token_label_grad": 4, "ce_fwd": 5,
           "ce_label_grad": 6, "ce_tan_bwd": 7}


def row_op(op, in0, in1=None, in2=None, labels=None, C=None, T=1, coef=0.0, round_out=False, out0=None, out1=None, out2=None):
    """One row kernel of the label leaf or the cross-entropy seeds through the engine's launcher (``bre_row_op``; the operands
    of each ``op`` are listed in include/breaching_b200.h).  CUDA fp32 tensors [rows, width]; logits-shaped tensors of the token
    ops may be wider than ``C`` (row stride Vs = their width).  Outputs are written in place; missing ones are allocated like
    ``in0`` ([rows] for the loss).  Returns (out0, out1, out2)."""
    lib = load_library()
    rows, Vs = in0.shape
    C = Vs if C is None else int(C)
    for t in (in0, in1, in2, out0, out1, out2):
        assert t is None or (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous())
    assert labels is None or (labels.is_cuda and labels.dtype == torch.int64 and labels.is_contiguous())
    fwd = op in ("token_ce_fwd", "ce_fwd")
    out0 = torch.empty_like(in0) if out0 is None else out0
    out1 = torch.empty(rows, dtype=torch.float32, device=in0.device) if fwd and out1 is None else out1
    out2 = torch.empty_like(in0) if fwd and out2 is None else out2
    stream = torch.cuda.current_stream(in0.device).cuda_stream
    with torch.cuda.device(in0.device):
        rc = lib.bre_row_op(ROW_OPS[op], _ptr(in0), _ptr(in1), _ptr(in2), _ptr(labels), rows, C, Vs, int(T), float(coef), int(bool(round_out)),
                            _ptr(out0), _ptr(out1), _ptr(out2), ctypes.c_void_p(stream))
    _check(lib, rc, "bre_row_op")
    return out0, out1, out2


def token_layernorm(sweep, x, gamma, beta, stats, in1=None, in2=None, in3=None, v_gamma=None, v_beta=None, eps=1e-5, want_param_grad=False,
                    round_out=False):
    """Stand-alone LayerNorm sweep (csrc/tokens.cu) on [rows, C] device tensors; returns ``out`` (and the gamma / beta
    gradients for sweep 1 with ``want_param_grad``).  ``round_out``: store ``out`` on the TF32 grid (as the engine does for
    tensor-core GEMM operands)."""
    lib = load_library()
    rows, C = x.shape
    out = torch.empty_like(x)
    gg = torch.empty(C, device=x.device) if want_param_grad else None
    gb = torch.empty(C, device=x.device) if want_param_grad else None
    stream = torch.cuda.current_stream(x.device).cuda_stream
    with torch.cuda.device(x.device):
        rc = lib.bre_token_layernorm(sweep, _ptr(x), _ptr(in1), _ptr(in2), _ptr(in3), _ptr(gamma), _ptr(beta), _ptr(v_gamma), _ptr(v_beta),
                                     float(eps), rows, C, _ptr(stats), _ptr(out), _ptr(gg), _ptr(gb), int(bool(round_out)), ctypes.c_void_p(stream))
    _check(lib, rc, "bre_token_layernorm")
    return (out, gg, gb) if want_param_grad else out


def token_match(rec, emb, subset=None):
    """Nearest vocabulary embedding of every row of ``rec`` [rows, d] under the reference's centred similarity (base_attack.py:126-133);
    ``subset`` (int64 ids) restricts the candidates and the result indexes into it.  Device tensors; returns int64 [rows]."""
    lib = load_library()
    rec = rec.detach().to(torch.float32).contiguous()
    emb = emb.detach().to(torch.float32).contiguous()
    if subset is not None:
        subset = subset.detach().to(torch.int64).contiguous()
    V = int(subset.numel()) if subset is not None else int(emb.shape[0])
    out = torch.empty(rec.shape[0], dtype=torch.int64, device=rec.device)
    stream = torch.cuda.current_stream(rec.device).cuda_stream
    with torch.cuda.device(rec.device):
        rc = lib.bre_token_match(_ptr(rec), _ptr(emb), _ptr(subset), int(rec.shape[0]), int(rec.shape[1]), V, _ptr(out), ctypes.c_void_p(stream))
    _check(lib, rc, "bre_token_match")
    return out


def token_attention(sweep, qkv, B, T, heads, P, Pd, in1=None, in2=None, in3=None, round_out=False, cluster=None):
    """Stand-alone multi-head self-attention sweep (csrc/tokens.cu); qkv [B*T, 3 d].  ``round_out``: store ``out`` on the TF32
    grid.  ``cluster``: None or 0 = the engine's choice (the resident-head kernel when 8 T dh + 4 T^2 floats fit 200 KB of shared
    memory, else the head split over the smallest cluster of CTAs whose column slices fit), 1 = the resident-head kernel, 2 .. 8 =
    the head split over that many CTAs.  A shape no kernel holds raises."""
    lib = load_library()
    d = qkv.shape[1] // 3
    out = torch.empty(qkv.shape[0], d if sweep in (0, 2) else 3 * d, device=qkv.device)
    stream = torch.cuda.current_stream(qkv.device).cuda_stream
    args = (sweep, _ptr(qkv), _ptr(in1), _ptr(in2), _ptr(in3), B, T, heads, d // heads, _ptr(P), _ptr(Pd), _ptr(out), int(bool(round_out)),
            ctypes.c_void_p(stream))
    with torch.cuda.device(qkv.device):
        if cluster is None:
            rc = lib.bre_token_attention(*args)
        else:
            rc = lib.bre_token_attention_ex(*args, int(cluster))
    _check(lib, rc, "bre_token_attention")
    return out


def token_attention_plan(T, dh, cluster=0):
    """CTAs per (sequence, head) the attention sweeps run with (1 = the resident-head kernel), or None when the shape is refused."""
    lib = load_library()
    n = ctypes.c_int32()
    _check(lib, lib.bre_token_attention_plan(int(T), int(dh), int(cluster), ctypes.byref(n)), "bre_token_attention_plan")
    return None if n.value < 0 else n.value
