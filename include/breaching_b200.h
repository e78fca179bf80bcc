/* breaching_b200 -- C ABI of the sm_90a gradient-inversion engine.
 *
 * Drop-in boundary (SURVEY.md section 8b).  The reference has no native code and no FFI of its own; the
 * interface a maintainer would bind is the body of
 *   OptimizationBasedAttacker._run_trial      breaching/attacks/optimization_based_attack.py:90-143
 *   closure of _compute_objective             breaching/attacks/optimization_based_attack.py:145-189
 *   GradientLoss.forward / _grad_fn_single_step  breaching/attacks/auxiliaries/objectives.py:26-46
 *   the *_sim / _euclidean list reductions    breaching/attacks/auxiliaries/objectives.py:91-95,135-141,160-164,185-196
 *   TotalVariation / Norm / DeepInversion / Feature regularizers   breaching/attacks/auxiliaries/regularizers.py
 *   optimizer_lookup (Adam/AdamW/SGD + LR)    breaching/attacks/auxiliaries/common.py:5-40
 *   _score_trial                              breaching/attacks/optimization_based_attack.py:191-204
 * Each entry point below names the reference lines it replaces.  INTEGRATION.md shows the ctypes stub.
 *
 * Conventions: plain C, no torch types.  All functions return 0 on success or a negative bre_status;
 * bre_last_error() gives the message of the last failure on the calling thread.  Pointers marked
 * "device or host" are copied with cudaMemcpyDefault (UVA), so either works; "device" pointers must
 * be resident on the engine's GPU.  One engine per GPU, not re-entrant.
 */
#ifndef BREACHING_B200_H
#define BREACHING_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct bre_engine bre_engine;

enum bre_status {
  BRE_OK = 0,
  BRE_ERR_INVALID = -1,     /* bad argument / unsupported configuration */
  BRE_ERR_CUDA = -2,        /* a CUDA runtime call failed */
  BRE_ERR_STATE = -3,       /* call order violated (e.g. run before load) */
  BRE_ERR_UNSUPPORTED = -4  /* feature not implemented by the engine (never silently falls back) */
};

/* ---- layer program (produced by breaching_b200.compiler from the nn.Module) ---------------------- */
enum bre_op_kind { BRE_OP_CONV = 1, BRE_OP_BNACT = 2, BRE_OP_MAXPOOL = 3, BRE_OP_AVGPOOL = 4, BRE_OP_LINEAR = 5,
                   /* token-sequence programs (transformer / TAG path): tensors are [rows = batch * seq_len, C, 1, 1] */
                   BRE_OP_POSADD = 6,      /* out = candidate + positional embedding `w` of position (row mod seq_len) */
                   BRE_OP_LAYERNORM = 7,   /* gamma, beta, eps */
                   BRE_OP_ATTENTION = 8,   /* tin = fused (q | k | v) projection, R = heads, S = seq_len, no mask */
                   BRE_OP_POSCONST = 9 };  /* out = candidate + constant table [S, C] of position (row mod S), w = -1: the fixed
                                              sinusoidal positions (no parameter; table from bre_engine_load_constant) */
enum bre_param_perm { BRE_PERM_NONE = 0, BRE_PERM_OIHW_TO_OHWI = 1, BRE_PERM_LINEAR_CHW_TO_HWC = 2 };

typedef struct bre_tensor_desc { int32_t N, C, H, W; } bre_tensor_desc; /* tensor 0 = candidate (NCHW) */

typedef struct bre_param_desc {
  int64_t numel;
  int32_t perm;          /* bre_param_perm: engine-internal layout of this tensor */
  int32_t d0, d1, d2;    /* OIHW->OHWI: d0=O, d1=I, d2=H*W ; LINEAR: d0=out, d1=C, d2=H*W ; NONE: d0 = elements to reserve if > numel
                            (zero tail, e.g. the rows of a vocabulary padded to the GEMM tile width; see option "logits_valid") */
} bre_param_desc;

typedef struct bre_op_desc {
  int32_t kind;
  int32_t tin, tout, res;         /* tensor ids (res = -1 if none) */
  int32_t R, S, stride, pad;      /* conv / maxpool geometry */
  int32_t w, b;                   /* parameter indices in model.parameters() order, -1 = none */
  int32_t has_bn, relu;           /* BNACT: out = relu?( bn?(in) + res? ) */
  int32_t gamma, beta;            /* parameter indices of BN weight / bias */
  int32_t bn_buffer;              /* index into the running-stat arrays passed to bre_engine_load_model */
  float eps;
  int32_t acc_in, acc_res;        /* reverse sweeps: accumulate into (1) or overwrite (0) the input delta */
  int32_t bn_train;               /* BNACT: BN uses the batch statistics of its input (model in train mode without buffers,
                                     base_attack.py:192-197) instead of running statistics */
} bre_op_desc;

/* ---- attack configuration (cfg_attack of the reference, flattened) ------------------------------- */
enum bre_objective {              /* objectives.py:496-506 objective_lookup */
  BRE_OBJ_EUCLIDEAN = 0, BRE_OBJ_COSINE = 1, BRE_OBJ_L1 = 2, BRE_OBJ_TAG_EUCLIDEAN = 3,
  BRE_OBJ_ANGULAR = 4, BRE_OBJ_FAST_COSINE = 5, BRE_OBJ_MASKED_COSINE = 6
};
enum bre_optimizer { BRE_OPT_ADAM = 0, BRE_OPT_ADAMW = 1, BRE_OPT_SGD = 2 }; /* common.py:6-17 */
enum bre_sign { BRE_SIGN_NONE = 0, BRE_SIGN_HARD = 1, BRE_SIGN_SOFT = 2 };  /* optimization_based_attack.py:175-184 */

typedef struct bre_attack_cfg {
  int32_t objective;              /* bre_objective */
  float obj_scale, task_regularization, tag_scale, mask_value, angular_fudge;
  int32_t optimizer;              /* bre_optimizer */
  float beta1, beta2, adam_eps, weight_decay, momentum;
  int32_t nesterov;
  int32_t signed_mode;            /* bre_sign */
  int32_t boxed;                  /* optimization_based_attack.py:117-118 */
  int32_t max_iterations;         /* cfg.optim.max_iterations (soft-sign schedule + LR table length) */
  float langevin_noise;           /* :167-170 */
  float grad_clip;                /* :171-174 ; < 0 = disabled */
  uint64_t noise_seed;            /* Philox key of the Langevin noise; the counter is (element, iteration, trial index) */
  /* regularizers.py -- a scale of 0 disables the term */
  float tv_scale, tv_inner_exp, tv_outer_exp, tv_eps; int32_t tv_double_opponents;
  float norm_scale, norm_p;
  float di_scale, di_first_bn_multiplier;
  float feat_scale;
  int32_t orthogonality;          /* regularizers.py:156-181 (the reference ignores its `scale`; != 0 enables the term) */
  int32_t objective_excludes_task;/* Pearlmutter* objectives (objectives.py:279-365, 468-493): task_regularization enters the
                                     candidate gradient (:362) but not the reported objective value */
} bre_attack_cfg;

/* ---- engine life cycle -------------------------------------------------------------------------- */
/* Build an engine for one model replica on `device`.  Replaces the per-trial set-up of _run_trial
 * (optimization_based_attack.py:93-107). */
int bre_engine_create(const bre_tensor_desc* tensors, int32_t n_tensors,
                      const bre_op_desc* ops, int32_t n_ops,
                      const bre_param_desc* params, int32_t n_params,
                      int32_t logits_tensor, const bre_attack_cfg* cfg, int32_t device, bre_engine** out);
void bre_engine_destroy(bre_engine* e);

/* Model state of the attacked network as the server payload holds it (base_attack.py:169-212):
 * `params[i]` = pointer to parameter i (model.parameters() order, torch-contiguous, fp32),
 * `bn_mean[j]` / `bn_var[j]` = running statistics of BN layer j (order of bre_op_desc.bn_buffer).
 * Pointers: device or host. */
int bre_engine_load_model(bre_engine* e, const float* const* params, int32_t n_params,
                          const float* const* bn_mean, const float* const* bn_var, int32_t n_bn);
/* The constant table of op `op` (a BRE_OP_POSCONST op: [S, C] fp32, numel = S * C; device or host), a buffer of the model such as
 * the reference's PositionalEmbedding.pe[0, :S].  Every such op needs its table before the first evaluation. */
int bre_engine_load_constant(bre_engine* e, int32_t op, const float* table, int64_t numel);

/* The user's shared gradient (shared_data[i]["gradients"], users.py:176-186), same order/layout as params,
 * per-tensor TAG weights (objectives.py:115-124; NULL = all ones), labels (int64, [N]),
 * normalisation box (base_attack.py:53-57): mean/std per input channel (NULL = 0/1).
 * Pointers: device or host. */
int bre_engine_load_targets(bre_engine* e, const float* const* grads, int32_t n_params,
                            const float* tensor_weights, const int64_t* labels, int32_t n_labels,
                            const float* mean, const float* std, int32_t n_channels);

/* FedAvg / multi-step local updates (objectives.py:48-72, users.py:336-413): the user ran `steps` SGD steps of size `lr`,
 * step k on the candidate slice [k*B mod total_images, ... + B) (B = batch of the layer program) with labels
 * labels[k*B .. (k+1)*B); the matched quantity becomes W_K - W_0.  Re-sizes the candidate state to `total_images`.
 * task_regularization and DeepInversion read the last local step (its task loss at W_{K-1}, the BN-input statistics of its
 * forward) and need lr != 0 (their adjoints seed that step's tangent backward scaled by -1/lr); the feature prior, train-mode
 * BatchNorm and lr == 0 with a prior are refused with BRE_ERR_UNSUPPORTED.
 * Call after bre_engine_load_model / load_targets and before bre_engine_begin_trial.  labels: device or host. */
int bre_engine_set_local_steps(bre_engine* e, int32_t total_images, int32_t steps, float lr, const int64_t* labels);

/* Joint data / label optimisation (OptimizationJointAttacker, optimization_with_label_attack.py:145-189): the closure hands
 * `labels.softmax(dim=-1)` to the loss as class probabilities (:154).  `probabilities` [N, classes] fp32 (device or host)
 * replaces the index labels in the task loss until cleared with NULL.  After bre_engine_objective_and_gradient,
 * bre_engine_label_gradient writes d(objective)/d(probabilities) [N, classes] (the caller chains it through its softmax,
 * as autograd does for the reference at :162).  bre_engine_set_labels replaces the index labels (scoring with
 * `labels.argmax`, :67-70). */
int bre_engine_load_soft_labels(bre_engine* e, const float* probabilities, int64_t numel);
int bre_engine_label_gradient(bre_engine* e, float* grad_out);
int bre_engine_set_labels(bre_engine* e, const int64_t* labels, int32_t n_labels);

/* Measured features for the `features` regulariser (regularizers.py:31-43): [N, F] fp32, device or host. */
int bre_engine_load_feature_targets(bre_engine* e, const float* measured, int64_t numel);

/* Start a trial: candidate [N,C,H,W] fp32 (device or host), LR table of length n_lr (host; entry `it` is
 * the step size used by optimiser step `it`, common.py:19-38).  Resets Adam state, best-so-far, history. */
int bre_engine_begin_trial(bre_engine* e, const float* candidate, const float* lr_table, int32_t n_lr);
/* Global index (>= 0, default 0) of the trials begun after this call.  The Langevin noise of element i in iteration `it` is drawn
 * from Philox(noise_seed; i, it, trial index), so restarts on one engine -- and the trials that the ranks of a multi-GPU run take
 * from one shared list -- get independent noise fields, as the reference's per-step randn_like gives them, when each is begun under
 * its own index; the same (seed, index) replays the same field. */
int bre_engine_set_trial_index(bre_engine* e, int32_t trial);

/* Enqueue `n_iters` iterations of optimization_based_attack.py:110-138 (closure + step + projection +
 * best-so-far + history) on the engine's stream; returns without waiting. */
int bre_engine_run(bre_engine* e, int32_t n_iters);
int bre_engine_sync(bre_engine* e);
/* Same as bre_engine_run + bre_engine_sync, bracketed by CUDA events on the engine's stream: *ms_out = device time. */
int bre_engine_run_timed(bre_engine* e, int32_t n_iters, float* ms_out);

/* After sync: iterations recorded in the history (== len(stats["Trial_k_Val"])), whether a non-finite
 * objective stopped the trial (:131-133), minimal objective so far and last task loss. */
int bre_engine_status(bre_engine* e, int32_t* iters_recorded, int32_t* stopped, double* min_objective,
                      double* last_task_loss);
int bre_engine_read_history(bre_engine* e, float* out_host, int32_t n);
/* Copy best / current candidate ([N,C,H,W] fp32) to `out` (device or host). */
int bre_engine_get_best(bre_engine* e, float* out);
int bre_engine_get_candidate(bre_engine* e, float* out);

/* _score_trial (optimization_based_attack.py:191-204): objective `scoring` (bre_objective: euclidean or
 * cosine, scale 1) of `candidate`; non-finite is reported as +inf. */
int bre_engine_score(bre_engine* e, const float* candidate, int32_t scoring, double* out_score);

/* ---- evaluation without an optimiser step (used by tests and by label/feature tooling) ----------- */
/* Runs the four sweeps + regularisers for `candidate` and returns the total objective and
 * d objective / d candidate (unprocessed, i.e. before noise / clip / sign) into grad_out (device or host). */
int bre_engine_objective_and_gradient(bre_engine* e, const float* candidate, double* objective, float* grad_out);
/* Objective terms of the last evaluation: match, task loss, tv, norm, deep inversion, features. */
int bre_engine_last_terms(bre_engine* e, double* terms6);
/* Debug access (tests): parameter-gradient list G / direction v in torch layout for parameter `index`;
 * which: 0 = G, 1 = v, 2 = W, 3 = g, 4 = v as the GEMMs read it, 5 = W as the GEMMs read it.  out: host, numel floats.
 * On the tensor-core back end the single-step direction of the weights of tensor-core layers is written to its TF32 shadow
 * only, so which = 1 returns stale memory for them; which = 4 / 5 return the TF32 shadow for those weights and the fp32
 * arena for every other parameter. */
int bre_engine_debug_param(bre_engine* e, int32_t which, int32_t index, float* out_host);
/* Multi-step engines: the local weights W_k of step `step` (0..K), torch layout like bre_engine_debug_param; which: 0 = W_k (fp32),
 * 1 = W_k as the GEMMs read it (its TF32 shadow for the weights of tensor-core layers), 2 = D = W_K - W_0 as accumulated
 * (`step` ignored).  W_0 is always valid.  W_{k+1}, its shadow and D_{k+1} are written by step k's update: valid after a full
 * evaluation, or after one stopped at debug_multistep_stop >= k + 1 (for D: exactly k + 1, or any reverse stop for D_K).
 *
 * Option "debug_multistep_stop" (bre_engine_set_option, default 0 = off) stops bre_engine_objective_and_gradient inside a
 * multi-step evaluation.  s = k + 1 (1 <= s <= K): after step k's forward and backward sweeps and its W_{k+1} / D updates;
 * step k stays bound: activations, deltas, probabilities, labels, W = W_k and G = G_k (bre_engine_debug_tensor / debug_param).
 * s = K + 1 + k: after step k's tangent-forward and tangent-backward sweeps, before its candidate-gradient axpy and adjoint
 * update; v and its TF32 shadow hold the direction u_{k+1} that step k used, G holds the tangent weight gradient H_k u_{k+1}
 * (k > 0 only) and the tangent delta of tensor 0 is the step's input gradient.  At the stop after the last step (s = 2K) the
 * prior seeds are in place: the logits tangent delta holds the cross-entropy tangent plus -tau/lr (p - y)/N (tau =
 * task_regularization), every BN input's tangent delta holds its DeepInversion adjoint scaled by -1/lr, and G and the step's input
 * gradient carry those seeds through the sweep.  The value and gradient returned by a stopped evaluation are not meaningful.
 * bre_engine_run refuses while a stop is set. */
int bre_engine_debug_step_param(bre_engine* e, int32_t which, int32_t step, int32_t index, float* out_host);
/* which: 0 = activation, 1 = delta (sweep B), 2 = tangent, 3 = tangent delta; NCHW fp32 to host.  Tensor 0 (the candidate)
 * has no tangent; its delta is the task-loss gradient and its tangent delta the candidate gradient.  With fuse_bnact, the
 * tangent of a conv output whose only consumer is the BN op fused into the conv's epilogue is not written in single-step
 * evaluations (it holds whatever an earlier evaluation left). */
int bre_engine_debug_tensor(bre_engine* e, int32_t which, int32_t tensor, float* out_host);
/* Candidate-side buffers of the optimiser step as the last iteration left them (tests), to host: which 0 = the candidate gradient
 * the step read (before noise / clip / sign), 1 = the separate task-loss gradient (BRE_ERR_STATE when the step reads none: no
 * task_regularization, or already folded into 0), 2 / 3 = the optimiser moments m / v (SGD: m = momentum buffer); candidate-shaped.
 * 4 / 5 / 6 = gradient, m, v of the label-logit leaf of a joint trial ([N, classes]); 7 = the soft targets q = softmax(label logits)
 * that the last joint iteration handed to the evaluation ([N, classes]). */
int bre_engine_debug_step_state(bre_engine* e, int32_t which, float* out_host);
/* What the engine did with op `op` (tests): bit 0 = it ran in the epilogue of the preceding tensor-core GEMM in the last forward
 * sweep (fuse_bnact), bit 1 = its input tangent was not stored in the last tangent-forward sweep (that fused case), bit 2 = the
 * op runs on the column path of the candidate-fed convolution, which rounds the candidate, weight and direction to TF32 itself. */
int bre_engine_debug_op(bre_engine* e, int32_t op, int32_t* flags);
/* Number of kernel launches per iteration (for gpu_launches in bench.py) and whether graphs are used. */
int bre_engine_launches_per_iteration(bre_engine* e, int32_t* out);
int bre_engine_set_option(bre_engine* e, const char* name, int64_t value);

/* Joint data + label optimisation on the device (OptimizationJointAttacker._run_trial, optimization_with_label_attack.py:89-143;
 * closure :145-189): like bre_engine_begin_trial, plus the label-logit leaf [N, classes] (rows = batch * seq_len for token
 * models).  Every bre_engine_run iteration then evaluates softmax(labels) as the soft targets of the task loss, the objective,
 * both gradients (candidate and label logits, post-processed separately), steps both leaves with the configured optimiser,
 * projects the candidate only, and keeps the best-so-far pair.  Pointers: device or host. */
int bre_engine_begin_joint_trial(bre_engine* e, const float* candidate, const float* label_logits, int64_t n_label_elems,
                                 const float* lr_table, int32_t n_lr);
/* Label logits of the joint trial: best != 0 -> the best-so-far copy, else the current iterate. */
int bre_engine_get_joint_labels(bre_engine* e, int32_t best, float* out);

/* Candidate augmentations of the closure (optimization_based_attack.py:149-153, auxiliaries/augmentations.py): the model and the
 * priors see view(candidate); `differentiable` != 0 pulls the gradient back through the transposed view, 0 replaces the candidate
 * by its view every iteration (the reference assigns candidate.data).  Pipeline: up to 4 permutation steps in config order
 * (kinds[s]: 1 = discrete_shift with params[s] = lim, 2 = flip with params[s] = p), then the optional continuous_shift
 * (bilinear grid sample, shift in pixels, "circular" wrap as in the reference), then the composite colour affine per (image,
 * channel): out = in * cj_scale + cj_shift (colorjitter; NULL = none; device or host [N * C]).  Random draws: Philox(seed,
 * iteration).  n_steps = 0, cs_enabled = 0 and cj_scale = NULL switch augmentations off. */
int bre_engine_set_augmentations(bre_engine* e, int32_t n_steps, const int32_t* kinds, const float* params, int32_t cs_enabled,
                                 float cs_shift, int32_t cs_circular, const float* cj_scale, const float* cj_shift,
                                 int32_t differentiable, uint64_t seed);
/* The draws of the last evaluation (for parity tests): roll offsets / flip flags per step, continuous-shift uniforms per image. */
int bre_engine_last_augmentation(bre_engine* e, int32_t* o1, int32_t* o2, float* sx, float* sy);
/* Stand-alone view (transpose = 0) or pull-back (transpose = 1: x is the gradient w.r.t. the view and is clobbered when the
 * continuous shift is on; scratch: same size) with explicit draws o1 / o2 per step and sx / sy per image (NULL = no continuous shift). */
int bre_augment_view(const float* x, float* out, int32_t N, int32_t C, int32_t H, int32_t W, int32_t n_steps, const int32_t* kinds,
                     const int32_t* o1, const int32_t* o2, float cs_shift, int32_t cs_circular, const float* sx, const float* sy,
                     const float* cj_scale, const float* cj_shift, int32_t transpose, float* scratch, void* stream);
/* continuous_shift with every option of the reference's RandomTransform (the entry points above sample bilinearly with zeros
 * padding, or "circular" = cs_circular, without grid flips): grid_sample mode cs_mode and padding_mode cs_padding (cs_circular
 * needs BRE_CS_ZEROS), and per-image grid flips: fliplr[n] / flipud[n] != 0 negates image n's x / y coordinate (NULL = none).
 * Sides up to 1024. */
enum { BRE_CS_BILINEAR = 0, BRE_CS_NEAREST = 1, BRE_CS_BICUBIC = 2 };
enum { BRE_CS_ZEROS = 0, BRE_CS_BORDER = 1, BRE_CS_REFLECTION = 2 };
int bre_engine_set_augmentations_ex(bre_engine* e, int32_t n_steps, const int32_t* kinds, const float* params, int32_t cs_enabled,
                                    float cs_shift, int32_t cs_circular, int32_t cs_mode, int32_t cs_padding, int32_t cs_fliplr,
                                    int32_t cs_flipud, const float* cj_scale, const float* cj_shift, int32_t differentiable, uint64_t seed);
int bre_augment_view_ex(const float* x, float* out, int32_t N, int32_t C, int32_t H, int32_t W, int32_t n_steps, const int32_t* kinds,
                        const int32_t* o1, const int32_t* o2, float cs_shift, int32_t cs_circular, int32_t cs_mode, int32_t cs_padding,
                        const float* sx, const float* sy, const int32_t* fliplr, const int32_t* flipud, const float* cj_scale,
                        const float* cj_shift, int32_t transpose, float* scratch, void* stream);

/* The view as an ordered list of up to 8 stages, each with its own input and output shape (augment.cu):
 *   BRE_AUG_PIXEL     a run of the shape-keeping kinds with the parameters of bre_engine_set_augmentations (n_steps, kinds,
 *                     params, cs_*, cj_scale / cj_shift [N * C], device or host, NULL = no colour);
 *   BRE_AUG_RESAMPLE  the window [y0, y0 + wh) x [x0, x0 + ww) resized bilinearly to Ho x Wo (F.interpolate, bilinear,
 *                     align_corners = False): zoom (window = input), centerzoom (fixed corner), focus (focus != 0: the corner is drawn
 *                     every evaluation as clamp(trunc(pert + in // 2 - size // 2), 0, in - size), pert uniform in [-focus_std, focus_std));
 *   BRE_AUG_BLUR      antialias: depthwise binomial filter of `width` (1..7), zero padding width // 2, `stride`.
 * The candidate is [N, C, H, W]; the last stage's output must be program tensor 0 (the model runs on the view).  The candidate-side
 * state (x, optimiser moments, best, box, candidate gradient) takes the candidate's shape.  A stage list that changes the shape needs
 * differentiable != 0.  n_stages = 0 switches augmentations off and restores the program's shape. */
enum { BRE_AUG_PIXEL = 0, BRE_AUG_RESAMPLE = 1, BRE_AUG_BLUR = 2 };
typedef struct bre_aug_stage {
  int32_t kind;
  int32_t n_steps, kinds[4];
  float params[4];
  int32_t cs_enabled, cs_circular;
  float cs_shift;
  const float* cj_scale;
  const float* cj_shift;
  int32_t y0, x0, wh, ww, Ho, Wo, focus;
  float focus_std;
  int32_t width, stride;
} bre_aug_stage;
int bre_engine_set_augmentation_stages(bre_engine* e, int32_t n_stages, const bre_aug_stage* stages, int32_t N, int32_t C, int32_t H,
                                       int32_t W, int32_t differentiable, uint64_t seed);
/* The same with the continuous_shift options of bre_engine_set_augmentations_ex per PIXEL stage (cs_fliplr / cs_flipud != 0: each
 * image's grid is flipped when its third / fourth uniform is > 0.5). */
typedef struct bre_aug_stage_ex {
  bre_aug_stage stage;
  int32_t cs_mode, cs_padding, cs_fliplr, cs_flipud;
} bre_aug_stage_ex;
int bre_engine_set_augmentation_stages_ex(bre_engine* e, int32_t n_stages, const bre_aug_stage_ex* stages, int32_t N, int32_t C, int32_t H,
                                          int32_t W, int32_t differentiable, uint64_t seed);
/* All draws of the last evaluation, per stage k (8 x 4 offsets, 8 x 64 uniforms): PIXEL stages as bre_engine_last_augmentation,
 * focus stages their window corner (o1[4 k], o2[4 k]) = (row, column). */
int bre_engine_augmentation_draws(bre_engine* e, int32_t* n_stages, int32_t* o1, int32_t* o2, float* sx, float* sy);
/* The grid flips of the last evaluation, per stage k and image n (8 x 64): fliplr[64 k + n], flipud[64 k + n] = 1 when image n's grid
 * was flipped (0 for stages without flips). */
int bre_engine_augmentation_flips(bre_engine* e, int32_t* n_stages, int32_t* fliplr, int32_t* flipud);
/* Stand-alone RESAMPLE / BLUR stage with an explicit window: transpose = 0 maps x [N, C, Hi, Wi] to the view, transpose = 1 pulls
 * x = the gradient at the view back to out [N, C, Hi, Wi] (fixed-order gathers, bitwise reproducible). */
int bre_augment_resample(const float* x, float* out, int32_t N, int32_t C, int32_t Hi, int32_t Wi, int32_t y0, int32_t x0, int32_t wh,
                         int32_t ww, int32_t Ho, int32_t Wo, int32_t transpose, void* stream);
int bre_augment_blur(const float* x, float* out, int32_t N, int32_t C, int32_t Hi, int32_t Wi, int32_t width, int32_t stride,
                     int32_t transpose, void* stream);

/* ---- the steps either side of the hot path (SURVEY.md section 8 f-2, f-3) ----------------------------------------- */
/* User-side update production (cases/users.py:148-169 `_compute_batch_gradient`): one forward + backward of the loaded model
 * on `data` (candidate layout, device or host) with index `labels` -> gradient of the mean task loss w.r.t. every parameter,
 * written to grads_out[i] (model.parameters() order, torch layout, device or host); loss_out (host, may be NULL) = task loss. */
int bre_engine_param_gradients(bre_engine* e, const float* data, const int64_t* labels, int32_t n_labels,
                               float* const* grads_out, int32_t n_params, double* loss_out);
/* Train-mode BN (user without public buffers, users.py:140-143): batch mean and *biased* variance that layer `bn_index` saw in
 * the last forward, from which the user's shipped buffers follow (momentum None: running_mean = mean, running_var = unbiased). */
int bre_engine_bn_batch_stats(bre_engine* e, int32_t bn_index, float* mean_out, float* var_out);
/* Model forward only (analysis/analysis.py:66-69 feature comparison): logits [N, classes] (device or host). */
int bre_engine_forward(bre_engine* e, const float* data, float* logits_out);
/* Per-example mean squared error between the de-normalised ([x * std + mean], per channel; NULL = identity), optionally
 * [0,1]-clamped reconstruction and ground truth (analysis/analysis.py:228-242); PSNR per example = 10 log10(1 / mse)
 * (analysis/metrics.py:108-130) follows on the host.  rec, ref: device fp32 [N, C, HW]; mean / std: host [C]; mse: host [N]. */
int bre_image_mse(const float* rec, const float* ref, int32_t N, int32_t C, int32_t HW, const float* mean, const float* std,
                  int32_t clamp01, double* mse_host, void* stream);

/* Bilinear resize of an NCHW fp32 batch on the device, F.interpolate(mode="bilinear", align_corners=False) semantics: the
 * stage-to-stage up-sampling of MultiScaleOptimizationAttacker (multiscale_optimization_attack.py:45-69). */
int bre_resize_bilinear(const float* src, float* dst, int32_t N, int32_t C, int32_t Hi, int32_t Wi, int32_t Ho, int32_t Wo, void* stream);

/* ---- stand-alone kernels (each is also a stage of the engine; exposed for parity tests + rooflines) */
/* Multi-tensor gradient-matching reduction (objectives.py:91-95,135-141,160-164,185-196).
 * G, g: device fp32 [n]; chunk_weights: device fp32 [ceil(n/1024)] or NULL.  sums5 (host, double):
 * <G,g>, |G|^2, |g|^2, sum (G-g)^2, sum w |G-g|; NULL = launch only, no read-back (for timing the bare kernel).  */
int bre_match_reduce(const float* G, const float* g, const float* chunk_weights, int64_t n, float mask_value,
                     double* sums5_host, void* stream);
/* TotalVariation value + gradient (regularizers.py:130-147) for x [N,3,H,W] device fp32;
 * grad (device) is overwritten when accumulate == 0. */
int bre_total_variation(const float* x, float* grad, int32_t N, int32_t H, int32_t W, float scale, float inner_exp,
                        float outer_exp, float eps, int32_t double_opponents, int32_t accumulate,
                        double* value_host, void* stream);
/* The tail of one iteration, alone: gradient post-processing (task term, Langevin noise, clip by the global norm, sign),
 * Adam / AdamW / SGD update, box projection, best-so-far and the trial bookkeeping (optimization_based_attack.py:112-135,166-184)
 * -- the grad-norm (when cfg->grad_clip >= 0), step and commit launches that bre_engine_run enqueues after the four sweeps -- on
 * caller-owned device buffers.  x, m, v, best, grad: [n] fp32, n = images * C * HW; grad_task: [n] or NULL (added times
 * cfg->task_regularization); lr_table [n_lr]: iterations >= n_lr step with 0; lo / hi [C]: box of channel (i / HW) % C, read only
 * when cfg->boxed; history [max_hist]: entry `recorded` is written while recorded < max_hist.  `io` (host) carries the scalar
 * state in and out; the call waits for the stream. */
typedef struct bre_step_scalars {
  double match, task_loss, tv, norm, di, feat; /* in: objective pieces; phi = their sum with task_loss times task_regularization
                                                  (times 0 when cfg->objective_excludes_task) */
  double fmin;                                 /* in / out: minimal objective so far (+inf at the start of a trial) */
  int32_t it, recorded, stopped, trial;        /* in / out (trial: in): 0-based index of this step, history length, stop flag */
  double grad_norm_sq, last_objective;         /* out: squared norm of the noised gradient (clip only), float(phi) */
} bre_step_scalars;
int bre_optimizer_step(float* x, float* m, float* v, float* best, const float* grad, const float* grad_task, const float* lr_table,
                       int32_t n_lr, const float* lo, const float* hi, int64_t n, int32_t C, int32_t HW, const bre_attack_cfg* cfg,
                       float* history, int32_t max_hist, bre_step_scalars* io, void* stream);
/* out[i] (device, i < n) = the standard normal draw of element first + i in iteration `it` of trial `trial` under `seed`: what the
 * step adds to that element's gradient, divided by langevin_noise * lr.  Same device function as the step kernels. */
int bre_langevin_noise(uint64_t seed, uint32_t trial, uint32_t it, uint64_t first, int64_t n, float* out, void* stream);
/* Token-sequence ops of the transformer / TAG path (language_models.py:150-205 as attacked in embedding space; SURVEY
 * section 8 rows a15 / a16), stand-alone, one call per sweep (0 forward, 1 backward, 2 tangent-forward, 3 tangent-backward;
 * rules in oracle/transformer_interp.py).  fp32 device pointers, [rows, C] row-major, rows = batch * seq_len.
 *   layernorm: x = the op's input; in1..in3 per sweep: (1) dy | (2) x' | (3) dy', dy, x'; stats [rows, 2] is written by
 *              sweep 0 and read by the others; sweep 1 also writes g_gamma / g_beta when non-NULL.
 *   attention: qkv [rows, 3 d] = (q | k | v) projections, heads x dh = d, no mask; in1..in3 per sweep: (1) dO [rows, d] |
 *              (2) (qkv)' | (3) dO', dO, (qkv)'; P / Pd [B, heads, T, T] are written by sweeps 0 / 2 and read later.
 * round_out != 0 stores `out` on the TF32 grid (cvt.rna), as the engine does for the operands of tensor-core GEMMs.  The attention
 * sweeps keep a whole head in one CTA's shared memory when 8 T dh + 4 T^2 floats fit in 200 KB; a wider head is split by columns
 * over the smallest thread-block cluster of c <= 8 CTAs whose slices fit (8 T (ceil(dh / c) | 1) + 6 T^2 floats per CTA, the
 * contractions over dh reduced through distributed shared memory in rank order); otherwise the call fails (-4). */
int bre_token_layernorm(int32_t sweep, const float* x, const float* in1, const float* in2, const float* in3, const float* gamma,
                        const float* beta, const float* v_gamma, const float* v_beta, float eps, int32_t rows, int32_t C, float* stats,
                        float* out, float* g_gamma, float* g_beta, int32_t round_out, void* stream);
int bre_token_attention(int32_t sweep, const float* qkv, const float* in1, const float* in2, const float* in3, int32_t B, int32_t T,
                        int32_t heads, int32_t dh, float* P, float* Pd, float* out, int32_t round_out, void* stream);
/* The attention sweeps with the kernel chosen by the caller: cluster = 0 picks as bre_token_attention does, 1 = the resident-head
 * kernel, 2 .. 8 = the head split over that many CTAs (the last takes the remainder of dh); -4 when that kernel does not fit. */
int bre_token_attention_ex(int32_t sweep, const float* qkv, const float* in1, const float* in2, const float* in3, int32_t B, int32_t T,
                           int32_t heads, int32_t dh, float* P, float* Pd, float* out, int32_t round_out, void* stream, int32_t cluster);
/* Host only: *ctas = the CTAs per (sequence, head) that bre_token_attention_ex(.., cluster) runs with (1 = resident), -1 = refused. */
int bre_token_attention_plan(int32_t T, int32_t dh, int32_t cluster, int32_t* ctas);

/* Token recovery of the text attacks (replaces `_postprocess_text_data._max_similarity`, breaching/attacks/base_attack.py:126-133):
 * tokens[n] = argmax_v <r_n - mean, e_v - mean> / |r_n - mean|^2 / |e_v - mean|^2 over the V rows of emb [*, d] (rows picked through
 * `subset` [V] when non-NULL; ids are then positions in that list).  rec [rows, d], tokens [rows] int64; device pointers. */
int bre_token_match(const float* rec, const float* emb, const int64_t* subset, int32_t rows, int32_t d, int32_t V, int64_t* tokens,
                    void* stream);

/* Implicit-GEMM convolution family, NHWC activations / OHWI weights, fp32:
 * mode 0 fprop  : out[N,Ho,Wo,Co]  = conv(in[N,H,W,Ci], w[Co,R,S,Ci]) (+ conv(in2, w2) when in2 != NULL)
 * mode 1 dgrad  : din[N,H,W,Ci]    = conv^T(dout[N,Ho,Wo,Co], w) (+ conv^T(dout2, w2))
 * mode 2 wgrad  : dw[Co,R,S,Ci]    = sum_pixels dout (x) in
 * backend 0 = SIMT fp32, 1 = TF32 tensor cores (where available, else BRE_ERR_UNSUPPORTED), 2 = the engine's dispatch
 * (tensor cores where the shape is covered, SIMT otherwise). */
int bre_conv_gemm(int32_t mode, int32_t backend, const float* a, const float* w, const float* a2, const float* w2,
                  float* out, int32_t N, int32_t H, int32_t W, int32_t Ci, int32_t Co, int32_t R, int32_t S,
                  int32_t stride, int32_t pad, void* stream);
/* The launch plan of the last GEMM issued by the calling host thread (any entry point: bre_conv_gemm or the engine), host-side
 * bookkeeping only.  out[11] = family (-1 none yet, 0 SIMT implicit GEMM, 1 dgrad_small_ci, 2 linear_small, 3 linear_tall, 4 tensor
 * core), mode, nsrc, tile rows, tile width, splits (grid z; linear_tall: reduction chunks), ring depth, producer (0 none, 1 TMA,
 * 2 cp.async, 3 TMA per parity class), total k-blocks, k-blocks per split (32-wide on the tensor cores, 16-wide on SIMT), vector
 * flags (SIMT: bit 0 A loads, bit 1 B loads, bit 2 stores; dgrad_small_ci / linear_small fprop: vector loads). */
int bre_debug_last_gemm_plan(int32_t* out);
/* The launch plan bre_conv_gemm would run for this contraction with nsrc sources (1 or 2) on `backend`, in the 11 fields of
 * bre_debug_last_gemm_plan (family -1: backend 1 does not cover the shape).  Assumes bre_conv_gemm's operands (NHWC / OHWI,
 * 16-byte aligned) and its 1024-tile workspace.  Host only: allocates, encodes and launches nothing. */
int bre_gemm_plan(int32_t mode, int32_t backend, int32_t N, int32_t H, int32_t W, int32_t Ci, int32_t Co, int32_t R, int32_t S,
                  int32_t stride, int32_t pad, int32_t nsrc, int32_t* out);
/* The plan of the cluster row kernels (row softmax, softmax chain, token cross-entropy, its tangent, token label gradient) for rows
 * of C elements: *cs = CTAs per row (1, 2, 4 or 8), *fits = 1 when each CTA's segment is cached in registers, 0 when it is streamed. */
int bre_debug_row_plan(int32_t C, int32_t* cs, int32_t* fits);
/* The row kernels of the label leaf and of the cross-entropy seeds, stand-alone through the engine's own launchers (parity tests).
 * fp32 device pointers; rows >= 1, 1 <= C <= Vs; logits-shaped buffers of the token ops have row stride Vs, every other buffer
 * row stride C (the other ops need Vs == C).  T: sequence length of the token ops (rows % T == 0); labels: int64 class indices
 * in [0, C) (not checked).
 *   BRE_ROW_SOFTMAX          out0 [rows, C] = softmax(in0) per row
 *   BRE_ROW_SOFTMAX_CHAIN    out0 [rows, C] <- in0 * (out0 - <in0, out0>) per row (in place; in0 = q)
 *   BRE_ROW_TOKEN_CE_FWD     in0 = logits, in1 = soft targets [rows, C]; out0 = p, out1 = loss per row [rows], out2 = dlogits
 *   BRE_ROW_TOKEN_CE_TAN_BWD in0 = p, in1 = logits tangent; out0 = tangent dlogits
 *   BRE_ROW_TOKEN_LABEL_GRAD in0 = logits, in1 = p, in2 = logits tangent, coef = task_regularization; out0 [rows, C]
 *   BRE_ROW_CE_FWD           in0 = logits, labels or in1 = soft targets; out0 = p, out1 = loss per row, out2 = dlogits
 *   BRE_ROW_CE_LABEL_GRAD    in0 = logits, in1 = p, in2 = logits tangent, coef = task_regularization; out0
 *   BRE_ROW_CE_TAN_BWD       in0 = p, in1 = logits tangent; out0 = tangent dlogits; with labels: plus coef (p - onehot) / rows
 * round_out != 0 stores dlogits / tangent dlogits on the TF32 grid (token ops and the labelled tangent only). */
enum { BRE_ROW_SOFTMAX = 0, BRE_ROW_SOFTMAX_CHAIN = 1, BRE_ROW_TOKEN_CE_FWD = 2, BRE_ROW_TOKEN_CE_TAN_BWD = 3, BRE_ROW_TOKEN_LABEL_GRAD = 4,
       BRE_ROW_CE_FWD = 5, BRE_ROW_CE_LABEL_GRAD = 6, BRE_ROW_CE_TAN_BWD = 7 };
int bre_row_op(int32_t op, const float* in0, const float* in1, const float* in2, const int64_t* labels, int32_t rows, int32_t C, int32_t Vs,
               int32_t T, float coef, int32_t round_out, float* out0, float* out1, float* out2, void* stream);

/* ---- L-BFGS on the device (torch.optim.LBFGS without line search; breaching/attacks/auxiliaries/common.py:18) ------------- */
/* torch's constants, passed in by the caller (breaching_b200/attacks/lbfgs.py holds them): max_iter inner iterations and max_eval
 * closure evaluations per optimizer.step, `history` curvature pairs (<= BRE_LBFGS_MAX_HISTORY), tolerance_grad, tolerance_change and
 * the curvature threshold a pair must pass (y.s > curvature_min). */
enum { BRE_LBFGS_MAX_HISTORY = 128 };
typedef struct bre_lbfgs_consts {
  int32_t max_iter, max_eval, history, reserved;
  double tol_grad, tol_change, curvature_min;
} bre_lbfgs_consts;
/* Scalar state of one optimiser (device memory).  The ring has history + 1 slots: live pairs are slots (first + k) % (history + 1),
 * k < count, oldest first; a candidate pair is written to the one spare slot and becomes live only if it passes the curvature test. */
typedef struct bre_lbfgs_scalars {
  double h_diag, t, loss, prev_loss, first_loss, gtd, d_max, g_max, g_abs_sum, ys;
  double first_terms[6];   /* objective terms of the first closure of the step (match, task_loss, tv, norm, di, feat) */
  int32_t first, count, total_iters, inner, evals, func_evals, brk, converged, pushed, reserved;
} bre_lbfgs_scalars;

/* L-BFGS trial on the device: one bre_engine_run iteration = one optimizer.step (closure, then a conditional-graph loop of up to
 * max_iter inner iterations, the re-evaluation of each under a conditional node) followed by the box projection, best-so-far (the
 * loss before the step against the candidate after it) and the history commit (optimization_based_attack.py:90-143 with
 * `optimizer.step(closure)`).  label_logits (device or host, NULL unless joint): [N, classes] label leaf of the joint attacker
 * (optimization_with_label_attack.py), optimised as one flat vector after the candidate.  Refused (BRE_ERR_UNSUPPORTED) with
 * augmentations, Langevin noise, token programs or with the option use_graph off. */
int bre_engine_begin_lbfgs_trial(bre_engine* e, const float* candidate, const float* label_logits, int64_t n_label, const float* lr_table,
                                 int32_t n_lr, const bre_lbfgs_consts* consts);
/* out[4] = inner iterations and closure evaluations over the trial, live pairs, oldest slot (synchronises the engine stream). */
int bre_engine_lbfgs_counters(bre_engine* e, int32_t* out);
/* One inner iteration's direction on caller-owned device buffers (parity tests): when state->total_iters > 0 the candidate pair
 * (y = g - prev_g, s = t * d) is written to the spare slot of S / Y [history + 1, n] and pushed if it passes the curvature test;
 * then d = -H g (torch's two-loop recursion, evaluated over the Gram matrices), prev_g = g, total_iters += 1.  gram (device doubles):
 * [SY (h+1)^2 | YY (h+1)^2 | rho h+1 | coefficients 2 (h+1)] with h = consts->history, SY[i][j] = s_i.y_j; state: device. */
int bre_lbfgs_direction(float* S, float* Y, double* gram, bre_lbfgs_scalars* state, const float* g, float* prev_g, float* d, int64_t n,
                        const bre_lbfgs_consts* consts, void* stream);

const char* bre_last_error(void);
const char* bre_version(void);

#ifdef __cplusplus
}
#endif
#endif /* BREACHING_B200_H */
