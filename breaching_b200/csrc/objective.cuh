// Objective-side kernels: multi-tensor gradient-matching reduction, direction v, image priors, the fused
// signed-gradient optimiser step and the device-side trial bookkeeping.
#pragma once
#include "../../include/breaching_b200.h"
#include "common.cuh"

namespace bre {

// the recorded objective of an evaluation: matching term + priors (+ task_regularization * task loss)
__device__ __forceinline__ double total_objective(const Scalars* sc, float task_reg) {
  double phi = sc->match + sc->tv + sc->norm + sc->di + sc->feat;
  if (task_reg != 0.f) phi += (double)task_reg * sc->task_loss;
  return phi;
}

constexpr int kChunk = 1024;  // arena granularity of the matching reduction (per-chunk TAG weight)

// Sums over [0, n): <G,g>, |G|^2, |g|^2, sum (G-g)^2, sum w_chunk |G-g| (all masked where |g| <= mask_value when
// mask_value >= 0).  Result in sc->{dot,nG,ng,sq,l1w}; when `finalize` the last block also evaluates the matching
// objective and the coefficients of v (objectives.py:91-95,135-141,160-164,185-196,210-214,234-244,261-273).
int launch_match_reduce(const float* G, const float* g, const float* chunk_w, long long n, float mask_value,
                        int objective, float scale, float tag_scale, float fudge, bool finalize, Scalars* sc,
                        double* partials, int* counter, cudaStream_t s);
constexpr int kMatchMaxBlocks = kNumSMs * 8;   // capacity of the partials buffers; the launch uses g_match_blocks_per_sm (default 4)

// v = c1*g + c2*G + c3*w_chunk*sign(G-g)  (coefficients read from sc).  With `vt` the TF32-rounded shadow of the direction is
// written in the same pass; `chunk_mode[chunk]` (device, may be null = 2) selects per 1024-element chunk: 0 = v only, 1 = vt only,
// 2 = both.
int launch_make_v(const float* G, const float* g, const float* chunk_w, float* v, long long n, float mask_value,
                  const Scalars* sc, cudaStream_t s, float* vt = nullptr, const unsigned char* chunk_mode = nullptr);

struct PriorArgs {   // TotalVariation (regularizers.py:130-147) + NormRegularization (:197-198)
  const float* x; float* grad; int N, H, W; int accumulate;
  float tv_scale, p, q, eps; int double_opponents;
  float norm_scale, norm_p;
};
int launch_image_priors(const PriorArgs& a, Scalars* sc, double* partials, int* counter, cudaStream_t s);
// the L^p norm prior alone, for candidates with any channel count (x, grad: n contiguous floats)
int launch_norm_prior(const float* x, float* grad, long long n, float scale, float p, int accumulate, Scalars* sc, double* partials,
                      int* counter, cudaStream_t s);
// OrthogonalityRegularization (regularizers.py:169-178): sum_{i != j} mean_k (x_ik x_jk)^2 over the batch; value added to (or,
// with overwrite, stored in) the `norm` slot of the scalar block, gradient accumulated into grad.  x, grad: [N, D].
int launch_orthogonality(const float* x, float* grad, int N, long long D, bool overwrite, Scalars* sc, double* partials, int* counter,
                         cudaStream_t s);

struct StepArgs {   // closure tail + optimiser + projection + best-so-far (optimization_based_attack.py:112-121,166-184)
  float* x; float* m; float* v; float* best;
  const float* grad; const float* grad_task;  // d match/dx (+priors) and d task_loss/dx (may be null)
  const float* lr_table; int n_lr;
  const float* lo; const float* hi;           // per-channel box
  long long n; int C; int HW;
  bre_attack_cfg cfg;
  float* grad_out = nullptr;   // set: pixel_step writes the processed gradient here and does not step (the L-BFGS closure)
};
int launch_grad_norm(const StepArgs& a, Scalars* sc, double* partials, int* counter, cudaStream_t s);
int launch_pixel_step(const StepArgs& a, Scalars* sc, cudaStream_t s);
constexpr int kStepMaxBlocks = kNumSMs * 8;    // grid cap of the two kernels above = capacity launch_grad_norm needs in `partials`
// out[i] = the N(0,1) draw that the two kernels above scale by langevin_noise * lr and add to the gradient of element first + i
// in iteration `it` of trial `trial` (the same device function, not a restatement)
int launch_langevin_noise(uint64_t seed, uint32_t trial, uint32_t it, uint64_t first, long long n, float* out, cudaStream_t s);
// label leaf of the joint attacks: q = softmax(label logits) per row; g <- q * (g - <q, g>) (chain through that softmax)
int launch_row_softmax(const float* ell, float* q, int rows, int C, cudaStream_t s);
int launch_softmax_chain(const float* q, float* g, int rows, int C, cudaStream_t s);
// history / fmin / iteration counter / non-finite stop flag
int launch_commit(Scalars* sc, float* history, int max_hist, float task_reg, cudaStream_t s);
// task_loss = mean(loss_n)
int launch_loss_mean(const float* loss_n, int N, Scalars* sc, cudaStream_t s);

struct DiLayer { const float* mean; const float* var; const float* rm; const float* rv; float* cm; float* cv; int C; float M; float mult; };
// DeepInversion value + per-channel adjoint coefficients for all BN layers (one block, layers in order)
// `layer_values`: device scratch of n_layers doubles (two launches: one block per layer, then the ordered sum)
// `adjoint_scale` multiplies the per-channel adjoint coefficients, not the value: -1/lr when the adjoint seeds the last local step
// of a FedAvg evaluation (DESIGN.md section 3.1)
int launch_di_finalize(const DiLayer* layers_dev, int n_layers, double* layer_values, Scalars* sc, cudaStream_t s,
                       double adjoint_scale = 1.0);
// features regulariser: value into sc->feat, adjoint accumulated into tdelta
int launch_feature_reg(const float* feat, const float* measured, float* tdelta, long long n, float scale, Scalars* sc,
                       cudaStream_t s);

}  // namespace bre
