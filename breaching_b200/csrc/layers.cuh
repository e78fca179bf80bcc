// Non-GEMM layer kernels of the four sweeps (NHWC activations): eval-mode BN + residual + ReLU (fused),
// max/avg pooling, softmax cross-entropy, per-channel reductions, layout permutes.
#pragma once
#include "common.cuh"

namespace bre {

// capacity (floats) callers must provide for the `partials` scratch of the slab reductions below
constexpr long long kSlabPartialFloats = 1 << 18;

struct BnConsts {          // per-channel constants of an eval-mode BN (weights are fixed during an attack)
  const float* scale;      // gamma * inv
  const float* shift;      // beta - gamma * mean * inv
  const float* inv;        // 1/sqrt(var + eps)
  const float* nrm;        // -mean * inv      (xhat = x * inv + nrm)
};

// dst[c] constants from (gamma, beta, running_mean, running_var)
int launch_bn_prepare(const float* gamma, const float* beta, const float* rm, const float* rv, float eps, int C,
                      float* scale, float* shift, float* inv, float* nrm, cudaStream_t s);

// out = relu?( bn?(in) + res? )
// round_out: store `out` rounded onto the TF32 grid (it is an operand of tensor-core GEMMs, see tf32_rna in common.cuh)
int launch_bnact_fwd(const float* in, const float* res, float* out, long long P, int C, bool has_bn, bool relu,
                     BnConsts bn, bool round_out, cudaStream_t s);

struct BnActBwdArgs {
  long long P; int C; bool has_bn, relu;
  BnConsts bn;
  const float* in;      // BN input z (for xhat)
  const float* out;     // activation (ReLU mask)
  const float* dout;    // delta of out
  float* din; bool acc_in;     // may be null
  float* dres; bool acc_res;   // may be null
  bool round_din;              // store din on the TF32 grid (GEMM operand of dgrad / wgrad)
  float* g_gamma; float* g_beta;  // parameter-gradient outputs (may be null)
  float* partials; int* counters; // scratch: >= slabs*Cpad*2 floats, >= Cgroups ints (zeroed, self-resetting)
  int defer;                      // != 0: stop after writing the slab partials; launch_bn_grad_finalize sums them later
};
int launch_bnact_bwd(const BnActBwdArgs& a, cudaStream_t s);
// deferred finalisation of g_gamma / g_beta for all BN layers of a sweep in one launch
struct BnGradSlot { const float* partials; int slabs, Cpad, C, first_block; float* g_gamma; float* g_beta; };
void bnact_bwd_plan(long long P, int C, int* slabs, int* Cpad);   // slab count / padded channel count launch_bnact_bwd will use
int launch_bn_grad_finalize(const BnGradSlot* table_dev, int n_layers, int total_blocks, cudaStream_t s);

struct BnActTanFwdArgs {
  long long P; int C; bool has_bn, relu;
  BnConsts bn;
  const float* in; const float* out;   // forward values (xhat, mask)
  const float* tin; const float* tres; // tangents (may be null = zero)
  const float* v_gamma; const float* v_beta;
  float* tout;
  bool round_out;                      // store tout on the TF32 grid
};
int launch_bnact_tan_fwd(const BnActTanFwdArgs& a, cudaStream_t s);

struct BnActTanBwdArgs {
  long long P; int C; bool has_bn, relu;
  BnConsts bn;
  const float* in; const float* out;
  const float* tdout;   // tangent delta of out
  const float* dout;    // sweep-B delta of out
  const float* v_gamma;
  const float* di_cm; const float* di_cv; const float* di_mean;  // DeepInversion adjoint (may be null)
  float* tdin; bool acc_in;
  float* tdres; bool acc_res;
  bool round_din;                      // store tdin on the TF32 grid
  // FedAvg (multi-step) only: tangent of the BN parameter gradients, needed for the Hessian-vector product that carries
  // the adjoint across local steps: tg_gamma = sum(tdu * xhat + du * tin * inv), tg_beta = sum(tdu)   (null = not needed)
  const float* tin; float* tg_gamma; float* tg_beta; float* partials; int* counters;
};
int launch_bnact_tan_bwd(const BnActTanBwdArgs& a, cudaStream_t s);
// out[i] = x[i] + alpha * y[i]   (parameter-arena updates of the local-step recursion)
int launch_axpby(const float* x, const float* y, float alpha, float* out, long long n, cudaStream_t s);
int launch_round_tf32(const float* src, float* dst, long long n, cudaStream_t s);   // dst = src rounded onto the TF32 grid (may alias)

// per-channel column sum: out[c] = sum_p x[p][c]   (conv / linear bias gradient)
// ---- train-mode BatchNorm (no server / user buffers, base_attack.py:192-197: batch statistics of the candidate) ----------
// Rules (oracle/program_interp.py, verified against autograd's double backward): with xh the normalised input, m(.) the
// per-channel mean over (N, H, W), inv = 1/sigma, du the ReLU-masked delta of the op's output
//   F :  statistics -> (inv, nrm, scale, shift), then the eval-mode kernel
//   B :  dx  = gamma inv (du - m(du) - xh m(du xh))                    [m(du), m(du xh) = G_beta / P, G_gamma / P]
//   TF:  xh' = inv (x' - m(x') - xh m(xh x'));  y' = v_gamma xh + gamma xh' + v_beta
//   TB:  dx' = (v_gamma inv - scale inv m(xh x')) w + scale (du' - m(du') - xh' m(du xh) - xh m(du' xh + du xh')),
//        w = du - m(du) - xh m(du xh)
struct BnTrainArgs {
  long long P; int C; bool relu;
  const float* in;  const float* out;                 // BN input value, post-activation value (ReLU mask)
  const float *inv, *nrm, *scale;                     // per-channel constants of this forward
  const float *v_gamma, *v_beta;                      // direction components (tangent sweeps)
  const float *sum_du, *sum_duxh;                     // G_beta, G_gamma of sweep B (sums over P)
  const float *m1, *m2;                               // TF means  m(x'), m(xh x')
  const float *b1, *b2;                               // TB means  m(du'), m(du' xh + du xh')
  const float *dout, *tdout;                          // delta / tangent delta of the op's output
  const float* xd;                                    // tangent of the BN input
  const float* tres;                                  // tangent of the residual branch (may be null)
  float* dst; bool acc; bool round_out;               // result of the pass (din / tout / tdin)
  float* dres; bool acc_res;                          // TB: tangent delta of the residual branch (may be null)
  // FedAvg (multi-step) only, null otherwise.  B: copies of sum_du / sum_duxh that outlive the G arena (the step's reverse pass
  // reads them after later steps have overwritten G).  TB statistics: the tangents of the gamma / beta gradients,
  // tg_gamma = sum(du' xh + du xh'), tg_beta = sum(du') -- the undivided sums behind b2 / b1.
  float *keep_du, *keep_duxh;
  float *tg_gamma, *tg_beta;
};
int launch_bn_train_prepare(const float* mean, const float* var, const float* gamma, const float* beta, float eps, int C, float* scale,
                            float* shift, float* inv, float* nrm, cudaStream_t s);
int launch_bn_train_bwd(const BnTrainArgs& a, cudaStream_t s);                                  // B, second pass
int launch_bn_train_tan_stats(const BnTrainArgs& a, float* m1, float* m2, float* partials, int* counters, cudaStream_t s);
int launch_bn_train_tan_fwd(const BnTrainArgs& a, cudaStream_t s);                              // TF, second pass
int launch_bn_train_tanbwd_stats(const BnTrainArgs& a, float* b1, float* b2, float* partials, int* counters, cudaStream_t s);
int launch_bn_train_tan_bwd(const BnTrainArgs& a, cudaStream_t s);                              // TB, second pass

int launch_channel_sum(const float* x, long long P, int C, float* out, float* partials, int* counters, cudaStream_t s);
// per-channel mean / biased variance over pixels (DeepInversion statistics, deepinversion.py:96-98)
int launch_channel_stats(const float* x, long long P, int C, float* mean, float* var, float* partials, int* counters,
                         cudaStream_t s);

// one launch for the statistics of many tensors (DeepInversion): table entry per tensor
struct StatSlot {
  const float* x; long long P, pps; int C, LX, LY, cg, slabs, Cpad, first_block, first_group;
  float* partials; float* mean; float* var;
};
bool channel_stats_plan(long long P, int C, StatSlot* slot, long long target_blocks);   // target_blocks: this tensor's share of the batched grid
int launch_channel_stats_batched(const StatSlot* table_dev, int n_layers, int total_blocks, int total_groups, cudaStream_t s);

struct PoolGeom { int N, H, W, C, Ho, Wo, k, stride, pad; };
int launch_maxpool_fwd(const float* in, float* out, int* idx, PoolGeom g, cudaStream_t s);
int launch_maxpool_bwd(const float* dout, const int* idx, float* din, bool acc, PoolGeom g, cudaStream_t s);
int launch_maxpool_gather(const float* tin, const int* idx, float* tout, PoolGeom g, cudaStream_t s);
int launch_avgpool_fwd(const float* in, float* out, int N, int HW, int C, cudaStream_t s);
int launch_avgpool_bwd(const float* dout, float* din, bool acc, int N, int HW, int C, cudaStream_t s);

// softmax cross-entropy (mean over N): p, per-sample loss and dlogits = (p - onehot)/N
// q (may be null): class-probability targets [N, C] instead of the index labels (joint data / label optimisation)
int launch_ce_fwd(const float* logits, const long long* labels, const float* q, int N, int C, float* p, float* loss_n,
                  float* dlogits, cudaStream_t s);
// d(objective)/dq from the tangent logits of the last tangent-forward sweep (+ task_reg * dL/dq)
int launch_ce_label_grad(const float* logits, const float* p, const float* zdot, int N, int C, float task_reg, float* out,
                         cudaStream_t s);
// tangent of dlogits: (p*zdot - p * sum(p*zdot)) / N
int launch_ce_tan_bwd(const float* p, const float* zdot, int N, int C, float* tdlogits, cudaStream_t s);
// the same plus coef * (p - onehot(labels)) / N (index labels), optionally stored on the TF32 grid: the task-loss seed of the last
// local step's tangent backward in a FedAvg evaluation (coef = -task_regularization / lr)
int launch_ce_tan_bwd_seeded(const float* p, const float* zdot, const long long* labels, int N, int C, float coef, float* tdlogits,
                             bool round_out, cudaStream_t s);

// column path of the candidate-fed convolution (stem_cols.cu): xcol[(n,p,q)][(r,s,c)] <- NCHW candidate (K padded to Kp, optional
// TF32 rounding); candidate gradient <- dcol by gathering; zero-padded [Co][Kp] copies of OHWI weight rows and back
int launch_stem_im2col(const float* x, float* xcol, int N, int C, int H, int W, int Ho, int Wo, int R, int S, int stride, int pad, int Kp,
                       bool round_out, cudaStream_t s);
int launch_stem_col2im(const float* dcol, float* grad, int N, int C, int H, int W, int Ho, int Wo, int R, int S, int stride, int pad, int Kp,
                       cudaStream_t s);
int launch_stem_pad_rows(const float* src, float* dst, int Co, int K, int Kp, bool inverse, bool round_out, cudaStream_t s);

// dst[(o*HW + hw)*I + i] = src[(o*I + i)*HW + hw]   (inverse=false: OIHW -> OHWI / NCHW -> NHWC)
int launch_permute(const float* src, float* dst, int O, int I, int HW, bool inverse, cudaStream_t s);
// y[i] += alpha * x[i]
int launch_axpy(const float* x, float* y, float alpha, long long n, cudaStream_t s);

}  // namespace bre
