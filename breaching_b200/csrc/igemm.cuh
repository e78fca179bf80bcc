// Implicit-GEMM convolution family (fprop / dgrad / wgrad, optional K-concatenated second source).
//
// These are the dense contractions of the hot path: model forward (objectives.py:44), the first backward
// (objectives.py:45) and -- via the K-concatenated "dual source" form [W | v] . [a_dot ; a] -- both halves
// of the second backward (optimization_based_attack.py:165), see DESIGN.md section 3.
#pragma once
#include "common.cuh"

namespace bre {

enum GemmMode { GEMM_FPROP = 0, GEMM_DGRAD = 1, GEMM_WGRAD = 2 };

struct ConvGeom {
  int N, H, W, Ci;   // input-shaped tensor
  int Ho, Wo, Co;    // output-shaped tensor
  int R, S, stride, pad;
};

// Optional consumer fused into the FPROP epilogue of the tensor-core back end: the BN + residual + ReLU op that follows a
// convolution (layers.cu bnact_fwd_kernel, kind 1) or its tangent (bnact_tan_fwd_kernel, kind 2).  The GEMM result is still
// written to `out` when `out` is non-null (the backward sweeps need the pre-BN value; nobody reads the pre-BN tangent).
struct GemmEpilogue {
  int kind;                 // 0 = none, 1 = value, 2 = tangent
  int has_bn, relu;
  int round_out;            // store out2 on the TF32 grid (it feeds tensor-core GEMMs, see tf32_rna)
  float* out2;              // [M][Nc] output of the fused op
  const float* res;         // residual branch (value / tangent), may be null
  const float* scale;       // alpha = gamma * invstd
  const float* shift;       // kind 1: beta - mean * alpha
  const float* inv;         // kind 2: invstd, -mean * invstd  (xhat = pre * inv + nrm)
  const float* nrm;
  const float* v_gamma;     // kind 2: direction components of gamma / beta
  const float* v_beta;
  const float* pre;         // kind 2: forward pre-BN value and post-activation value (ReLU mask)
  const float* post;
};

struct GemmArgs {
  int mode;
  GemmEpilogue epi;
  ConvGeom g;
  int nsrc;               // 1 or 2 (dual source: K-concatenation, fprop / dgrad only)
  const float* act[2];    // fprop: in ; dgrad: dout ; wgrad: in
  const float* wgt[2];    // fprop/dgrad: weights OHWI ; wgrad: dout
  // addressing of the input-shaped tensor (gathered operand of fprop/wgrad, *output* of dgrad):
  // offset(img, pixel, c) = img * x_sN + pixel * x_sP + c * x_sC   (NHWC: HWC, C, 1 ; NCHW: CHW, 1, HW)
  long long x_sN;
  int x_sP, x_sC;
  float* out;
  const float* bias;      // fprop only, per output channel (may be null)
  int accumulate;         // out += result
  float* ws;              // split-K workspace (>= ws_tiles * 4096 floats)
  int* counters;          // >= max tiles ints, zero-initialised, self-resetting
  int ws_tiles;
  int force_fp32;         // engine: run this contraction on the fp32 kernels even on the tensor-core back end (precision knob)
  // bit s: wgt[s] (fprop / dgrad) was fully written before the *predecessor* kernel of this launch started, so the tensor-core back end
  // may start loading it before griddepcontrol.wait (model weights; the direction v once a serialised launch follows make_v)
  unsigned wgt_static;
};

constexpr int IG_BM = 64, IG_BN = 64, IG_BK = 16, IG_THREADS = 256;

// The launch plan of one GEMM: the kernel family, tiles, split, ring depth, operand producer and vector flags.  plan_gemm decides
// it from the arguments alone; the family launchers run it as given.  Host side only, never passed to a kernel.
enum GemmFamily { GEMM_FAM_SIMT = 0, GEMM_FAM_DGRAD_SMALL_CI = 1, GEMM_FAM_LINEAR_SMALL = 2, GEMM_FAM_LINEAR_TALL = 3, GEMM_FAM_TC = 4 };
enum GemmProducer { GEMM_PROD_NONE = 0, GEMM_PROD_TMA = 1, GEMM_PROD_CP_ASYNC = 2, GEMM_PROD_CLASSES = 3 };
struct GemmPlan {
  int family = -1, mode = -1, nsrc = 0;   // family -1: no kernel of the back end covers the contraction
  int tile_rows = 0, tile_width = 0;   // output tile (SIMT / tensor core); linear_small: rows of the kernel instance
  int splits = 1, stages = 0;          // split-K factor (grid z; linear_tall: reduction chunks), ring depth
  int producer = GEMM_PROD_NONE;
  int total_kblocks = 0, kblocks_per_split = 0;   // k-blocks of TC_BK = 32 (tensor core) / IG_BK = 16 (SIMT) over all sources
  int vec = 0;                         // SIMT: bit 0 vector A loads, bit 1 vector B loads, bit 2 vector stores; dgrad_small_ci /
                                       // linear_small fprop: vector loads
};
constexpr int GEMM_PLAN_FIELDS = 11;
// what launch_gemm ran last on the calling host thread (bre_debug_last_gemm_plan)
const GemmPlan& last_gemm_plan();

// Switches of the GEMM launch rules (experiments, and the references of the bitwise tests), read from the environment once per
// process: BRE_TC_* (tensor-core plans), BRE_LINEAR_* (which contractions the small-row linear kernels take).
struct GemmSwitches {
  int tc_tma;              // BRE_TC_TMA=0: the cp.async producer everywhere
  int tc_strided_tma;      // BRE_TC_STRIDED_TMA=0: strided dgrad on the cp.async producer instead of per-class tensor maps
  int tc_narrow;           // BRE_TC_NARROW=0: 128 x 64 tiles wherever the width allows
  int tc_stream;           // BRE_TC_STREAM=0: 128-row tiles also where the m-tile holds <= 64 rows
  int tc_stages;           // BRE_TC_STAGES=2|4|8: forced ring depth (anything else: by rule)
  int tc_shortk_stages;    // BRE_TC_SHORTK_STAGES (default 2: short reductions on many tiles run a 2-deep ring; 4 turns it off)
  int tc_max_splits;       // BRE_TC_MAX_SPLITS: cap of the split-K factor (0: none)
  int tc_target_ctas;      // BRE_TC_TARGET_CTAS: CTAs the split-K rule aims at (0: one per SM)
  int tc_proxy_fence;      // BRE_TC_PROXY_FENCE=1: async-proxy fence before every wgmma k-block also after TMA writes
  int tc_prefetch;         // BRE_TC_PREFETCH=0: no prefetch.tensormap
  int tc_producers;        // BRE_TC_PRODUCERS=1..4: TMA issuing lanes (default 2)
  int linear_small;        // BRE_LINEAR_SMALL=0: linear layers on <= 16 rows on the SIMT GEMM
  int linear_small_rows;   // BRE_LINEAR_SMALL_ROWS=1: linear layers on <= 32 rows with a short reduction on the small-row kernels
  int linear_tall;         // BRE_LINEAR_TALL=0: the tall-K linear dgrad on the GEMM back ends
};
const GemmSwitches& gemm_switches();

// One GEMM: the plan and its launch.  backend 0 = SIMT fp32 kernels, 1 = tensor cores only (empty plan where they do not cover the
// shape), 2 = the engine's dispatch (tensor cores where covered, the fp32 kernels otherwise).  plan_gemm allocates, encodes and
// launches nothing.  launch_gemm returns BRE_ERR_UNSUPPORTED (-4) for an empty plan.
GemmPlan plan_gemm(const GemmArgs& a, int backend);
int launch_gemm(const GemmArgs& a, int backend, cudaStream_t stream);

// The family launchers (called by launch_gemm) run the plan they are given.
// linear layers on <= 32 rows (the classification head at small batch): dedicated fp32 kernels (linear_small.cu)
bool linear_small_supported(const GemmArgs& a);
bool linear_small_preferred(const GemmArgs& a);   // small-row linear with a short reduction -> these kernels, not the GEMM
GemmPlan linear_small_plan(const GemmArgs& a);
int launch_linear_small(const GemmArgs& a, const GemmPlan& p, cudaStream_t stream);
// dgrad of a linear layer with <= 32 rows, <= 128 inputs and >= 8192 outputs (the token models' decoder): chunked reduction in
// fp32 registers + a fixed-order fold (linear_small.cu); uses a.ws for the per-chunk partial sums
bool linear_tall_supported(const GemmArgs& a);
GemmPlan linear_tall_plan(const GemmArgs& a);
int launch_linear_tall(const GemmArgs& a, const GemmPlan& p, cudaStream_t stream);
// TF32 tensor-core back end (igemm_tc.cu).  tc_plan: the plan of a covered shape, on the TMA producers where allow_tma and the
// geometry allow them; empty where no plan without them exists (widths that are only a multiple of 32).  launch_igemm_tc replaces
// `p` by tc_plan(a, false) when a tensor map of the plan does not encode.
bool igemm_tc_supported(const GemmArgs& a);
GemmPlan tc_plan(const GemmArgs& a, bool allow_tma);
int launch_igemm_tc(const GemmArgs& a, GemmPlan& p, cudaStream_t stream);

inline void gemm_dims(const GemmArgs& a, int& M, int& Nc, int& K) {
  const ConvGeom& g = a.g;
  if (a.mode == GEMM_FPROP) { M = g.N * g.Ho * g.Wo; Nc = g.Co; K = g.R * g.S * g.Ci; }
  else if (a.mode == GEMM_DGRAD) { M = g.N * g.H * g.W; Nc = g.Ci; K = g.R * g.S * g.Co; }
  else { M = g.Co; Nc = g.R * g.S * g.Ci; K = g.N * g.Ho * g.Wo; }
}

}  // namespace bre
