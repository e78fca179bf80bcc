// Small-batch linear layers (the classification head at batch 1-16, token-model projections at <= 32 rows): fprop / dgrad / wgrad of  out[n][co] = sum_k in[n][k] W[co][k]
// with the optional K-concatenated second source of the tangent sweeps.  At these sizes the contraction is a handful of
// matrix-vector products over a [Co][Ci] weight matrix (ResNet-18 head: 397 x 512 = 0.8 MB): HBM/L2-latency bound, no reuse to
// tile for -- the 64x64-tile implicit GEMM would run a single row of tiles.  fp32 throughout (bit-class parity with the fp32 SIMT back end: the
// same products, summed in a fixed order).
#include "igemm.cuh"
#include <type_traits>

namespace bre {
namespace {

constexpr int LS_MAXN = 32;

// ---- fprop: one warp per output channel, all rows --------------------------------------------------------------------------
template <int NB>
__global__ void __launch_bounds__(256) linear_small_fprop_kernel(GemmArgs a, int vec) {
  pdl_prologue();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int Co = a.g.Co, Ci = a.g.Ci, N = a.g.N;
  if (warp >= Co) return;
  float acc[NB];
#pragma unroll
  for (int n = 0; n < NB; ++n) acc[n] = 0.f;
  for (int s = 0; s < a.nsrc; ++s) {
    const float* __restrict__ w = a.wgt[s] + (long long)warp * Ci;
    const float* __restrict__ x = a.act[s];
    if (vec) {
      for (int k = lane * 4; k < Ci; k += 128) {
        const float4 wv = __ldg(reinterpret_cast<const float4*>(w + k));
#pragma unroll
        for (int n = 0; n < NB; ++n) {
          if (n < N) {
            const float4 xv = __ldg(reinterpret_cast<const float4*>(x + n * a.x_sN + k));
            acc[n] = fmaf(wv.x, xv.x, fmaf(wv.y, xv.y, fmaf(wv.z, xv.z, fmaf(wv.w, xv.w, acc[n]))));
          }
        }
      }
    } else {
      for (int k = lane; k < Ci; k += 32) {
        const float wv = __ldg(w + k);
#pragma unroll
        for (int n = 0; n < NB; ++n)
          if (n < N) acc[n] = fmaf(wv, __ldg(x + n * a.x_sN + k), acc[n]);
      }
    }
  }
  const float b = a.bias != nullptr ? __ldg(a.bias + warp) : 0.f;
#pragma unroll
  for (int n = 0; n < NB; ++n) {
    const float t = warp_sum(acc[n]);
    if (lane == 0 && n < N) a.out[(long long)n * Co + warp] = t + b;
  }
}

// ---- dgrad: block = 32 input channels x 32 groups of output channels (one warp per group, lanes along ci: coalesced 128-byte
//      rows of W); every thread keeps four independent weight loads in flight; fixed-order reduction over the groups ----------------
template <int NB>
__global__ void __launch_bounds__(1024) linear_small_dgrad_kernel(GemmArgs a) {
  pdl_prologue();
  constexpr int G = NB >= 16 ? 8 : (NB >= 8 ? 16 : 32);   // groups of output channels = warps per block (17 KB of partials)
  __shared__ float part[G][NB][33];
  const int cx = threadIdx.x & 31, grp = threadIdx.x >> 5;
  const int ci = blockIdx.x * 32 + cx;
  const int Co = a.g.Co, Ci = a.g.Ci, N = a.g.N;
  float acc[NB];
#pragma unroll
  for (int n = 0; n < NB; ++n) acc[n] = 0.f;
  if (ci < Ci) {
    for (int s = 0; s < a.nsrc; ++s) {
      const float* __restrict__ w = a.wgt[s];
      const float* __restrict__ dy = a.act[s];
      int co = grp;
      for (; co + 3 * G < Co; co += 4 * G) {
        float wv[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) wv[u] = __ldg(w + (long long)(co + u * G) * Ci + ci);
#pragma unroll
        for (int u = 0; u < 4; ++u) {
#pragma unroll
          for (int n = 0; n < NB; ++n)
            if (n < N) acc[n] = fmaf(wv[u], __ldg(dy + (long long)n * Co + co + u * G), acc[n]);
        }
      }
      for (; co < Co; co += G) {
        const float wv = __ldg(w + (long long)co * Ci + ci);
#pragma unroll
        for (int n = 0; n < NB; ++n)
          if (n < N) acc[n] = fmaf(wv, __ldg(dy + (long long)n * Co + co), acc[n]);
      }
    }
  }
#pragma unroll
  for (int n = 0; n < NB; ++n) part[grp][n][cx] = acc[n];
  __syncthreads();
  for (int idx = threadIdx.x; idx < NB * 32; idx += 32 * G) {
    const int n = idx >> 5, c = idx & 31;
    const int cc = blockIdx.x * 32 + c;
    if (n >= N || cc >= Ci) continue;
    float t = 0.f;
#pragma unroll
    for (int g2 = 0; g2 < G; ++g2) t += part[g2][n][c];
    float* o = a.out + (long long)n * a.x_sN + (long long)cc * a.x_sC;
    *o = a.accumulate ? *o + t : t;
  }
}

// ---- wgrad: one thread per weight element -------------------------------------------------------------------------------------------
template <int NB>
__global__ void __launch_bounds__(256) linear_small_wgrad_kernel(GemmArgs a) {
  pdl_prologue();
  const int Co = a.g.Co, Ci = a.g.Ci, N = a.g.N;
  const long long total = (long long)Co * Ci;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int co = (int)(i / Ci), ci = (int)(i - (long long)co * Ci);
    float t = 0.f;
    for (int s = 0; s < a.nsrc; ++s) {
      const float* __restrict__ x = a.act[s];    // in  [N][Ci]
      const float* __restrict__ dy = a.wgt[s];   // dout [N][Co]
#pragma unroll
      for (int n = 0; n < NB; ++n)
        if (n < N) t = fmaf(__ldg(dy + (long long)n * Co + co), __ldg(x + n * a.x_sN + ci), t);
    }
    a.out[i] = a.accumulate ? a.out[i] + t : t;
  }
}

template <int NB>
int launch_nb(const GemmArgs& a, int vec, cudaStream_t stream) {
  const int Co = a.g.Co, Ci = a.g.Ci;
  if (a.mode == GEMM_FPROP) {
    BRE_KLAUNCH((linear_small_fprop_kernel<NB>), ceil_div((long long)Co * 32, 256), 256, 0, stream, a, vec);
  } else if (a.mode == GEMM_DGRAD) {
    BRE_KLAUNCH((linear_small_dgrad_kernel<NB>), ceil_div(Ci, 32), 32 * (NB >= 16 ? 8 : (NB >= 8 ? 16 : 32)), 0, stream, a);
  } else {
    long long blocks = ((long long)Co * Ci + 255) / 256;
    if (blocks > kNumSMs * 8) blocks = kNumSMs * 8;
    BRE_KLAUNCH((linear_small_wgrad_kernel<NB>), (int)blocks, 256, 0, stream, a);
  }
  BRE_CHECK_LAUNCH();
  return 0;
}

// ---- tall-K dgrad: din[n][ci] = sum_co dy[n][co] W[co][ci] with few rows (n <= 32), a narrow input (ci <= 128) and a very long
//      reduction (the 96 -> 50257 decoder of the token models: Co = 50304).  As an implicit GEMM this is one row of 128 x 32 output
//      tiles whose split-K is capped by the cluster size, so few CTAs stream the 19 MB weight matrix.  Here the reduction is cut into ~2 chunks per SM; a block keeps all
//      n x ci partial sums of its chunk in registers (warp = 8 rows x one half of the chunk's output channels, lanes along ci, so the
//      weight rows are read as coalesced 128-byte lines exactly once per block) and a second small kernel adds the per-chunk
//      partials in a fixed order.  Same products as the GEMM back ends (the operands are the same arrays), fp32 accumulation.
constexpr int LT_ROWS = 32, LT_MAXC = 96, LT_PITCH = LT_ROWS + 4;

__device__ __forceinline__ void lt_cp_async16(float* smem_dst, const float* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}

// The weight rows of a chunk are one contiguous block of memory ([Co][Ci] row-major): they are brought into shared memory with 16-byte
// cp.async granules, every load of the block in flight at once (with register loads the kernel runs as a chain of dependent HBM
// round trips per block).  The products then run out of shared memory: per output channel a warp reads CJ
// conflict-free 128-byte rows and two broadcast 16-byte vectors for 8 CJ fused multiply-adds per lane.
template <int CJ>   // CJ = Ci / 32
__global__ void __launch_bounds__(256, 4) linear_tall_dgrad_kernel(GemmArgs a, int chunk, float* __restrict__ partials) {
  extern __shared__ __align__(16) float lt_smem[];
  float* w_s = lt_smem;                                                                              // [chunk][Ci]; reused for the final fold
  float(*dy_s)[LT_PITCH] = reinterpret_cast<float(*)[LT_PITCH]>(lt_smem + LT_MAXC * CJ * 32);        // [co][n], 16-byte aligned rows
  pdl_prologue();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int half = warp >> 2, r0 = (warp & 3) * 8;              // warps 0-3: even output channels, 4-7: odd; 8 rows each
  const int Co = a.g.Co, N = a.g.N;
  constexpr int Ci = CJ * 32;
  const int c0 = blockIdx.x * chunk, cn = min(chunk, Co - c0);
  float acc[8][CJ];
#pragma unroll
  for (int r = 0; r < 8; ++r)
#pragma unroll
    for (int j = 0; j < CJ; ++j) acc[r][j] = 0.f;
  for (int s = 0; s < a.nsrc; ++s) {
    const float* __restrict__ wsrc = a.wgt[s] + (long long)c0 * Ci;
    const float* __restrict__ dy = a.act[s] + c0;
    __syncthreads();                                             // the previous source has been consumed
    for (int i = threadIdx.x; i < cn * (Ci / 4); i += 256) lt_cp_async16(w_s + 4 * i, wsrc + 4 * i);
    asm volatile("cp.async.commit_group;" ::: "memory");
    for (int i = threadIdx.x; i < chunk * LT_ROWS; i += 256) {   // coalesced along co, transposed into [co][n]
      const int n = i / chunk, c = i - n * chunk;
      dy_s[c][n] = (n < N && c < cn) ? __ldg(dy + (long long)n * Co + c) : 0.f;
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
#pragma unroll 4
    for (int c = half; c < cn; c += 2) {
      float wv[CJ];
#pragma unroll
      for (int j = 0; j < CJ; ++j) wv[j] = w_s[c * Ci + 32 * j + lane];
      const float4 d0 = *reinterpret_cast<const float4*>(&dy_s[c][r0]);
      const float4 d1 = *reinterpret_cast<const float4*>(&dy_s[c][r0 + 4]);
      const float dv[8] = {d0.x, d0.y, d0.z, d0.w, d1.x, d1.y, d1.z, d1.w};
#pragma unroll
      for (int r = 0; r < 8; ++r)
#pragma unroll
        for (int j = 0; j < CJ; ++j) acc[r][j] = fmaf(dv[r], wv[j], acc[r][j]);
    }
  }
  __syncthreads();
  float* fold = w_s;                                             // [4 row groups][8 rows][Ci]: the odd half's sums
  if (half == 1) {
#pragma unroll
    for (int r = 0; r < 8; ++r)
#pragma unroll
      for (int j = 0; j < CJ; ++j) fold[((warp & 3) * 8 + r) * Ci + 32 * j + lane] = acc[r][j];
  }
  __syncthreads();
  if (half == 0) {
    float* __restrict__ dst = partials + (long long)blockIdx.x * LT_ROWS * Ci;
#pragma unroll
    for (int r = 0; r < 8; ++r)
#pragma unroll
      for (int j = 0; j < CJ; ++j) dst[(r0 + r) * Ci + 32 * j + lane] = acc[r][j] + fold[(warp * 8 + r) * Ci + 32 * j + lane];
  }
}

// out[n][ci] (+)= sum over chunks of partials[chunk][n][ci]: block = 32 adjacent outputs x 32 interleaved slices of the chunk list
// (warp w adds chunks w, w + 32, ...: coalesced 128-byte rows, four loads in flight), folded over the slices in a fixed order
__global__ void __launch_bounds__(1024) linear_tall_fold_kernel(const float* __restrict__ partials, int chunks, int Ci, int N, long long x_sN,
                                                                int accumulate, float* __restrict__ out) {
  __shared__ float part[32][33];
  pdl_prologue();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int o = blockIdx.x * 32 + lane;                 // index into [LT_ROWS][Ci]
  const long long per = (long long)LT_ROWS * Ci;
  const float* __restrict__ src = partials + o;
  float t = 0.f;
  int c = warp;
  for (; c + 96 < chunks; c += 128) {
    const float v0 = __ldcg(src + c * per), v1 = __ldcg(src + (c + 32) * per), v2 = __ldcg(src + (c + 64) * per), v3 = __ldcg(src + (c + 96) * per);
    t += v0; t += v1; t += v2; t += v3;
  }
  for (; c < chunks; c += 32) t += __ldcg(src + c * per);
  part[warp][lane] = t;
  __syncthreads();
  if (warp == 0) {
    float sum = 0.f;
#pragma unroll
    for (int k = 0; k < 32; ++k) sum += part[k][lane];
    const int n = o / Ci, ci = o - n * Ci;
    if (n < N) {
      float* dst = out + (long long)n * x_sN + ci;
      *dst = accumulate ? *dst + sum : sum;
    }
  }
}

inline int tall_chunk(int Co) {   // ~4 blocks per SM, an even number of output channels per block, 32 .. LT_MAXC
  int chunk = ceil_div(Co, 4 * kNumSMs);
  chunk += chunk & 1;
  return chunk < 32 ? 32 : (chunk > LT_MAXC ? LT_MAXC : chunk);
}

}  // namespace

bool linear_tall_supported(const GemmArgs& a) {
  const ConvGeom& g = a.g;
  if (!gemm_switches().linear_tall || a.mode != GEMM_DGRAD) return false;
  if (!(g.R == 1 && g.S == 1 && g.H == 1 && g.W == 1 && g.Ho == 1 && g.Wo == 1 && g.stride == 1 && g.pad == 0)) return false;
  if (g.N < 1 || g.N > LT_ROWS || g.Ci % 32 != 0 || g.Ci > 128 || g.Co < 8192 || a.x_sC != 1 || a.epi.kind != 0) return false;
  if (a.nsrc < 1 || a.nsrc > 2 || a.ws == nullptr) return false;
  for (int s = 0; s < a.nsrc; ++s)
    if ((reinterpret_cast<uintptr_t>(a.wgt[s]) & 15) != 0) return false;   // 16-byte cp.async granules of the weight rows
  const long long need = (long long)ceil_div(g.Co, tall_chunk(g.Co)) * LT_ROWS * g.Ci;
  return need <= (long long)a.ws_tiles * IG_BM * IG_BN;
}

GemmPlan linear_tall_plan(const GemmArgs& a) {
  const int chunk = tall_chunk(a.g.Co);
  GemmPlan p;
  p.family = GEMM_FAM_LINEAR_TALL; p.mode = a.mode; p.nsrc = a.nsrc; p.tile_rows = LT_ROWS; p.tile_width = a.g.Ci;
  p.splits = ceil_div(a.g.Co, chunk); p.total_kblocks = a.g.Co; p.kblocks_per_split = chunk;
  return p;
}

int launch_linear_tall(const GemmArgs& a, const GemmPlan& p, cudaStream_t stream) {
  const int Ci = a.g.Ci;
  const int chunk = p.kblocks_per_split, chunks = p.splits;
  auto go = [&](auto cj_tag) -> int {
    constexpr int CJ = decltype(cj_tag)::value;
    const size_t smem = (size_t)(LT_MAXC * CJ * 32 + LT_MAXC * LT_PITCH) * sizeof(float);
    static bool attr_done = false;
    if (!attr_done) {
      if (cudaFuncSetAttribute(linear_tall_dgrad_kernel<CJ>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
        set_error("tall linear dgrad: shared memory opt-in failed");
        return -2;
      }
      attr_done = true;
    }
    BRE_KLAUNCH((linear_tall_dgrad_kernel<CJ>), chunks, 256, smem, stream, a, chunk, a.ws);
    return 0;
  };
  int rc = 0;
  switch (Ci / 32) {
    case 1: rc = go(std::integral_constant<int, 1>{}); break;
    case 2: rc = go(std::integral_constant<int, 2>{}); break;
    case 3: rc = go(std::integral_constant<int, 3>{}); break;
    default: rc = go(std::integral_constant<int, 4>{}); break;
  }
  if (rc != 0) return rc;
  BRE_KLAUNCH(linear_tall_fold_kernel, LT_ROWS * Ci / 32, 1024, 0, stream, (const float*)a.ws, chunks, Ci, a.g.N, a.x_sN, a.accumulate, a.out);
  BRE_CHECK_LAUNCH();
  return 0;
}

bool linear_small_supported(const GemmArgs& a) {
  const ConvGeom& g = a.g;
  return g.R == 1 && g.S == 1 && g.H == 1 && g.W == 1 && g.Ho == 1 && g.Wo == 1 && g.stride == 1 && g.pad == 0 && g.N >= 1 && g.N <= LS_MAXN &&
         a.x_sC == 1 && a.epi.kind == 0 && a.nsrc >= 1 && a.nsrc <= 2 && !(a.mode == GEMM_FPROP && a.accumulate);
}

// Kernel instance: the smallest row count NB >= N; fprop loads 16-byte vectors where the rows and both operands allow.
GemmPlan linear_small_plan(const GemmArgs& a) {
  GemmPlan p;
  p.family = GEMM_FAM_LINEAR_SMALL; p.mode = a.mode; p.nsrc = a.nsrc;
  p.tile_rows = 1;
  while (p.tile_rows < a.g.N) p.tile_rows *= 2;
  if (a.mode == GEMM_FPROP) {
    auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
    bool vec = (a.g.Ci % 4 == 0) && (a.x_sN % 4 == 0);
    for (int s = 0; s < a.nsrc; ++s) vec = vec && al16(a.act[s]) && al16(a.wgt[s]);
    p.vec = vec ? 1 : 0;
  }
  return p;
}

int launch_linear_small(const GemmArgs& a, const GemmPlan& p, cudaStream_t stream) {
  switch (p.tile_rows) {
    case 1: return launch_nb<1>(a, p.vec, stream);
    case 2: return launch_nb<2>(a, p.vec, stream);
    case 4: return launch_nb<4>(a, p.vec, stream);
    case 8: return launch_nb<8>(a, p.vec, stream);
    case 16: return launch_nb<16>(a, p.vec, stream);
    default: return launch_nb<32>(a, p.vec, stream);
  }
}

// Experiment switch (BRE_LINEAR_SMALL_ROWS=1): send linear layers on <= 32 rows with a short reduction (token models at batch 1:
// 96 -> 288 / 96 / 1536 projections) to the matrix-vector kernels even where the tensor-core kernel covers the shape.  At 32 rows
// 32 accumulators per thread and 32 broadcast loads per weight element are no match for one MMA, so the default is off.
bool linear_small_preferred(const GemmArgs& a) {
  if (!gemm_switches().linear_small_rows || a.mode == GEMM_WGRAD || !linear_small_supported(a)) return false;
  const int K = (a.mode == GEMM_FPROP ? a.g.Ci : a.g.Co) * a.nsrc;
  return K <= 512;
}

}  // namespace bre
