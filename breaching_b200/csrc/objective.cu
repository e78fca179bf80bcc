// Objective-side kernels (see objective.cuh).  All HBM/L2-bound: 128-bit loads, warp-shuffle reductions,
// one deterministic cross-block reduction per kernel (last-arriving block sums the partials in order), no atomics
// on data, no host synchronisation: every scalar the next stage needs stays in the device-resident Scalars block.
#include "objective.cuh"
#include "cluster_rows.cuh"

namespace bre {

namespace {

// --------------------------------------------------------------------------------------------------
// matching reduction
// --------------------------------------------------------------------------------------------------
__device__ void finalize_objective(Scalars* sc, int objective, float scale, float tag_scale, float fudge) {
  const double dot = sc->dot, nG = sc->nG, ng = sc->ng, sq = sc->sq, l1w = sc->l1w;
  double match = 0.0, c1 = 0.0, c2 = 0.0, c3 = 0.0;
  switch (objective) {
    case BRE_OBJ_EUCLIDEAN: match = 0.5 * sq * scale; c1 = -scale; c2 = scale; break;
    case BRE_OBJ_L1: match = 0.5 * l1w * scale; c3 = 0.5 * scale; break;
    case BRE_OBJ_TAG_EUCLIDEAN: match = 0.5 * scale * (sq + tag_scale * l1w); c1 = -scale; c2 = scale; c3 = 0.5 * scale * tag_scale; break;
    case BRE_OBJ_COSINE:
    case BRE_OBJ_MASKED_COSINE:
    case BRE_OBJ_FAST_COSINE:
    case BRE_OBJ_ANGULAR: {
      const double denom = sqrt(nG) * sqrt(ng);
      const double cosv = dot / denom;
      double alpha = -1.0 / denom;                   // d(1 - cos)/dG = alpha * g + beta * G
      double beta = dot / (nG * sqrt(nG) * sqrt(ng));
      if (objective == BRE_OBJ_FAST_COSINE) beta = 0.0;
      if (objective == BRE_OBJ_ANGULAR) {
        const double lo = -1.0 + fudge, hi = 1.0 - fudge;
        const double c = cosv < lo ? lo : (cosv > hi ? hi : cosv);
        match = acos(c) / 3.14159265358979323846 * scale;
        const double inside = (cosv > lo && cosv < hi) ? 1.0 : 0.0;
        const double f = inside * scale / (3.14159265358979323846 * sqrt(1.0 - c * c));
        c1 = f * alpha; c2 = f * beta;
      } else {
        match = (1.0 - cosv) * scale;
        c1 = scale * alpha; c2 = scale * beta;
      }
      break;
    }
    default: break;
  }
  sc->match = match;
  sc->c1 = (float)c1; sc->c2 = (float)c2; sc->c3 = (float)c3;
}

template <int U>
__global__ void __launch_bounds__(256) match_reduce_kernel(const float* __restrict__ G, const float* __restrict__ g,
                                                          const float* __restrict__ chunk_w, long long n, long long nchunks,
                                                          float mask_value, int objective, float scale, float tag_scale,
                                                          float fudge, bool finalize, Scalars* sc, double* partials,
                                                          int* counter) {
  pdl_prologue();
  __shared__ double scratch[32];
  __shared__ int s_last;
  double acc[5] = {0, 0, 0, 0, 0};
  const bool masked = mask_value >= 0.f;
  // U chunks in flight per block iteration: 2 U independent 128-bit loads per thread
  for (long long base = (long long)blockIdx.x * U; base < nchunks; base += (long long)gridDim.x * U) {
    float a[U][4], b[U][4];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long i = (base + u) * kChunk + threadIdx.x * 4;
#pragma unroll
      for (int j = 0; j < 4; ++j) { a[u][j] = 0.f; b[u][j] = 0.f; }
      if (base + u < nchunks) {
        if (i + 3 < n) {
          const float4 va = __ldg(reinterpret_cast<const float4*>(G + i));
          const float4 vb = __ldg(reinterpret_cast<const float4*>(g + i));
          a[u][0] = va.x; a[u][1] = va.y; a[u][2] = va.z; a[u][3] = va.w;
          b[u][0] = vb.x; b[u][1] = vb.y; b[u][2] = vb.z; b[u][3] = vb.w;
        } else {
          for (int j = 0; j < 4; ++j)
            if (i + j < n) { a[u][j] = G[i + j]; b[u][j] = g[i + j]; }
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const float w = (chunk_w != nullptr && base + u < nchunks) ? __ldg(chunk_w + base + u) : 1.f;
      float s0 = 0, s1 = 0, s2 = 0, s3 = 0, s4 = 0;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float x = a[u][j], y = b[u][j];
        if (masked && !(fabsf(y) > mask_value)) { x = 0.f; y = 0.f; }
        const float df = x - y;
        s0 = fmaf(x, y, s0); s1 = fmaf(x, x, s1); s2 = fmaf(y, y, s2); s3 = fmaf(df, df, s3); s4 += fabsf(df);
      }
      acc[0] += s0; acc[1] += s1; acc[2] += s2; acc[3] += s3; acc[4] += (double)w * s4;
    }
  }
  // block reduction of the five sums with one barrier: warp shuffles, then [5][8] doubles through shared memory
  __shared__ double wsum[5][8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    const double t = warp_sum(acc[k]);
    if (lane == 0) wsum[k][warp] = t;
  }
  __syncthreads();
  if (threadIdx.x < 5) {
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += wsum[threadIdx.x][w];
    partials[(long long)blockIdx.x * 5 + threadIdx.x] = t;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const int prev = atomicAdd(counter, 1);
    s_last = (prev == (int)gridDim.x - 1);
    if (s_last) *counter = 0;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // last block: thread t sums the partials of blocks t, t + 256, ... (fixed assignment), then the same block reduction:
  // launch-invariant summation order, three dependent memory round trips instead of gridDim.x
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    double t = 0.0;
    for (int b = threadIdx.x; b < (int)gridDim.x; b += 256) t += __ldcg(partials + (long long)b * 5 + k);
    t = warp_sum(t);
    if (lane == 0) wsum[k][warp] = t;
  }
  __syncthreads();
  if (threadIdx.x < 5) {
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += wsum[threadIdx.x][w];
    (&sc->dot)[threadIdx.x] = t;
  }
  __syncthreads();
  if (threadIdx.x == 0 && finalize) finalize_objective(sc, objective, scale, tag_scale, fudge);
}

__global__ void __launch_bounds__(256) make_v_kernel(const float* __restrict__ G, const float* __restrict__ g,
                                                    const float* __restrict__ chunk_w, float* __restrict__ v, long long n,
                                                    long long nchunks, float mask_value, const Scalars* sc, float* __restrict__ vt,
                                                    const unsigned char* __restrict__ chunk_mode) {
  pdl_prologue();
  const float c1 = sc->c1, c2 = sc->c2, c3 = sc->c3;
  const bool masked = mask_value >= 0.f;
  for (long long ch = blockIdx.x; ch < nchunks; ch += gridDim.x) {
    const long long i = ch * kChunk + threadIdx.x * 4;
    if (i >= n) continue;
    const float w3 = c3 * (chunk_w != nullptr ? __ldg(chunk_w + ch) : 1.f);
    float a[4] = {0, 0, 0, 0}, b[4] = {0, 0, 0, 0}, r[4];
    const bool full = i + 3 < n;
    if (full) {
      const float4 va = __ldg(reinterpret_cast<const float4*>(G + i));
      const float4 vb = __ldg(reinterpret_cast<const float4*>(g + i));
      a[0] = va.x; a[1] = va.y; a[2] = va.z; a[3] = va.w;
      b[0] = vb.x; b[1] = vb.y; b[2] = vb.z; b[3] = vb.w;
    } else {
      for (int j = 0; j < 4; ++j)
        if (i + j < n) { a[j] = G[i + j]; b[j] = g[i + j]; }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float df = a[j] - b[j];
      const float sg = df > 0.f ? 1.f : (df < 0.f ? -1.f : 0.f);
      float val = fmaf(c1, b[j], fmaf(c2, a[j], w3 * sg));
      if (masked && !(fabsf(b[j]) > mask_value)) val = 0.f;
      r[j] = val;
    }
    // chunk_mode (with vt): 0 = fp32 direction only, 1 = only its TF32-rounded shadow (operand of tensor-core GEMMs, nobody reads
    // the fp32 value), 2 = both.  One pass instead of make_v + a separate rounding pass over the whole arena.
    const int mode = (vt != nullptr) ? (chunk_mode != nullptr ? (int)__ldg(chunk_mode + ch) : 2) : 0;
    if (mode != 1) {
      if (full) *reinterpret_cast<float4*>(v + i) = make_float4(r[0], r[1], r[2], r[3]);
      else
        for (int j = 0; j < 4; ++j)
          if (i + j < n) v[i + j] = r[j];
    }
    if (mode != 0) {
      if (full) *reinterpret_cast<float4*>(vt + i) = make_float4(tf32_rna(r[0]), tf32_rna(r[1]), tf32_rna(r[2]), tf32_rna(r[3]));
      else
        for (int j = 0; j < 4; ++j)
          if (i + j < n) vt[i + j] = tf32_rna(r[j]);
    }
  }
}

// --------------------------------------------------------------------------------------------------
// image priors: total variation (+ double opponents) and L^p norm, value and gradient in one pass
// --------------------------------------------------------------------------------------------------
__device__ __forceinline__ float powx(float a, float e) {
  if (e == 1.f) return a;
  if (e == 0.f) return 1.f;
  if (e == 2.f) return a * a;
  if (e == 0.5f) return sqrtf(a);
  if (e == -0.5f) return rsqrtf(a);
  return powf(a, e);
}

struct TvD { float f, fh, fw; };
// t00 = t(i,j), t10 = t(i+1,j), t01 = t(i,j+1)
__device__ __forceinline__ TvD tv_point(float t00, float t10, float t01, float p, float q, float eps) {
  const float dh = t10 - t00, dw = t01 - t00;
  const float a = fabsf(dh) + eps, b = fabsf(dw) + eps;
  const float s = powx(a, p) + powx(b, p);
  TvD r;
  r.f = powx(s, q);
  const float common = q * powx(s, q - 1.f) * p;
  const float sh = dh > 0.f ? 1.f : (dh < 0.f ? -1.f : 0.f);
  const float sw = dw > 0.f ? 1.f : (dw < 0.f ? -1.f : 0.f);
  r.fh = common * powx(a, p - 1.f) * sh;
  r.fw = common * powx(b, p - 1.f) * sw;
  return r;
}

constexpr int TV_TW = 32, TV_TH = 8;

__global__ void __launch_bounds__(TV_TW * TV_TH) image_priors_kernel(PriorArgs a, Scalars* sc, double* partials, int* counter) {
  pdl_prologue();
  __shared__ float xs[3][TV_TH + 2][TV_TW + 2];
  __shared__ double scratch[32];
  __shared__ int s_last;
  const int n = blockIdx.z;
  const int i0 = blockIdx.y * TV_TH, j0 = blockIdx.x * TV_TW;
  const int tid = threadIdx.y * TV_TW + threadIdx.x;
  const long long plane = (long long)a.H * a.W;
  const float* xn = a.x + (long long)n * 3 * plane;
  for (int e = tid; e < 3 * (TV_TH + 2) * (TV_TW + 2); e += TV_TW * TV_TH) {
    const int c = e / ((TV_TH + 2) * (TV_TW + 2));
    const int r = e - c * ((TV_TH + 2) * (TV_TW + 2));
    const int li = r / (TV_TW + 2), lj = r - li * (TV_TW + 2);
    const int i = i0 + li - 1, j = j0 + lj - 1;
    float val = 0.f;
    if (i >= 0 && i < a.H && j >= 0 && j < a.W) val = __ldg(xn + c * plane + (long long)i * a.W + j);
    xs[c][li][lj] = val;
  }
  __syncthreads();
  const int i = i0 + threadIdx.y, j = j0 + threadIdx.x;
  const int li = threadIdx.y + 1, lj = threadIdx.x + 1;
  const bool valid = i < a.H && j < a.W;
  double tv_sum = 0.0, norm_sum = 0.0;
  float gx[3] = {0.f, 0.f, 0.f};
  if (valid) {
    const int nplanes = a.double_opponents ? 6 : 3;
    if (a.tv_scale != 0.f) {
      const float coef = a.tv_scale / ((float)a.N * (float)nplanes * (float)a.H * (float)a.W);
      for (int k = 0; k < nplanes; ++k) {
        int ca, cb;  // plane = x[ca] - x[cb] (cb < 0: plain channel)
        if (k < 3) { ca = k; cb = -1; } else if (k == 3) { ca = 0; cb = 1; } else if (k == 4) { ca = 0; cb = 2; } else { ca = 1; cb = 2; }
        auto T = [&](int y, int x) -> float { return cb < 0 ? xs[ca][y][x] : xs[ca][y][x] - xs[cb][y][x]; };
        const float t00 = T(li, lj);
        const TvD d0 = tv_point(t00, T(li + 1, lj), T(li, lj + 1), a.p, a.q, a.eps);
        float gk = -d0.fh - d0.fw;
        tv_sum += (double)d0.f;
        if (i >= 1) gk += tv_point(T(li - 1, lj), t00, T(li - 1, lj + 1), a.p, a.q, a.eps).fh;
        if (j >= 1) gk += tv_point(T(li, lj - 1), T(li + 1, lj - 1), t00, a.p, a.q, a.eps).fw;
        gk *= coef;
        gx[ca] += gk;
        if (cb >= 0) gx[cb] -= gk;
      }
    }
    if (a.norm_scale != 0.f) {
      const float coef = a.norm_scale / ((float)a.N * 3.f * (float)a.H * (float)a.W);
      for (int c = 0; c < 3; ++c) {
        const float xv = xs[c][li][lj];
        norm_sum += (double)powx(xv, a.norm_p);
        gx[c] += coef * powx(xv, a.norm_p - 1.f);
      }
    }
    for (int c = 0; c < 3; ++c) {
      float* gp = a.grad + ((long long)n * 3 + c) * plane + (long long)i * a.W + j;
      *gp = a.accumulate ? *gp + gx[c] : gx[c];
    }
  }
  // deterministic value reduction
  const int nblocks = gridDim.x * gridDim.y * gridDim.z;
  const int bid = (blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
  // block_sum uses threadIdx.x only for lane/warp ids: linearise
  {
    const int lane = tid & 31, warp = tid >> 5;
    double t0 = warp_sum(tv_sum), t1 = warp_sum(norm_sum);
    if (lane == 0) { scratch[warp] = t0; scratch[8 + warp] = t1; }
    __syncthreads();
    if (tid == 0) {
      double s0 = 0, s1 = 0;
      for (int w = 0; w < TV_TW * TV_TH / 32; ++w) { s0 += scratch[w]; s1 += scratch[8 + w]; }
      partials[2LL * bid] = s0; partials[2LL * bid + 1] = s1;
    }
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    const int prev = atomicAdd(counter, 1);
    s_last = (prev == nblocks - 1);
    if (s_last) *counter = 0;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  double s0 = 0, s1 = 0;
  for (int b = tid; b < nblocks; b += TV_TW * TV_TH) { s0 += __ldcg(partials + 2LL * b); s1 += __ldcg(partials + 2LL * b + 1); }
  // fixed-order tree: per-thread strided partials, then warp/block reduction (order is launch-invariant)
  {
    const int lane = tid & 31, warp = tid >> 5;
    s0 = warp_sum(s0); s1 = warp_sum(s1);
    __syncthreads();
    if (lane == 0) { scratch[warp] = s0; scratch[8 + warp] = s1; }
    __syncthreads();
    if (tid == 0) {
      double t0 = 0, t1 = 0;
      for (int w = 0; w < TV_TW * TV_TH / 32; ++w) { t0 += scratch[w]; t1 += scratch[8 + w]; }
      const double np = a.double_opponents ? 6.0 : 3.0;
      sc->tv = a.tv_scale != 0.f ? (double)a.tv_scale * t0 / ((double)a.N * np * a.H * a.W) : 0.0;
      sc->norm = a.norm_scale != 0.f ? (double)a.norm_scale / (double)a.norm_p * t1 / ((double)a.N * 3.0 * a.H * a.W) : 0.0;
    }
  }
}

// NormRegularization (regularizers.py:184-200) for candidates that are not 3-channel images (the tiled kernel above is
// specialised for RGB): value mean(x^p) / p * scale into sc->norm, gradient accumulated into grad; sc->tv = 0.
__global__ void __launch_bounds__(256) norm_prior_kernel(const float* __restrict__ x, float* __restrict__ grad, long long n, float scale,
                                                         float p, int accumulate, Scalars* sc, double* partials, int* counter) {
  pdl_prologue();
  __shared__ double scratch[32];
  __shared__ int s_last;
  const float coef = scale / (float)n;
  double sum = 0.0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float xv = x[i];
    sum += (double)powx(xv, p);
    const float gk = coef * powx(xv, p - 1.f);
    grad[i] = accumulate ? grad[i] + gk : gk;
  }
  const double bs = block_sum(sum, scratch);
  if (threadIdx.x == 0) partials[blockIdx.x] = bs;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const int prev = atomicAdd(counter, 1);
    s_last = (prev == (int)gridDim.x - 1);
    if (s_last) *counter = 0;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  double t = 0.0;
  for (int b = threadIdx.x; b < (int)gridDim.x; b += blockDim.x) t += __ldcg(partials + b);
  t = block_sum(t, scratch);
  if (threadIdx.x == 0) { sc->norm = (double)scale / (double)p * t / (double)n; sc->tv = 0.0; }
}

// --------------------------------------------------------------------------------------------------
// Philox4x32-10, the counter-based generator of the Langevin noise.  Key = the 64-bit seed; counter words = (element index low,
// element index high, iteration, trial index): the grad-norm and the step kernel recompute the same draw for an element, and
// every (trial, iteration, element) has its own.
// --------------------------------------------------------------------------------------------------
__device__ __forceinline__ void philox_round(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
  const uint32_t hi0 = __umulhi(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
  const uint32_t hi1 = __umulhi(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
  const uint32_t n0 = hi1 ^ c[1] ^ k0, n1 = lo1, n2 = hi0 ^ c[3] ^ k1, n3 = lo0;
  c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
}
// N(0,1) by Box-Muller from the first two output words: uniforms on the open 24-bit grid ((w >> 8) + 0.5) / 2^24
__device__ __forceinline__ float gaussian_noise(uint64_t seed, uint32_t trial, uint32_t it, uint64_t idx) {
  uint32_t c[4] = {(uint32_t)idx, (uint32_t)(idx >> 32), it, trial};
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) { philox_round(c, k0, k1); k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
  const float u1 = ((float)(c[0] >> 8) + 0.5f) * (1.0f / 16777216.0f);
  const float u2 = ((float)(c[1] >> 8) + 0.5f) * (1.0f / 16777216.0f);
  return sqrtf(-2.0f * logf(u1)) * cospif(2.0f * u2);
}

__device__ __forceinline__ float raw_gradient(const StepArgs& a, const Scalars* sc, long long i, float lr) {
  float gr = a.grad[i];
  if (a.grad_task != nullptr && a.cfg.task_regularization != 0.f) gr = fmaf(a.cfg.task_regularization, a.grad_task[i], gr);
  if (a.cfg.langevin_noise > 0.f)
    gr = fmaf(a.cfg.langevin_noise * lr, gaussian_noise(a.cfg.noise_seed, (uint32_t)sc->trial, (uint32_t)sc->it, (uint64_t)i), gr);
  return gr;
}

// the bare N(0,1) draws of elements [first, first + n) (parity tests of the generator)
__global__ void __launch_bounds__(256) langevin_noise_kernel(uint64_t seed, uint32_t trial, uint32_t it, uint64_t first, long long n,
                                                             float* __restrict__ out) {
  pdl_prologue();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = gaussian_noise(seed, trial, it, first + (uint64_t)i);
}

__global__ void __launch_bounds__(256) grad_norm_kernel(StepArgs a, Scalars* sc, double* partials, int* counter) {
  pdl_prologue();
  __shared__ double scratch[32];
  __shared__ int s_last;
  const int it = sc->it;
  const float lr = it < a.n_lr ? a.lr_table[it] : 0.f;
  double acc = 0.0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < a.n; i += (long long)gridDim.x * blockDim.x) {
    const float gr = raw_gradient(a, sc, i, lr);
    acc += (double)gr * gr;
  }
  const double t = block_sum(acc, scratch);
  if (threadIdx.x == 0) partials[blockIdx.x] = t;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const int prev = atomicAdd(counter, 1);
    s_last = (prev == (int)gridDim.x - 1);
    if (s_last) *counter = 0;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // last block: all 256 threads fold the per-block partials (fixed order: thread-strided, then the block tree)
  double s = 0.0;
  for (int b = threadIdx.x; b < (int)gridDim.x; b += blockDim.x) s += __ldcg(partials + b);
  s = block_sum(s, scratch);
  if (threadIdx.x == 0) sc->grad_norm_sq = s;
}

__global__ void __launch_bounds__(256) pixel_step_kernel(StepArgs a, Scalars* sc) {
  pdl_prologue();
  if (sc->stopped) return;
  __shared__ float s_c[8];
  const int it = sc->it;
  const bre_attack_cfg& cfg = a.cfg;
  if (threadIdx.x == 0) {
    const double t = (double)(it + 1);
    const double lr = it < a.n_lr ? (double)a.lr_table[it] : 0.0;
    double bc1 = 1.0, bc2s = 1.0;
    if (cfg.optimizer != BRE_OPT_SGD) {
      bc1 = 1.0 - pow((double)cfg.beta1, t);
      bc2s = sqrt(1.0 - pow((double)cfg.beta2, t));
    }
    s_c[0] = (float)lr;
    s_c[1] = (float)(lr / bc1);                 // step_size = lr / bias_correction1   (torch.optim.Adam)
    s_c[2] = (float)bc2s;                       // sqrt(bias_correction2)
    s_c[3] = (float)(1.0 - lr * (double)cfg.weight_decay);
    s_c[4] = 1.0f - (float)it / (float)cfg.max_iterations;  // soft-sign scaling (optimization_based_attack.py:177-180)
    float clip_mul = 1.f;
    if (cfg.grad_clip >= 0.f) {
      const float nrm = (float)sqrt(sc->grad_norm_sq);
      if (nrm > cfg.grad_clip) clip_mul = cfg.grad_clip / (nrm + 1e-6f);
    }
    s_c[5] = clip_mul;
    const float phi = (float)total_objective(sc, cfg.objective_excludes_task ? 0.f : cfg.task_regularization);
    s_c[6] = (phi < (float)sc->fmin) ? 1.f : 0.f;
  }
  __syncthreads();
  const float lr = s_c[0], step = s_c[1], bc2s = s_c[2], decay = s_c[3], soft = s_c[4], clip_mul = s_c[5];
  const bool improved = s_c[6] != 0.f;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < a.n; i += (long long)gridDim.x * blockDim.x) {
    float gr = raw_gradient(a, sc, i, lr) * clip_mul;
    if (cfg.signed_mode == BRE_SIGN_HARD) gr = gr > 0.f ? 1.f : (gr < 0.f ? -1.f : gr);  // keeps 0 and NaN like torch.sign
    else if (cfg.signed_mode == BRE_SIGN_SOFT) gr = tanhf(gr * soft) / soft;
    if (a.grad_out != nullptr) { a.grad_out[i] = gr; continue; }
    float x = a.x[i];
    if (cfg.optimizer == BRE_OPT_SGD) {
      float dgr = gr;
      if (cfg.momentum != 0.f) {
        const float buf = it == 0 ? gr : fmaf(cfg.momentum, a.m[i], gr);
        a.m[i] = buf;
        dgr = cfg.nesterov ? fmaf(cfg.momentum, buf, gr) : buf;
      }
      x = fmaf(-lr, dgr, x);
    } else {
      if (cfg.optimizer == BRE_OPT_ADAMW) x *= decay;
      float m = a.m[i], v = a.v[i];
      m = fmaf(1.f - cfg.beta1, gr - m, m);                 // exp_avg.lerp_(grad, 1 - beta1)
      v = fmaf(1.f - cfg.beta2, gr * gr, v * cfg.beta2);    // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, 1 - beta2)
      a.m[i] = m; a.v[i] = v;
      const float denom = sqrtf(v) / bc2s + cfg.adam_eps;
      x = fmaf(-step, m / denom, x);
    }
    if (cfg.boxed) {
      const int c = (int)((i / a.HW) % a.C);
      x = fmaxf(fminf(x, __ldg(a.hi + c)), __ldg(a.lo + c));
    }
    a.x[i] = x;
    if (improved) a.best[i] = x;
  }
}

// ---- label leaf of the joint data + label optimisation (optimization_with_label_attack.py:145-189) ----------------------
// One thread-block cluster per row (cluster_rows.cuh): token models have 50 257 classes per row.
// q = softmax(label logits) per row: what the closure hands to the task loss (:154)
__global__ void __launch_bounds__(kRowThreads, 2) row_softmax_kernel(const float* __restrict__ ell, float* __restrict__ q, int C) {
  pdl_prologue();
  __shared__ RowReduce ws;
  int c0, c1;
  row_segment(C, c0, c1);
  const float* z = ell + (long long)blockIdx.x * C;
  float* o = q + (long long)blockIdx.x * C;
  if (seg_fits(C)) {   // segment in registers: one load, one reduction
    SegCache zc;
    seg_load(zc, z, c0, c1, -3.402823466e+38f);
    float m;
    double sum;
    seg_softmax_pair(zc, m, sum);
    row_allreduce_softmax(m, sum, ws, 0);
    const float inv = (float)(1.0 / sum);
#pragma unroll
    for (int k = 0; k < kSegCache; ++k) {
      const int c = c0 + k * kRowThreads + (int)threadIdx.x;
      if (c < c1) o[c] = expf(zc.v[k] - m) * inv;
    }
    cluster_exit();
    return;
  }
  float mx = -3.402823466e+38f;
  for (int c = c0 + threadIdx.x; c < c1; c += kRowThreads) mx = fmaxf(mx, z[c]);
  mx = (float)row_allreduce<ROW_MAX>((double)mx, ws, 0);
  double part = 0.0;
  for (int c = c0 + threadIdx.x; c < c1; c += kRowThreads) part += (double)expf(z[c] - mx);
  const float inv = (float)(1.0 / row_allreduce<ROW_SUM>(part, ws, 1));
  for (int c = c0 + threadIdx.x; c < c1; c += kRowThreads) o[c] = expf(z[c] - mx) * inv;
  cluster_exit();
}

// chain d(objective)/dq through the softmax onto the label logits (what autograd does at :162): g <- q * (g - <q, g>)
__global__ void __launch_bounds__(kRowThreads, 2) softmax_chain_kernel(const float* __restrict__ q, float* __restrict__ g, int C) {
  pdl_prologue();
  __shared__ RowReduce ws;
  int c0, c1;
  row_segment(C, c0, c1);
  const float* qq = q + (long long)blockIdx.x * C;
  float* gg = g + (long long)blockIdx.x * C;
  if (seg_fits(C)) {
    SegCache qc, gc;
    seg_load(qc, qq, c0, c1, 0.f);
    seg_load(gc, gg, c0, c1, 0.f);
    double part = 0.0;
#pragma unroll
    for (int k = 0; k < kSegCache; ++k) part += (double)qc.v[k] * (double)gc.v[k];
    const float dot = (float)row_allreduce<ROW_SUM>(part, ws, 0);
#pragma unroll
    for (int k = 0; k < kSegCache; ++k) {
      const int c = c0 + k * kRowThreads + (int)threadIdx.x;
      if (c < c1) gg[c] = qc.v[k] * (gc.v[k] - dot);
    }
    cluster_exit();
    return;
  }
  double part = 0.0;
  for (int c = c0 + threadIdx.x; c < c1; c += kRowThreads) part += (double)qq[c] * (double)gg[c];
  const float dot = (float)row_allreduce<ROW_SUM>(part, ws, 0);
  for (int c = c0 + threadIdx.x; c < c1; c += kRowThreads) gg[c] = qq[c] * (gg[c] - dot);
  cluster_exit();
}

__global__ void commit_kernel(Scalars* sc, float* history, int max_hist, float task_reg) {
  pdl_prologue();
  if (sc->stopped) return;
  const float phi = (float)total_objective(sc, task_reg);
  if (phi < (float)sc->fmin) sc->fmin = (double)phi;
  sc->last_objective = (double)phi;
  if (!isfinite(phi)) {
    sc->stopped = 1;
  } else {
    if (sc->recorded < max_hist) history[sc->recorded] = phi;
    sc->recorded += 1;
  }
  sc->it += 1;
}

__global__ void loss_mean_kernel(const float* loss_n, int N, Scalars* sc) {
  pdl_prologue();
  double s = 0.0;
  for (int n = 0; n < N; ++n) s += (double)loss_n[n];
  sc->task_loss = (double)(float)(s / N);
}

// DeepInversion value and adjoint coefficients: one block per BN layer (not one block walking all 20-53 layers), then a one-warp sum of the per-layer values in layer order.
// `adjoint_scale` multiplies the adjoint coefficients only (1 in single-step evaluations, -1/lr for the seeds of a FedAvg step).
__global__ void __launch_bounds__(256) di_layer_kernel(const DiLayer* layers, double* layer_values, double adjoint_scale) {
  pdl_prologue();
  __shared__ double scratch[32];
  __shared__ double s_n[2];
  const DiLayer L = layers[blockIdx.x];
  double av = 0.0, am = 0.0;
  for (int c = threadIdx.x; c < L.C; c += blockDim.x) {
    const double dv = (double)L.rv[c] - (double)L.var[c], dm = (double)L.rm[c] - (double)L.mean[c];
    av += dv * dv; am += dm * dm;
  }
  const double tv = block_sum(av, scratch);
  if (threadIdx.x == 0) s_n[0] = sqrt(tv);
  const double tm = block_sum(am, scratch);
  if (threadIdx.x == 0) s_n[1] = sqrt(tm);
  __syncthreads();
  const double nv = s_n[0], nm = s_n[1];
  if (threadIdx.x == 0) layer_values[blockIdx.x] = (double)L.mult * (nv + nm);
  for (int c = threadIdx.x; c < L.C; c += blockDim.x) {
    const float cm = nm > 0.0 ? (float)((double)L.mult * ((double)L.mean[c] - (double)L.rm[c]) / nm / (double)L.M * adjoint_scale) : 0.f;
    const float cv = nv > 0.0 ? (float)((double)L.mult * ((double)L.var[c] - (double)L.rv[c]) / nv * 2.0 / (double)L.M * adjoint_scale) : 0.f;
    L.cm[c] = cm; L.cv[c] = cv;
  }
}
__global__ void di_sum_kernel(const double* layer_values, int n_layers, Scalars* sc) {
  pdl_prologue();
  if (threadIdx.x != 0) return;
  double value = 0.0;
  for (int l = 0; l < n_layers; ++l) value += layer_values[l];
  sc->di = value;
}

__global__ void __launch_bounds__(256) feature_reg_kernel(const float* __restrict__ feat, const float* __restrict__ measured,
                                                         float* tdelta, long long n, float scale, Scalars* sc) {
  pdl_prologue();
  __shared__ double scratch[32];
  double acc = 0.0;
  const float coef = 2.f * scale / (float)n;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) {
    const float df = feat[i] - measured[i];
    acc += (double)df * df;
    tdelta[i] = fmaf(coef, df, tdelta[i]);
  }
  const double t = block_sum(acc, scratch);
  if (threadIdx.x == 0) sc->feat = (double)scale * t / (double)n;
}

}  // namespace

// ---- OrthogonalityRegularization ---------------------------------------------------------------------------------
// R = sum_{i != j} (1/D) sum_k x_ik^2 x_jk^2 = (1/D) sum_k [S_k^2 - Q_k],  S_k = sum_j x_jk^2, Q_k = sum_j x_jk^4
// dR/dx_ik = (4/D) x_ik (S_k - x_ik^2).  One thread per position k, the batch (small) in a register loop.
__global__ void orthogonality_kernel(const float* __restrict__ x, float* __restrict__ grad, int N, long long D, bool overwrite,
                                     Scalars* sc, double* partials, int* counter) {
  pdl_prologue();
  __shared__ double scratch[32];
  __shared__ int s_last;
  double part = 0.0;
  const float scale = 4.0f / (float)D;
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < D; k += (long long)gridDim.x * blockDim.x) {
    float S = 0.f, Q = 0.f;
    for (int j = 0; j < N; ++j) { const float v = x[(long long)j * D + k]; const float v2 = v * v; S += v2; Q = fmaf(v2, v2, Q); }
    part += (double)S * (double)S - (double)Q;
    for (int j = 0; j < N; ++j) {
      const float v = x[(long long)j * D + k];
      grad[(long long)j * D + k] += scale * v * (S - v * v);
    }
  }
  const double tot = block_sum(part, scratch);
  if (threadIdx.x == 0) {
    partials[blockIdx.x] = tot;
    __threadfence();
    const int prev = atomicAdd(counter, 1);
    s_last = (prev == (int)gridDim.x - 1);
    if (s_last) *counter = 0;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  double acc = 0.0;
  for (int b = threadIdx.x; b < (int)gridDim.x; b += blockDim.x) acc += partials[b];
  const double all = block_sum(acc, scratch);
  if (threadIdx.x == 0) {
    const double r = all / (double)D;
    sc->norm = overwrite ? r : sc->norm + r;
  }
}

int launch_orthogonality(const float* x, float* grad, int N, long long D, bool overwrite, Scalars* sc, double* partials, int* counter,
                         cudaStream_t s) {
  if (N < 2) return 0;   // regularizers.py:170-171: a single image contributes 0
  long long blocks = (D + 255) / 256;
  const long long cap = (long long)kNumSMs * 4;
  const int grid = (int)(blocks < cap ? blocks : cap);
  BRE_KLAUNCH(orthogonality_kernel, grid, 256, 0, s, x, grad, N, D, overwrite, sc, partials, counter);
  BRE_CHECK_LAUNCH();
  return 0;
}

// launch shape of the matching reduction
static int g_match_blocks_per_sm = 4, g_match_unroll = 4;

int launch_match_reduce(const float* G, const float* g, const float* chunk_w, long long n, float mask_value,
                        int objective, float scale, float tag_scale, float fudge, bool finalize, Scalars* sc,
                        double* partials, int* counter, cudaStream_t s) {
  const long long nchunks = (n + kChunk - 1) / kChunk;
  const int unroll = g_match_unroll == 8 ? 8 : 4;
  const long long groups = (nchunks + unroll - 1) / unroll;
  int cap = kNumSMs * g_match_blocks_per_sm;
  if (cap > kMatchMaxBlocks) cap = kMatchMaxBlocks;
  const int grid = (int)(groups < cap ? (groups > 0 ? groups : 1) : cap);
  if (unroll == 8)
    BRE_KLAUNCH(match_reduce_kernel<8>, grid, 256, 0, s, G, g, chunk_w, n, nchunks, mask_value, objective, scale, tag_scale, fudge,
                finalize, sc, partials, counter);
  else
    BRE_KLAUNCH(match_reduce_kernel<4>, grid, 256, 0, s, G, g, chunk_w, n, nchunks, mask_value, objective, scale, tag_scale, fudge,
                finalize, sc, partials, counter);
  BRE_CHECK_LAUNCH();
  return 0;
}

int launch_make_v(const float* G, const float* g, const float* chunk_w, float* v, long long n, float mask_value,
                  const Scalars* sc, cudaStream_t s, float* vt, const unsigned char* chunk_mode) {
  const long long nchunks = (n + kChunk - 1) / kChunk;
  const int cap = kNumSMs * 8;
  const int grid = (int)(nchunks < cap ? (nchunks > 0 ? nchunks : 1) : cap);
  BRE_KLAUNCH(make_v_kernel, grid, 256, 0, s, G, g, chunk_w, v, n, nchunks, mask_value, sc, vt, chunk_mode);
  BRE_CHECK_LAUNCH();
  return 0;
}

int launch_image_priors(const PriorArgs& a, Scalars* sc, double* partials, int* counter, cudaStream_t s) {
  dim3 grid(ceil_div(a.W, TV_TW), ceil_div(a.H, TV_TH), a.N), block(TV_TW, TV_TH);
  BRE_KLAUNCH(image_priors_kernel, grid, block, 0, s, a, sc, partials, counter);
  BRE_CHECK_LAUNCH();
  return 0;
}

int launch_norm_prior(const float* x, float* grad, long long n, float scale, float p, int accumulate, Scalars* sc, double* partials,
                      int* counter, cudaStream_t s) {
  long long b = (n + 255) / 256;
  if (b > kNumSMs * 4) b = kNumSMs * 4;
  BRE_KLAUNCH(norm_prior_kernel, (int)b, 256, 0, s, x, grad, n, scale, p, accumulate, sc, partials, counter);
  BRE_CHECK_LAUNCH();
  return 0;
}

static inline int step_grid(long long n) {
  long long b = (n + 255) / 256;
  const long long cap = kStepMaxBlocks;
  return (int)(b < cap ? (b > 0 ? b : 1) : cap);
}

int launch_grad_norm(const StepArgs& a, Scalars* sc, double* partials, int* counter, cudaStream_t s) {
  BRE_KLAUNCH(grad_norm_kernel, step_grid(a.n), 256, 0, s, a, sc, partials, counter);
  BRE_CHECK_LAUNCH();
  return 0;
}
int launch_pixel_step(const StepArgs& a, Scalars* sc, cudaStream_t s) {
  BRE_KLAUNCH(pixel_step_kernel, step_grid(a.n), 256, 0, s, a, sc);
  BRE_CHECK_LAUNCH();
  return 0;
}
int launch_langevin_noise(uint64_t seed, uint32_t trial, uint32_t it, uint64_t first, long long n, float* out, cudaStream_t s) {
  BRE_KLAUNCH(langevin_noise_kernel, step_grid(n), 256, 0, s, seed, trial, it, first, n, out);
  BRE_CHECK_LAUNCH();
  return 0;
}
int launch_row_softmax(const float* ell, float* q, int rows, int C, cudaStream_t s) {
  if (launch_row_kernel(row_softmax_kernel, rows, C, s, ell, q, C) != cudaSuccess) { set_error("row softmax: launch failed"); return -2; }
  BRE_CHECK_LAUNCH();
  return 0;
}
int launch_softmax_chain(const float* q, float* g, int rows, int C, cudaStream_t s) {
  if (launch_row_kernel(softmax_chain_kernel, rows, C, s, q, g, C) != cudaSuccess) { set_error("softmax chain: launch failed"); return -2; }
  BRE_CHECK_LAUNCH();
  return 0;
}
int launch_commit(Scalars* sc, float* history, int max_hist, float task_reg, cudaStream_t s) {
  BRE_KLAUNCH(commit_kernel, 1, 1, 0, s, sc, history, max_hist, task_reg);
  BRE_CHECK_LAUNCH();
  return 0;
}
int launch_loss_mean(const float* loss_n, int N, Scalars* sc, cudaStream_t s) {
  BRE_KLAUNCH(loss_mean_kernel, 1, 1, 0, s, loss_n, N, sc);
  BRE_CHECK_LAUNCH();
  return 0;
}
int launch_di_finalize(const DiLayer* layers_dev, int n_layers, double* layer_values, Scalars* sc, cudaStream_t s, double adjoint_scale) {
  BRE_KLAUNCH(di_layer_kernel, n_layers, 256, 0, s, layers_dev, layer_values, adjoint_scale);
  BRE_KLAUNCH(di_sum_kernel, 1, 32, 0, s, (const double*)layer_values, n_layers, sc);
  BRE_CHECK_LAUNCH();
  return 0;
}
int launch_feature_reg(const float* feat, const float* measured, float* tdelta, long long n, float scale, Scalars* sc,
                       cudaStream_t s) {
  BRE_KLAUNCH(feature_reg_kernel, 1, 256, 0, s, feat, measured, tdelta, n, scale, sc);
  BRE_CHECK_LAUNCH();
  return 0;
}

}  // namespace bre

// tuning hook for the launch shape of the matching reduction (not part of the reference-facing ABI)
extern "C" void bre_debug_match_config(int blocks_per_sm, int unroll) {
  if (blocks_per_sm >= 1 && blocks_per_sm <= 8) bre::g_match_blocks_per_sm = blocks_per_sm;
  if (unroll == 4 || unroll == 8) bre::g_match_unroll = unroll;
}
