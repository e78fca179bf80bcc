// Token-sequence ops of the TAG / transformer path (SURVEY.md section 8 rows a15 / a16, BASELINE config 5): LayerNorm and
// multi-head self-attention in the four sweeps of the engine (forward, backward, tangent-forward, tangent-backward).  Rules
// and a float64-verified CPU statement of every formula: oracle/transformer_interp.py (header) and
// oracle/program_interp.py (OP_LAYERNORM / OP_ATTENTION of compiler.compile_transformer).  Tensors are [rows, C] fp32
// row-major with rows = batch * seq_len; attention reads the fused projection [rows, 3 d] = (q | k | v), head h in columns
// h*dh .. (h+1)*dh of each third.
//
// Sizes on this path are tiny (config 5: rows = 32, d = 96, 8 heads of 12): one warp per row for LayerNorm, one block per
// (sequence, head) for attention with the whole head resident in shared memory; plain fp32, deterministic (no atomics).
// First correct version -- exposed through a stand-alone C ABI (bre_token_layernorm / bre_token_attention) for kernel-level
// parity tests; the engine's sweeps do not dispatch to them yet.
#include <float.h>

#include "tokens.cuh"
#include "cluster_rows.cuh"

namespace bre {
namespace {

// ---- LayerNorm -----------------------------------------------------------------------------------------------------
// sweep 0 (F):  y = gamma xh + beta, stats[row] = (mean, inv)
// sweep 1 (B):  dx = inv (t - mean(t) - xh mean(t xh)),  t = dy gamma          [in1 = dy]
// sweep 2 (TF): y' = v_gamma xh + gamma xh' + v_beta,  xh' = inv (x' - mean(x') - xh mean(xh x'))   [in1 = x']
// sweep 3 (TB): dx' = inv u' - u mean(xh x') inv^2                              [in1 = dy', in2 = dy, in3 = x']
//               t' = dy' gamma + dy v_gamma, u = t - mean(t) - xh mean(t xh),
//               u' = t' - mean(t') - xh' mean(t xh) - xh mean(t' xh + t xh')
// kRound: store `out` on the TF32 grid (a template parameter so that the unrounded kernel is the plain one)
template <bool kRound>
__global__ void layernorm_kernel(int sweep, const float* __restrict__ x, const float* __restrict__ in1, const float* __restrict__ in2,
                                 const float* __restrict__ in3, const float* __restrict__ gamma, const float* __restrict__ beta,
                                 const float* __restrict__ v_gamma, const float* __restrict__ v_beta, float eps, int rows, int C,
                                 float* __restrict__ stats, float* __restrict__ out, int accumulate) {
  constexpr bool round_out = kRound;
  pdl_prologue();
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* xr = x + (long long)row * C;
  const float invC = 1.0f / (float)C;
  float mean, inv;
  if (sweep == 0) {
    float s = 0.f;
    for (int c = lane; c < C; c += 32) s += xr[c];
    mean = warp_sum(s) * invC;
    float q = 0.f;
    for (int c = lane; c < C; c += 32) { const float dlt = xr[c] - mean; q = fmaf(dlt, dlt, q); }
    inv = 1.0f / sqrtf(warp_sum(q) * invC + eps);
    if (lane == 0) { stats[2 * row] = mean; stats[2 * row + 1] = inv; }
    for (int c = lane; c < C; c += 32) {
      const float y = fmaf(gamma[c], (xr[c] - mean) * inv, beta[c]);
      out[(long long)row * C + c] = round_out ? tf32_rna(y) : y;
    }
    return;
  }
  mean = stats[2 * row];
  inv = stats[2 * row + 1];
  const float* a1 = in1 + (long long)row * C;
  float* o = out + (long long)row * C;
  if (sweep == 1) {
    float s0 = 0.f, s1 = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float t = a1[c] * gamma[c], xh = (xr[c] - mean) * inv;
      s0 += t; s1 = fmaf(t, xh, s1);
    }
    const float m0 = warp_sum(s0) * invC, m1 = warp_sum(s1) * invC;
    for (int c = lane; c < C; c += 32) {
      const float xh = (xr[c] - mean) * inv;
      const float v = inv * (a1[c] * gamma[c] - m0 - xh * m1);
      const float r = accumulate ? o[c] + v : v;
      o[c] = round_out ? tf32_rna(r) : r;
    }
  } else if (sweep == 2) {
    float s0 = 0.f, s1 = 0.f;
    for (int c = lane; c < C; c += 32) { const float xd = a1[c]; s0 += xd; s1 = fmaf((xr[c] - mean) * inv, xd, s1); }
    const float m0 = warp_sum(s0) * invC, m1 = warp_sum(s1) * invC;
    for (int c = lane; c < C; c += 32) {
      const float xh = (xr[c] - mean) * inv;
      const float xhd = inv * (a1[c] - m0 - xh * m1);
      const float yd = fmaf(v_gamma[c], xh, fmaf(gamma[c], xhd, v_beta[c]));
      o[c] = round_out ? tf32_rna(yd) : yd;
    }
  } else {
    const float* dyB = in2 + (long long)row * C;
    const float* xd = in3 + (long long)row * C;
    // pass 1: the means that xh' needs
    float s0 = 0.f, s1 = 0.f;
    for (int c = lane; c < C; c += 32) { s0 += xd[c]; s1 = fmaf((xr[c] - mean) * inv, xd[c], s1); }
    const float mxd = warp_sum(s0) * invC, mxhxd = warp_sum(s1) * invC;
    // pass 2: means of t, t xh, t', t' xh + t xh'
    float r0 = 0.f, r1 = 0.f, r2 = 0.f, r3 = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float xh = (xr[c] - mean) * inv;
      const float xhd = inv * (xd[c] - mxd - xh * mxhxd);
      const float t = dyB[c] * gamma[c];
      const float td = fmaf(a1[c], gamma[c], dyB[c] * v_gamma[c]);
      r0 += t; r1 = fmaf(t, xh, r1); r2 += td; r3 += fmaf(td, xh, t * xhd);
    }
    const float mt = warp_sum(r0) * invC, mtxh = warp_sum(r1) * invC, mtd = warp_sum(r2) * invC, mmix = warp_sum(r3) * invC;
    for (int c = lane; c < C; c += 32) {
      const float xh = (xr[c] - mean) * inv;
      const float xhd = inv * (xd[c] - mxd - xh * mxhxd);
      const float t = dyB[c] * gamma[c];
      const float td = fmaf(a1[c], gamma[c], dyB[c] * v_gamma[c]);
      const float u = t - mt - xh * mtxh;
      const float ud = td - mtd - xhd * mtxh - xh * mmix;
      const float v = inv * ud - u * mxhxd * inv * inv;
      const float r = accumulate ? o[c] + v : v;
      o[c] = round_out ? tf32_rna(r) : r;
    }
  }
}

// gamma / beta gradients of LayerNorm: G_gamma[c] = sum_rows dy xh, G_beta[c] = sum_rows dy.  Block = 32 columns x 8 row slices
// (warp w takes rows w, w + 8, ...: coalesced 128-byte row segments, 8 independent chains), folded over the slices in a fixed order.
__global__ void __launch_bounds__(256) layernorm_param_grad_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                                                                   const float* __restrict__ stats, int rows, int C,
                                                                   float* __restrict__ g_gamma, float* __restrict__ g_beta) {
  __shared__ float fg[8][32], fb[8][32];
  pdl_prologue();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + lane;
  float sg = 0.f, sb = 0.f;
  if (c < C) {
    for (int r = warp; r < rows; r += 8) {
      const float d = dy[(long long)r * C + c];
      sg = fmaf(d, (x[(long long)r * C + c] - stats[2 * r]) * stats[2 * r + 1], sg);
      sb += d;
    }
  }
  fg[warp][lane] = sg;
  fb[warp][lane] = sb;
  __syncthreads();
  if (warp == 0 && c < C) {
    float tg = 0.f, tb = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) { tg += fg[k][lane]; tb += fb[k][lane]; }
    g_gamma[c] = tg;
    g_beta[c] = tb;
  }
}

// ---- multi-head self-attention (no mask) ---------------------------------------------------------------------------
// One block of 256 threads per (sequence b, head h); Q, K, V [T][dh] (+ their tangents), the probabilities P [T][T] and scratch
// matrices live in shared memory; P (and the tangent P') are also kept in global memory [B, heads, T, T] between sweeps.
// Every sweep has two phases: (A) one warp per query row, lanes along the key index -- scores, the row reductions of the softmax
// and of its first / second derivative via warp shuffles; (B) all threads over the (row, channel) outputs, each a T-long dot
// product (not one *thread* per query row, which serialises the key loop).
//   sweep 0 (F):  O = P V                                  writes out [rows, d], P
//   sweep 1 (B):  d(qkv) from dO (= in1 [rows, d])          writes out [rows, 3 d]
//   sweep 2 (TF): O' from (qkv)' (= in1 [rows, 3 d])        writes out [rows, d], P'
//   sweep 3 (TB): d(qkv)' from dO' (= in1), dO (= in2), (qkv)' (= in3), P, P'     writes out [rows, 3 d]
constexpr int ATT_THREADS = 256;
constexpr size_t kAttSmemLimit = 200 * 1024;   // dynamic shared memory the attention kernel opts in to
template <bool kRound>
__global__ void __launch_bounds__(ATT_THREADS) attention_kernel(int sweep, const float* __restrict__ qkv, const float* __restrict__ in1,
                                                              const float* __restrict__ in2, const float* __restrict__ in3, int T, int heads,
                                                              int dh, float* __restrict__ P, float* __restrict__ Pd, float* __restrict__ out,
                                                              int accumulate) {
  constexpr bool round_out = kRound;
  pdl_prologue();
  extern __shared__ float sm[];
  const int b = blockIdx.x / heads, h = blockIdx.x % heads;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = ATT_THREADS / 32;
  const int d = heads * dh;
  const float scale = 1.0f / sqrtf((float)dh);
  float* sQ = sm;                 // [T][dh]
  float* sK = sQ + T * dh;
  float* sV = sK + T * dh;
  float* sA = sV + T * dh;        // [T][dh]  dO  /  Q'
  float* sB = sA + T * dh;        // [T][dh]         K'
  float* sC = sB + T * dh;        // [T][dh]         V'
  float* sP = sC + T * dh;        // [T][T]
  float* sM = sP + T * T;         // [T][T]  dS  (B)  /  P' (TF, TB)
  float* sN = sM + T * T;         // [T][T]  dS' (TB)
  float* sdO = sN + T * T;        // [T][dh] dO  (TB)
  float* sdOd = sdO + T * dh;     // [T][dh] dO' (TB)
  float* sdS = sdOd + T * dh;     // [T][T]  dS  (TB)
  const long long row0 = (long long)b * T;
  const long long pb = (long long)blockIdx.x * T * T;
  auto load_qkv = [&](const float* src, float* q, float* k, float* v) {
    for (int e = tid; e < T * dh; e += ATT_THREADS) {
      const int i = e / dh, c = e - i * dh;
      const float* r = src + (row0 + i) * 3 * d + h * dh + c;
      q[e] = r[0]; k[e] = r[d]; v[e] = r[2 * d];
    }
  };
  auto load_rows = [&](const float* src, float* dst) {   // [rows, d] -> this head's [T][dh]
    for (int e = tid; e < T * dh; e += ATT_THREADS) {
      const int i = e / dh, c = e - i * dh;
      dst[e] = src[(row0 + i) * d + h * dh + c];
    }
  };
  auto dot = [&](const float* x, const float* y) {
    float s = 0.f;
    for (int c = 0; c < dh; ++c) s = fmaf(x[c], y[c], s);
    return s;
  };
  auto store_qkv_grad = [&](int i, int c, float dq, float dk, float dv) {
    float* o = out + (row0 + i) * 3 * d + h * dh + c;
    const float vq = dq * scale, vk = dk * scale;
    const float rq = accumulate ? o[0] + vq : vq, rk = accumulate ? o[d] + vk : vk, rv = accumulate ? o[2 * d] + dv : dv;
    o[0] = round_out ? tf32_rna(rq) : rq;
    o[d] = round_out ? tf32_rna(rk) : rk;
    o[2 * d] = round_out ? tf32_rna(rv) : rv;
  };
  load_qkv(qkv, sQ, sK, sV);
  if (sweep == 0) {
    __syncthreads();
    for (int i = warp; i < T; i += nwarps) {                      // (A) softmax of row i
      float mx = -3.0e38f;
      for (int j = lane; j < T; j += 32) { const float sc = dot(sQ + i * dh, sK + j * dh) * scale; sP[i * T + j] = sc; mx = fmaxf(mx, sc); }
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      float den = 0.f;
      for (int j = lane; j < T; j += 32) { const float e = expf(sP[i * T + j] - mx); sP[i * T + j] = e; den += e; }
      den = warp_sum(den);
      const float rden = 1.0f / den;
      for (int j = lane; j < T; j += 32) { const float p = sP[i * T + j] * rden; sP[i * T + j] = p; P[pb + i * T + j] = p; }
    }
    __syncthreads();
    for (int e = tid; e < T * dh; e += ATT_THREADS) {             // (B) O = P V
      const int i = e / dh, c = e - i * dh;
      float o = 0.f;
      for (int j = 0; j < T; ++j) o = fmaf(sP[i * T + j], sV[j * dh + c], o);
      out[(row0 + i) * d + h * dh + c] = round_out ? tf32_rna(o) : o;
    }
    return;
  }
  for (int e = tid; e < T * T; e += ATT_THREADS) sP[e] = P[pb + e];
  if (sweep == 1) {
    load_rows(in1, sA);                                           // dO
    __syncthreads();
    for (int i = warp; i < T; i += nwarps) {                      // (A) dS = P (dP - r), dP_ij = dO_i . V_j, r = sum_j dP_ij P_ij
      float r = 0.f;
      for (int j = lane; j < T; j += 32) { const float dp = dot(sA + i * dh, sV + j * dh); sM[i * T + j] = dp; r = fmaf(dp, sP[i * T + j], r); }
      r = warp_sum(r);
      for (int j = lane; j < T; j += 32) sM[i * T + j] = sP[i * T + j] * (sM[i * T + j] - r);
    }
    __syncthreads();
    for (int e = tid; e < T * dh; e += ATT_THREADS) {             // (B)
      const int i = e / dh, c = e - i * dh;
      float dq = 0.f, dk = 0.f, dv = 0.f;
      for (int j = 0; j < T; ++j) {
        dq = fmaf(sM[i * T + j], sK[j * dh + c], dq);
        dk = fmaf(sM[j * T + i], sQ[j * dh + c], dk);
        dv = fmaf(sP[j * T + i], sA[j * dh + c], dv);
      }
      store_qkv_grad(i, c, dq, dk, dv);
    }
    return;
  }
  if (sweep == 2) {
    load_qkv(in1, sA, sB, sC);   // Q', K', V'
    __syncthreads();
    for (int i = warp; i < T; i += nwarps) {                      // (A) P' = P (S' - sum_j P S')
      float acc = 0.f;
      for (int j = lane; j < T; j += 32) {
        const float sd = (dot(sA + i * dh, sK + j * dh) + dot(sQ + i * dh, sB + j * dh)) * scale;
        sM[i * T + j] = sd;
        acc = fmaf(sP[i * T + j], sd, acc);
      }
      acc = warp_sum(acc);
      for (int j = lane; j < T; j += 32) { const float pd = sP[i * T + j] * (sM[i * T + j] - acc); sM[i * T + j] = pd; Pd[pb + i * T + j] = pd; }
    }
    __syncthreads();
    for (int e = tid; e < T * dh; e += ATT_THREADS) {             // (B) O' = P' V + P V'
      const int i = e / dh, c = e - i * dh;
      float o = 0.f;
      for (int j = 0; j < T; ++j) o += sM[i * T + j] * sV[j * dh + c] + sP[i * T + j] * sC[j * dh + c];
      out[(row0 + i) * d + h * dh + c] = round_out ? tf32_rna(o) : o;
    }
    return;
  }
  // sweep 3: tangent backward.  Needs Q', K', V' (in3), dO (in2), dO' (in1), P, P'.
  float* sQd = sA; float* sKd = sB; float* sVd = sC;
  load_qkv(in3, sQd, sKd, sVd);
  float* sPd = sM;                    // P'
  for (int e = tid; e < T * T; e += ATT_THREADS) sPd[e] = Pd[pb + e];
  load_rows(in2, sdO);
  load_rows(in1, sdOd);
  __syncthreads();
  for (int i = warp; i < T; i += nwarps) {                        // (A) dS, dS' of row i
    float r = 0.f, rd = 0.f;
    for (int j = lane; j < T; j += 32) {
      const float dp = dot(sdO + i * dh, sV + j * dh);
      const float dpd = dot(sdOd + i * dh, sV + j * dh) + dot(sdO + i * dh, sVd + j * dh);
      sdS[i * T + j] = dp;       // dP for now
      sN[i * T + j] = dpd;       // dP' for now
      r = fmaf(dp, sP[i * T + j], r);
      rd += dpd * sP[i * T + j] + dp * sPd[i * T + j];
    }
    r = warp_sum(r);
    rd = warp_sum(rd);
    for (int j = lane; j < T; j += 32) {
      const float dp = sdS[i * T + j], dpd = sN[i * T + j];
      sN[i * T + j] = sPd[i * T + j] * (dp - r) + sP[i * T + j] * (dpd - rd);   // dS'
      sdS[i * T + j] = sP[i * T + j] * (dp - r);                               // dS
    }
  }
  __syncthreads();
  for (int e = tid; e < T * dh; e += ATT_THREADS) {               // (B)
    const int i = e / dh, c = e - i * dh;
    float dq = 0.f, dk = 0.f, dv = 0.f;
    for (int j = 0; j < T; ++j) {
      dq += sN[i * T + j] * sK[j * dh + c] + sdS[i * T + j] * sKd[j * dh + c];
      dk += sN[j * T + i] * sQ[j * dh + c] + sdS[j * T + i] * sQd[j * dh + c];
      dv += sPd[j * T + i] * sdO[j * dh + c] + sP[j * T + i] * sdOd[j * dh + c];
    }
    store_qkv_grad(i, c, dq, dk, dv);
  }
}

// ---- positional embedding ------------------------------------------------------------------------------------------
template <bool kRound>
__global__ void posadd_kernel(const float* __restrict__ x, const float* __restrict__ pos, float* __restrict__ out, long long total, int C, int T) {
  constexpr bool round_out = kRound;
  pdl_prologue();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / C;
    const int c = (int)(i - row * C);
    const float v = pos[(row % T) * C + c];
    const float y = x != nullptr ? x[i] + v : v;
    out[i] = round_out ? tf32_rna(y) : y;
  }
}

__global__ void pos_grad_kernel(const float* __restrict__ d, float* __restrict__ g_pos, int rows, int C, int T) {
  pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;   // (t, c)
  if (i >= T * C) return;
  const int t = i / C, c = i - t * C;
  float s = 0.f;
  for (int b = 0; b < rows / T; ++b) s += d[((long long)b * T + t) * C + c];
  g_pos[i] = s;
}

// ---- next-token cross-entropy with probability targets ----------------------------------------------------------------
__device__ __forceinline__ void row_softmax_stats(const float* z, int V, double* scratch, float& mx_out, float& sum_out) {
  __shared__ float wmax[32];
  __shared__ float s_max, s_sum;
  float mx = -FLT_MAX;
  for (int c = threadIdx.x; c < V; c += blockDim.x) mx = fmaxf(mx, z[c]);
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x == 0) {
    float m = wmax[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) m = fmaxf(m, wmax[w]);
    s_max = m;
  }
  __syncthreads();
  mx = s_max;
  double part = 0.0;
  for (int c = threadIdx.x; c < V; c += blockDim.x) part += (double)expf(z[c] - mx);
  const double tot = block_sum(part, scratch);
  if (threadIdx.x == 0) s_sum = (float)tot;
  __syncthreads();
  mx_out = mx;
  sum_out = s_sum;
}

// softmax statistics of the row this cluster serves: (max, sum of exp) over all segments
__device__ __forceinline__ void cluster_softmax_stats(const float* z, int c0, int c1, RowReduce& ws, int slot0, float& mx_out, float& sum_out) {
  float mx = -FLT_MAX;
  for (int c = c0 + threadIdx.x; c < c1; c += kRowThreads) mx = fmaxf(mx, z[c]);
  mx = (float)row_allreduce<ROW_MAX>((double)mx, ws, slot0);
  double part = 0.0;
  for (int c = c0 + threadIdx.x; c < c1; c += kRowThreads) part += (double)expf(z[c] - mx);
  sum_out = (float)row_allreduce<ROW_SUM>(part, ws, slot0 + 1);
  mx_out = mx;
}

template <bool kRound>
__global__ void __launch_bounds__(kRowThreads, 2) token_ce_fwd_kernel(const float* __restrict__ logits, const float* __restrict__ q, int rows, int V,
                                                                  int Vs, int T, float* p, float* loss_n, float* dlogits) {
  constexpr bool round_out = kRound;
  pdl_prologue();
  __shared__ RowReduce ws;
  const int row = blockIdx.x;
  int c0, c1;
  row_segment(V, c0, c1);
  const float* z = logits + (long long)row * Vs;   // logits-shaped tensors: row stride Vs >= V (vocabulary padded for the GEMM tiles)
  const bool scored = (row % T) != T - 1;
  const float invM = 1.0f / (float)(rows - rows / T);
  const float* qn = q + (long long)(row + 1) * V;   // target of the next position (never read for the last position)
  if (seg_fits(V)) {   // the segment of the logits and of the target row in registers: one load each, two reductions instead of three
    SegCache zc, qc;
    seg_load(zc, z, c0, c1, -3.402823466e+38f);
    if (scored) seg_load(qc, qn, c0, c1, 0.f);
    float m;
    double dsum;
    seg_softmax_pair(zc, m, dsum);
    row_allreduce_softmax(m, dsum, ws, 0);
    const float fsum = (float)dsum, lse_c = m + logf(fsum);
    double lp = 0.0;
#pragma unroll
    for (int k = 0; k < kSegCache; ++k) {
      const int c = c0 + k * kRowThreads + (int)threadIdx.x;
      if (c >= c1) continue;
      const float pc = expf(zc.v[k] - m) / fsum;
      p[(long long)row * Vs + c] = pc;
      if (scored) {
        const float g = (pc - qc.v[k]) * invM;
        dlogits[(long long)row * Vs + c] = round_out ? tf32_rna(g) : g;
        lp -= (double)qc.v[k] * (double)(zc.v[k] - lse_c);
      } else {
        dlogits[(long long)row * Vs + c] = 0.f;
      }
    }
    const double lt = row_allreduce<ROW_SUM>(lp, ws, 2);
    if (threadIdx.x == 0 && cluster_rank() == 0) loss_n[row] = scored ? (float)(lt * (double)rows * (double)invM) : 0.f;
    cluster_exit();
    return;
  }
  float mx, sum;
  cluster_softmax_stats(z, c0, c1, ws, 0, mx, sum);
  const float lse = mx + logf(sum);
  double lpart = 0.0;
  for (int c = c0 + threadIdx.x; c < c1; c += kRowThreads) {
    const float pc = expf(z[c] - mx) / sum;
    p[(long long)row * Vs + c] = pc;
    if (scored) {
      const float qc = qn[c];
      const float g = (pc - qc) * invM;
      dlogits[(long long)row * Vs + c] = round_out ? tf32_rna(g) : g;
      lpart -= (double)qc * (double)(z[c] - lse);
    } else {
      dlogits[(long long)row * Vs + c] = 0.f;
    }
  }
  const double ltot = row_allreduce<ROW_SUM>(lpart, ws, 2);
  if (threadIdx.x == 0 && cluster_rank() == 0) loss_n[row] = scored ? (float)(ltot * (double)rows * (double)invM) : 0.f;
  cluster_exit();
}

template <bool kRound>
__global__ void __launch_bounds__(kRowThreads, 2) token_ce_tan_bwd_kernel(const float* __restrict__ p, const float* __restrict__ zdot, int rows, int V,
                                                                      int Vs, int T, float* tdl) {
  constexpr bool round_out = kRound;
  pdl_prologue();
  __shared__ RowReduce ws;
  const int row = blockIdx.x;
  int c0, c1;
  row_segment(V, c0, c1);
  const float* pp = p + (long long)row * Vs;
  const float* zz = zdot + (long long)row * Vs;
  const bool scored = (row % T) != T - 1;
  const float invM = 1.0f / (float)(rows - rows / T);
  if (seg_fits(V)) {
    SegCache pc, zc;
    seg_load(pc, pp, c0, c1, 0.f);
    seg_load(zc, zz, c0, c1, 0.f);
    double pr = 0.0;
#pragma unroll
    for (int k = 0; k < kSegCache; ++k) pr += (double)pc.v[k] * (double)zc.v[k];
    const float dt = (float)row_allreduce<ROW_SUM>(pr, ws, 0);
#pragma unroll
    for (int k = 0; k < kSegCache; ++k) {
      const int c = c0 + k * kRowThreads + (int)threadIdx.x;
      if (c >= c1) continue;
      const float g = scored ? pc.v[k] * (zc.v[k] - dt) * invM : 0.f;
      tdl[(long long)row * Vs + c] = round_out ? tf32_rna(g) : g;
    }
    cluster_exit();
    return;
  }
  double part = 0.0;
  for (int c = c0 + threadIdx.x; c < c1; c += kRowThreads) part += (double)pp[c] * (double)zz[c];
  const float dot = (float)row_allreduce<ROW_SUM>(part, ws, 0);
  for (int c = c0 + threadIdx.x; c < c1; c += kRowThreads) {
    const float g = scored ? pp[c] * (zz[c] - dot) * invM : 0.f;
    tdl[(long long)row * Vs + c] = round_out ? tf32_rna(g) : g;
  }
  cluster_exit();
}

__global__ void __launch_bounds__(kRowThreads, 2) token_label_grad_kernel(const float* __restrict__ logits, const float* __restrict__ p,
                                                                      const float* __restrict__ zdot, int rows, int V, int Vs, int T,
                                                                      float task_reg, float* __restrict__ out) {
  pdl_prologue();
  __shared__ RowReduce ws;
  const int row = blockIdx.x;                      // output row = target position (b, t); source = logits row (b, t - 1)
  int c0, c1;
  row_segment(V, c0, c1);
  float* o = out + (long long)row * V;
  if (row % T == 0) {                              // position 0 is never a target (uniform over the cluster: no barrier is skipped)
    for (int c = c0 + threadIdx.x; c < c1; c += kRowThreads) o[c] = 0.f;
    return;
  }
  const long long src = row - 1;
  const float* z = logits + src * Vs;
  const float* pp = p + src * Vs;
  const float* zz = zdot + src * Vs;
  if (seg_fits(V)) {
    // p and z-dot in registers; the logits of the (rare) task-regularised form are streamed (a third cached segment spills)
    SegCache pc, zc;
    seg_load(pc, pp, c0, c1, 0.f);
    seg_load(zc, zz, c0, c1, 0.f);
    double pr = 0.0;
#pragma unroll
    for (int k = 0; k < kSegCache; ++k) pr += (double)pc.v[k] * (double)zc.v[k];
    const float dt = (float)row_allreduce<ROW_SUM>(pr, ws, 0);
    float m = 0.f, fsum = 1.f;
    if (task_reg != 0.f) cluster_softmax_stats(z, c0, c1, ws, 1, m, fsum);
    const float iM = 1.0f / (float)(rows - rows / T);
    const float lse_c = m + logf(fsum);
#pragma unroll
    for (int k = 0; k < kSegCache; ++k) {
      const int c = c0 + k * kRowThreads + (int)threadIdx.x;
      if (c >= c1) continue;
      float v = -(zc.v[k] - dt) * iM;
      if (task_reg != 0.f) v -= task_reg * (z[c] - lse_c) * iM;
      o[c] = v;
    }
    cluster_exit();
    return;
  }
  double part = 0.0;
  for (int c = c0 + threadIdx.x; c < c1; c += kRowThreads) part += (double)pp[c] * (double)zz[c];
  const float dot = (float)row_allreduce<ROW_SUM>(part, ws, 0);
  float mx = 0.f, sum = 1.f;
  if (task_reg != 0.f) cluster_softmax_stats(z, c0, c1, ws, 1, mx, sum);
  const float invM = 1.0f / (float)(rows - rows / T);
  const float lse = mx + logf(sum);
  for (int c = c0 + threadIdx.x; c < c1; c += kRowThreads) {
    float v = -(zz[c] - dot) * invM;
    if (task_reg != 0.f) v -= task_reg * (z[c] - lse) * invM;
    o[c] = v;
  }
  cluster_exit();
}

}  // namespace

static int check_launch(const char* what) {
  const cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess) { set_error(std::string(what) + ": " + cudaGetErrorString(err)); return -2; }
  return 0;
}

int launch_token_layernorm(int sweep, const float* x, const float* in1, const float* in2, const float* in3, const float* gamma,
                           const float* beta, const float* v_gamma, const float* v_beta, float eps, int rows, int C, float* stats, float* out,
                           int accumulate, bool round_out, cudaStream_t s) {
  const int warps = 4;
  const cudaError_t lerr = launch_kernel(round_out ? layernorm_kernel<true> : layernorm_kernel<false>, dim3((rows + warps - 1) / warps), dim3(warps * 32), 0, s,
                                         1, sweep, x, in1, in2, in3, gamma, beta, v_gamma, v_beta, eps, rows, C, stats, out, accumulate);
  if (lerr != cudaSuccess) { set_error(std::string("token layernorm: ") + cudaGetErrorString(lerr)); return -2; }
  return check_launch("token layernorm");
}
int launch_token_ln_param_grad(const float* x, const float* dy, const float* stats, int rows, int C, float* g_gamma, float* g_beta,
                               cudaStream_t s) {
  const cudaError_t lerr = launch_kernel(layernorm_param_grad_kernel, dim3((C + 31) / 32), dim3(256), 0, s, 1, x, dy, stats, rows, C, g_gamma, g_beta);
  if (lerr != cudaSuccess) { set_error(std::string("token layernorm parameter gradient: ") + cudaGetErrorString(lerr)); return -2; }
  return check_launch("token layernorm parameter gradient");
}
int launch_token_attention(int sweep, const float* qkv, const float* in1, const float* in2, const float* in3, int B, int T, int heads, int dh,
                           float* P, float* Pd, float* out, int accumulate, bool round_out, cudaStream_t s) {
  // the whole head stays resident in shared memory (8 T dh + 4 T^2 floats) under the 200 KB opt-in; longer sequences need a tiled kernel
  const size_t smem = (size_t)(8LL * T * dh + 4LL * T * T) * sizeof(float);
  if (smem > kAttSmemLimit) {
    set_error("token attention: seq_len " + std::to_string(T) + " with head size " + std::to_string(dh) + " needs " + std::to_string(smem) +
              " B of shared memory, over the " + std::to_string(kAttSmemLimit) + " B opt-in limit of the resident-head kernel");
    return -4;
  }
  static bool attr_done = false;
  if (!attr_done) {
    if (cudaFuncSetAttribute(attention_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kAttSmemLimit) != cudaSuccess ||
        cudaFuncSetAttribute(attention_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kAttSmemLimit) != cudaSuccess) {
      set_error("token attention: shared memory opt-in failed");
      return -2;
    }
    attr_done = true;
  }
  const cudaError_t lerr = launch_kernel(round_out ? attention_kernel<true> : attention_kernel<false>, dim3(B * heads), dim3(ATT_THREADS), smem, s, 1, sweep,
                                         qkv, in1, in2, in3, T, heads, dh, P, Pd, out, accumulate);
  if (lerr != cudaSuccess) { set_error(std::string("token attention: ") + cudaGetErrorString(lerr)); return -2; }
  return check_launch("token attention");
}
int launch_token_posadd(const float* x, const float* pos, float* out, int rows, int C, int T, bool round_out, cudaStream_t s) {
  const long long total = (long long)rows * C;
  const cudaError_t lerr = launch_kernel(round_out ? posadd_kernel<true> : posadd_kernel<false>, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, s, 1, x,
                                         pos, out, total, C, T);
  if (lerr != cudaSuccess) { set_error(std::string("token posadd: ") + cudaGetErrorString(lerr)); return -2; }
  return check_launch("token posadd");
}
int launch_token_pos_grad(const float* d, float* g_pos, int rows, int C, int T, cudaStream_t s) {
  const cudaError_t lerr = launch_kernel(pos_grad_kernel, dim3((T * C + 255) / 256), dim3(256), 0, s, 1, d, g_pos, rows, C, T);
  if (lerr != cudaSuccess) { set_error(std::string("token positional gradient: ") + cudaGetErrorString(lerr)); return -2; }
  return check_launch("token positional gradient");
}
int launch_token_ce_fwd(const float* logits, const float* q, int rows, int V, int Vs, int T, float* p, float* loss_n, float* dlogits, bool round_out,
                        cudaStream_t s) {
  if (launch_row_kernel(round_out ? token_ce_fwd_kernel<true> : token_ce_fwd_kernel<false>, rows, V, s, logits, q, rows, V, Vs, T, p, loss_n, dlogits) !=
      cudaSuccess) { set_error("token cross-entropy: launch failed"); return -2; }
  return check_launch("token cross-entropy");
}
int launch_token_ce_tan_bwd(const float* p, const float* zdot, int rows, int V, int Vs, int T, float* tdlogits, bool round_out, cudaStream_t s) {
  if (launch_row_kernel(round_out ? token_ce_tan_bwd_kernel<true> : token_ce_tan_bwd_kernel<false>, rows, V, s, p, zdot, rows, V, Vs, T, tdlogits) !=
      cudaSuccess) { set_error("token cross-entropy tangent: launch failed"); return -2; }
  return check_launch("token cross-entropy tangent");
}
int launch_token_label_grad(const float* logits, const float* p, const float* zdot, int rows, int V, int Vs, int T, float task_reg,
                            float* out, cudaStream_t s) {
  if (launch_row_kernel(token_label_grad_kernel, rows, V, s, logits, p, zdot, rows, V, Vs, T, task_reg, out) != cudaSuccess) { set_error("token label gradient: launch failed"); return -2; }
  return check_launch("token label gradient");
}

// ---- token recovery (base_attack.py:123-167): nearest vocabulary embedding of every reconstructed position ---------------------------
// score[n][v] = <r_n - mean r_n, e_v - mean e_v> / |r_n - mean|^2 / |e_v - mean|^2   (squared norms: the reference's formula), token[n] =
// argmax_v (the smallest v among equal maxima, a NaN score counts as maximal like torch.argmax).  A block keeps the centred
// reconstructions transposed in shared memory; a warp walks its share of the vocabulary rows: it centres one row cooperatively, then lane
// n forms the dot product with reconstruction n (conflict-free column reads, broadcast embedding reads).  Stage 2 folds the per-block
// winners in block order.
constexpr int TM_THREADS = 256, TM_WARPS = TM_THREADS / 32;
__device__ __forceinline__ bool tm_better(float s, long long v, float best, long long bi) {
  if (bi < 0) return true;
  const bool sn = s != s, bn = best != best;
  if (sn != bn) return sn;
  if (!sn && s != best) return s > best;
  return v < bi;
}
__global__ void __launch_bounds__(TM_THREADS) token_match_partial_kernel(const float* __restrict__ rec, const float* __restrict__ emb,
                                                                        const long long* __restrict__ subset, int rows, int d, int V, int per_block,
                                                                        float* __restrict__ best_val, long long* __restrict__ best_idx) {
  extern __shared__ float tm_smem[];
  float* rc = tm_smem;                              // [d][33]: centred reconstructions of the current group of 32 rows, transposed
  float* rn = rc + (size_t)d * 33;                  // [32] squared norms
  float* ev = rn + 32;                              // [TM_WARPS][d] centred embedding row of each warp
  float* wv = ev + (size_t)TM_WARPS * d;            // [TM_WARPS][32] per-warp winners
  long long* wi = reinterpret_cast<long long*>((reinterpret_cast<uintptr_t>(wv + TM_WARPS * 32) + 7) & ~(uintptr_t)7);   // (odd d: keep the 8-byte alignment)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int v0 = blockIdx.x * per_block, v1 = min(V, v0 + per_block);
  for (int g0 = 0; g0 < rows; g0 += 32) {
    __syncthreads();
    for (int n = warp; n < 32; n += TM_WARPS) {     // centre reconstruction g0 + n (one warp per row)
      const bool ok = g0 + n < rows;
      float sum = 0.f;
      for (int k = lane; k < d; k += 32) sum += ok ? rec[(long long)(g0 + n) * d + k] : 0.f;
      const float mean = warp_sum(sum) / (float)d;
      float sq = 0.f;
      for (int k = lane; k < d; k += 32) {
        const float c = ok ? rec[(long long)(g0 + n) * d + k] - mean : 0.f;
        rc[k * 33 + n] = c;
        sq = fmaf(c, c, sq);
      }
      sq = warp_sum(sq);
      if (lane == 0) rn[n] = sq;
    }
    __syncthreads();
    float best = 0.f;
    long long bi = -1;
    float* e = ev + (size_t)warp * d;
    for (int v = v0 + warp; v < v1; v += TM_WARPS) {
      const float* src = emb + (subset != nullptr ? subset[v] : (long long)v) * d;
      float sum = 0.f;
      for (int k = lane; k < d; k += 32) sum += src[k];
      const float mean = warp_sum(sum) / (float)d;
      float sq = 0.f;
      __syncwarp();
      for (int k = lane; k < d; k += 32) { const float c = src[k] - mean; e[k] = c; sq = fmaf(c, c, sq); }
      sq = warp_sum(sq);
      __syncwarp();
      float dot = 0.f;
      for (int k = 0; k < d; ++k) dot = fmaf(rc[k * 33 + lane], e[k], dot);
      const float score = dot / rn[lane] / sq;
      if (tm_better(score, v, best, bi)) { best = score; bi = v; }
    }
    wv[warp * 32 + lane] = best;
    wi[warp * 32 + lane] = bi;
    __syncthreads();
    if (warp == 0 && g0 + lane < rows) {
      float b = wv[lane];
      long long i = wi[lane];
      for (int w = 1; w < TM_WARPS; ++w) {
        const long long cand = wi[w * 32 + lane];
        if (cand >= 0 && tm_better(wv[w * 32 + lane], cand, b, i)) { b = wv[w * 32 + lane]; i = cand; }
      }
      best_val[(long long)blockIdx.x * rows + g0 + lane] = b;
      best_idx[(long long)blockIdx.x * rows + g0 + lane] = i;
    }
  }
}
__global__ void token_match_final_kernel(const float* __restrict__ best_val, const long long* __restrict__ best_idx, int blocks, int rows,
                                         long long* __restrict__ tokens) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= rows) return;
  float b = 0.f;
  long long i = -1;
  for (int k = 0; k < blocks; ++k) {
    const long long cand = best_idx[(long long)k * rows + n];
    if (cand >= 0 && tm_better(best_val[(long long)k * rows + n], cand, b, i)) { b = best_val[(long long)k * rows + n]; i = cand; }
  }
  tokens[n] = i;
}

}  // namespace bre

extern "C" {

// Token recovery: tokens[n] = argmax_v of the reference's centred similarity between rec[n][:] and emb[v][:] (emb rows picked through
// `subset` [V] when non-null; the returned ids are positions in that list).  All pointers are device pointers.
int bre_token_match(const float* rec, const float* emb, const int64_t* subset, int32_t rows, int32_t d, int32_t V, int64_t* tokens,
                    void* stream) {
  using namespace bre;
  if (!rec || !emb || !tokens || rows < 1 || d < 1 || V < 1) { set_error("bre_token_match: bad arguments"); return -1; }
  const size_t smem = ((size_t)d * 33 + 32 + (size_t)TM_WARPS * d + TM_WARPS * 32) * sizeof(float) + (size_t)TM_WARPS * 32 * sizeof(long long) + 8;
  if (smem > 200 * 1024) { set_error("bre_token_match: embedding too wide for the resident kernel"); return -4; }
  cudaStream_t s = (cudaStream_t)stream;
  static bool attr_done = false;
  if (!attr_done) {
    if (cudaFuncSetAttribute(token_match_partial_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024) != cudaSuccess) {
      set_error("bre_token_match: shared memory opt-in failed");
      return -2;
    }
    attr_done = true;
  }
  int blocks = (V + 63) / 64;
  if (blocks > kNumSMs * 4) blocks = kNumSMs * 4;
  const int per_block = (V + blocks - 1) / blocks;
  blocks = (V + per_block - 1) / per_block;
  float* best_val = nullptr;
  long long* best_idx = nullptr;
  if (cudaMallocAsync((void**)&best_val, sizeof(float) * (size_t)blocks * rows, s) != cudaSuccess ||
      cudaMallocAsync((void**)&best_idx, sizeof(long long) * (size_t)blocks * rows, s) != cudaSuccess) {
    set_error("bre_token_match: scratch allocation failed");
    return -2;
  }
  token_match_partial_kernel<<<blocks, TM_THREADS, smem, s>>>(rec, emb, reinterpret_cast<const long long*>(subset), rows, d, V, per_block, best_val,
                                                             best_idx);
  token_match_final_kernel<<<(rows + 127) / 128, 128, 0, s>>>(best_val, best_idx, blocks, rows, reinterpret_cast<long long*>(tokens));
  const cudaError_t err = cudaGetLastError();
  cudaFreeAsync(best_val, s);
  cudaFreeAsync(best_idx, s);
  if (err != cudaSuccess) { set_error(std::string("bre_token_match failed: ") + cudaGetErrorString(err)); return -2; }
  return 0;
}

// Stand-alone LayerNorm sweeps over [rows, C] fp32 device tensors (see layernorm_kernel for the meaning of in1..in3 per sweep).
// sweep 1 additionally writes the parameter gradients when g_gamma / g_beta are non-null.
int bre_token_layernorm(int32_t sweep, const float* x, const float* in1, const float* in2, const float* in3, const float* gamma,
                        const float* beta, const float* v_gamma, const float* v_beta, float eps, int32_t rows, int32_t C, float* stats,
                        float* out, float* g_gamma, float* g_beta, int32_t round_out, void* stream) {
  using namespace bre;
  if (!x || !out || !stats || !gamma || rows < 1 || C < 1 || sweep < 0 || sweep > 3) { set_error("bre_token_layernorm: bad arguments"); return -1; }
  cudaStream_t s = (cudaStream_t)stream;
  int rc = launch_token_layernorm(sweep, x, in1, in2, in3, gamma, beta, v_gamma, v_beta, eps, rows, C, stats, out, 0, round_out != 0, s);
  if (rc == 0 && sweep == 1 && g_gamma && g_beta) rc = launch_token_ln_param_grad(x, in1, stats, rows, C, g_gamma, g_beta, s);
  return rc;
}

// Stand-alone attention sweeps: qkv [B*T, 3 d], P / Pd [B, heads, T, T] scratch kept by the caller between sweeps.
int bre_token_attention(int32_t sweep, const float* qkv, const float* in1, const float* in2, const float* in3, int32_t B, int32_t T,
                        int32_t heads, int32_t dh, float* P, float* Pd, float* out, int32_t round_out, void* stream) {
  using namespace bre;
  if (!qkv || !out || !P || B < 1 || T < 1 || heads < 1 || dh < 1 || sweep < 0 || sweep > 3) {
    set_error("bre_token_attention: bad arguments");
    return -1;
  }
  return launch_token_attention(sweep, qkv, in1, in2, in3, B, T, heads, dh, P, Pd, out, 0, round_out != 0, (cudaStream_t)stream);
}

}  // extern "C"
