// fp32 SIMT implicit-GEMM back end (CUDA cores).  Bit-faithful fp32 arithmetic: this is the parity
// back end and the fallback for shapes the TF32 tensor-core back end (igemm_tc.cu) does not cover
// (tiny channel counts such as the 3-channel stem, ragged K).
//
// Tile 64x64x16, 256 threads, 4x4 outputs per thread, register-prefetch double buffering, deterministic
// split-K (partials to a workspace, the last-arriving CTA of a tile reduces them in fixed order).
#include <stdlib.h>

#include "igemm.cuh"

namespace bre {

namespace {

struct Dims {
  int M, Nc, K;
  int steps_per_src, total_steps, steps_per_split;
  int vecA, vecB, vecOut;
};

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

template <int MODE>
__global__ void __launch_bounds__(IG_THREADS) igemm_simt_kernel(GemmArgs a, Dims d) {
  pdl_prologue();
  __shared__ __align__(16) float As[2][IG_BK][IG_BM + 4];
  __shared__ __align__(16) float Bs[2][IG_BK][IG_BN + 4];
  __shared__ int s_last;

  const ConvGeom g = a.g;
  const int tid = threadIdx.x;
  const int m0 = blockIdx.x * IG_BM, n0 = blockIdx.y * IG_BN;
  const int z = blockIdx.z;
  const int s_begin = z * d.steps_per_split;
  const int s_end = min(d.total_steps, s_begin + d.steps_per_split);

  // thread mappings of the two loader flavours
  const int kc_row = tid >> 2, kc_k = (tid & 3) << 2;    // K-contiguous operand: 1 row, 4 consecutive k
  const int mc_k = tid >> 4, mc_col = (tid & 15) << 2;   // M/N-contiguous operand: 1 k, 4 consecutive rows
  const int HoWo = g.Ho * g.Wo, HW = g.H * g.W;

  // ---- per-thread fixed decode -----------------------------------------------------------------
  // FPROP A / DGRAD A: one row (pixel) per thread
  bool a_valid = false;
  int a_img = 0, a_y = 0, a_x = 0;   // FPROP: (h0, w0) = top-left of the window ; DGRAD: (h, w) of the input pixel
  if (MODE == GEMM_FPROP) {
    const int m = m0 + kc_row;
    a_valid = m < d.M;
    if (a_valid) {
      a_img = m / HoWo;
      const int rem = m - a_img * HoWo;
      const int p = rem / g.Wo, q = rem - p * g.Wo;
      a_y = p * g.stride - g.pad;
      a_x = q * g.stride - g.pad;
    }
  } else if (MODE == GEMM_DGRAD) {
    const int m = m0 + kc_row;
    a_valid = m < d.M;
    if (a_valid) {
      a_img = m / HW;
      const int rem = m - a_img * HW;
      a_y = rem / g.W;
      a_x = rem - a_y * g.W;
    }
  }
  // WGRAD B: 4 consecutive columns n = (rs, c)
  int wb_c = 0, wb_r = 0, wb_s = 0;
  if (MODE == GEMM_WGRAD) {
    const int n = n0 + mc_col;
    if (n < d.Nc) {
      const int rs = n / g.Ci;
      wb_c = n - rs * g.Ci;
      wb_r = rs / g.S;
      wb_s = rs - wb_r * g.S;
    }
  }

  float ra[4], rb[4];

  auto load_tiles = [&](int step) {
    const int src = step / d.steps_per_src;
    const int kbase = (step - src * d.steps_per_src) * IG_BK;
    const float* __restrict__ act = a.act[src];
    const float* __restrict__ wgt = a.wgt[src];
#pragma unroll
    for (int j = 0; j < 4; ++j) { ra[j] = 0.f; rb[j] = 0.f; }

    if (MODE == GEMM_FPROP) {
      // A(m, k) = in[img, h0 + r, w0 + s, c],  k = (r, s, c)
      const int kk = kbase + kc_k;
      if (a_valid && kk < d.K) {
        if (d.vecA) {
          const int rs = kk / g.Ci, c = kk - rs * g.Ci;
          const int r = rs / g.S, s = rs - r * g.S;
          const int h = a_y + r, w = a_x + s;
          if (h >= 0 && h < g.H && w >= 0 && w < g.W) {
            const float4 v = ldg4(act + a_img * a.x_sN + (long long)(h * g.W + w) * a.x_sP + c);
            ra[0] = v.x; ra[1] = v.y; ra[2] = v.z; ra[3] = v.w;
          }
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int kj = kk + j;
            if (kj < d.K) {
              const int rs = kj / g.Ci, c = kj - rs * g.Ci;
              const int r = rs / g.S, s = rs - r * g.S;
              const int h = a_y + r, w = a_x + s;
              if (h >= 0 && h < g.H && w >= 0 && w < g.W)
                ra[j] = __ldg(act + a_img * a.x_sN + (long long)(h * g.W + w) * a.x_sP + (long long)c * a.x_sC);
            }
          }
        }
      }
      // B(n, k) = W[n][k]
      const int n = n0 + kc_row;
      if (n < d.Nc && kk < d.K) {
        const float* wp = wgt + (long long)n * d.K + kk;
        if (d.vecB) {
          const float4 v = ldg4(wp);
          rb[0] = v.x; rb[1] = v.y; rb[2] = v.z; rb[3] = v.w;
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (kk + j < d.K) rb[j] = __ldg(wp + j);
        }
      }
    } else if (MODE == GEMM_DGRAD) {
      // A(m, k) = dout[img, (h + pad - r)/stride, (w + pad - s)/stride, ko],  k = (r, s, ko)
      const int kk = kbase + kc_k;
      if (a_valid && kk < d.K) {
        if (d.vecA) {
          const int rs = kk / g.Co, ko = kk - rs * g.Co;
          const int r = rs / g.S, s = rs - r * g.S;
          const int hp = a_y + g.pad - r, wp = a_x + g.pad - s;
          if (hp >= 0 && wp >= 0) {
            const int p = hp / g.stride, q = wp / g.stride;
            if (p * g.stride == hp && q * g.stride == wp && p < g.Ho && q < g.Wo) {
              const float4 v = ldg4(act + ((long long)(a_img * g.Ho + p) * g.Wo + q) * g.Co + ko);
              ra[0] = v.x; ra[1] = v.y; ra[2] = v.z; ra[3] = v.w;
            }
          }
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int kj = kk + j;
            if (kj < d.K) {
              const int rs = kj / g.Co, ko = kj - rs * g.Co;
              const int r = rs / g.S, s = rs - r * g.S;
              const int hp = a_y + g.pad - r, wp = a_x + g.pad - s;
              if (hp >= 0 && wp >= 0) {
                const int p = hp / g.stride, q = wp / g.stride;
                if (p * g.stride == hp && q * g.stride == wp && p < g.Ho && q < g.Wo)
                  ra[j] = __ldg(act + ((long long)(a_img * g.Ho + p) * g.Wo + q) * g.Co + ko);
              }
            }
          }
        }
      }
      // B(n = ci, k) = W[ko][r][s][ci]
      const int k1 = kbase + mc_k;
      const int n = n0 + mc_col;
      if (k1 < d.K && n < d.Nc) {
        const int rs = k1 / g.Co, ko = k1 - rs * g.Co;
        const float* wp = wgt + ((long long)ko * (g.R * g.S) + rs) * g.Ci + n;
        if (d.vecB) {
          const float4 v = ldg4(wp);
          rb[0] = v.x; rb[1] = v.y; rb[2] = v.z; rb[3] = v.w;
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (n + j < d.Nc) rb[j] = __ldg(wp + j);
        }
      }
    } else {  // GEMM_WGRAD
      const int k1 = kbase + mc_k;  // pixel (img, p, q)
      if (k1 < d.K) {
        // A(m = ko, k) = dout[pixel][ko]
        const int m = m0 + mc_col;
        if (m < d.M) {
          const float* dp = wgt + (long long)k1 * g.Co + m;
          if (d.vecA) {
            const float4 v = ldg4(dp);
            ra[0] = v.x; ra[1] = v.y; ra[2] = v.z; ra[3] = v.w;
          } else {
#pragma unroll
            for (int j = 0; j < 4; ++j)
              if (m + j < d.M) ra[j] = __ldg(dp + j);
          }
        }
        // B(n = (r, s, c), k) = in[img, p*stride - pad + r, q*stride - pad + s, c]
        const int n = n0 + mc_col;
        if (n < d.Nc) {
          const int img = k1 / HoWo;
          const int rem = k1 - img * HoWo;
          const int p = rem / g.Wo, q = rem - p * g.Wo;
          const int hb = p * g.stride - g.pad, wb = q * g.stride - g.pad;
          if (d.vecB) {
            const int h = hb + wb_r, w = wb + wb_s;
            if (h >= 0 && h < g.H && w >= 0 && w < g.W) {
              const float4 v = ldg4(act + img * a.x_sN + (long long)(h * g.W + w) * a.x_sP + wb_c);
              rb[0] = v.x; rb[1] = v.y; rb[2] = v.z; rb[3] = v.w;
            }
          } else {
            int c = wb_c, r = wb_r, s = wb_s;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              if (n + j < d.Nc) {
                const int h = hb + r, w = wb + s;
                if (h >= 0 && h < g.H && w >= 0 && w < g.W)
                  rb[j] = __ldg(act + img * a.x_sN + (long long)(h * g.W + w) * a.x_sP + (long long)c * a.x_sC);
              }
              if (++c == g.Ci) { c = 0; if (++s == g.S) { s = 0; ++r; } }
            }
          }
        }
      }
    }
  };

  auto store_tiles = [&](int buf) {
    if (MODE == GEMM_FPROP) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        As[buf][kc_k + j][kc_row] = ra[j];
        Bs[buf][kc_k + j][kc_row] = rb[j];
      }
    } else if (MODE == GEMM_DGRAD) {
#pragma unroll
      for (int j = 0; j < 4; ++j) As[buf][kc_k + j][kc_row] = ra[j];
      *reinterpret_cast<float4*>(&Bs[buf][mc_k][mc_col]) = make_float4(rb[0], rb[1], rb[2], rb[3]);
    } else {
      *reinterpret_cast<float4*>(&As[buf][mc_k][mc_col]) = make_float4(ra[0], ra[1], ra[2], ra[3]);
      *reinterpret_cast<float4*>(&Bs[buf][mc_k][mc_col]) = make_float4(rb[0], rb[1], rb[2], rb[3]);
    }
  };

  const int ty = tid >> 4, tx = tid & 15;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  if (s_begin < s_end) {
    load_tiles(s_begin);
    store_tiles(0);
  }
  __syncthreads();
  for (int step = s_begin; step < s_end; ++step) {
    const int buf = (step - s_begin) & 1;
    const bool more = step + 1 < s_end;
    if (more) load_tiles(step + 1);
#pragma unroll
    for (int kk = 0; kk < IG_BK; ++kk) {
      const float4 av = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4]);
      const float4 bv = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
      const float ar[4] = {av.x, av.y, av.z, av.w};
      const float br[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ar[i], br[j], acc[i][j]);
    }
    if (more) store_tiles(buf ^ 1);
    __syncthreads();
  }

  // ---- split-K: deterministic reduction by the last-arriving CTA of this output tile --------------
  const int splits = gridDim.z;
  if (splits > 1) {
    const int tile = blockIdx.y * gridDim.x + blockIdx.x;
    float* wsb = a.ws + ((long long)tile * splits + z) * (IG_BM * IG_BN);
#pragma unroll
    for (int i = 0; i < 4; ++i)
      *reinterpret_cast<float4*>(wsb + (ty * 4 + i) * IG_BN + tx * 4) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
    __threadfence();
    __syncthreads();
    if (tid == 0) {
      const int prev = atomicAdd(a.counters + tile, 1);
      s_last = (prev == splits - 1);
      if (s_last) a.counters[tile] = 0;  // self-reset for the next launch
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    const float* wst = a.ws + (long long)tile * splits * (IG_BM * IG_BN);
    for (int zz = 0; zz < splits; ++zz) {
      const float* p = wst + (long long)zz * (IG_BM * IG_BN);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float4 v = __ldcg(reinterpret_cast<const float4*>(p + (ty * 4 + i) * IG_BN + tx * 4));
        acc[i][0] += v.x; acc[i][1] += v.y; acc[i][2] += v.z; acc[i][3] += v.w;
      }
    }
  }

  // ---- epilogue ----------------------------------------------------------------------------------
  const int n = n0 + tx * 4;
  if (n >= d.Nc) return;
  float bias4[4] = {0.f, 0.f, 0.f, 0.f};
  if (MODE == GEMM_FPROP && a.bias != nullptr) {
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (n + j < d.Nc) bias4[j] = __ldg(a.bias + n + j);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= d.M) continue;
    long long row;
    int cs = 1;
    if (MODE == GEMM_DGRAD) {
      const int img = m / HW;
      row = img * a.x_sN + (long long)(m - img * HW) * a.x_sP;
      cs = a.x_sC;
    } else {
      row = (long long)m * d.Nc;
    }
    float* op = a.out + row + (long long)n * cs;
    if (d.vecOut) {
      float4 v = make_float4(acc[i][0] + bias4[0], acc[i][1] + bias4[1], acc[i][2] + bias4[2], acc[i][3] + bias4[3]);
      if (a.accumulate) {
        const float4 o = *reinterpret_cast<const float4*>(op);
        v.x += o.x; v.y += o.y; v.z += o.z; v.w += o.w;
      }
      *reinterpret_cast<float4*>(op) = v;
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (n + j < d.Nc) {
          float v = acc[i][j] + bias4[j];
          float* q = op + (long long)j * cs;
          if (a.accumulate) v += *q;
          *q = v;
        }
      }
    }
  }
}

// ---- dgrad onto a tensor with very few channels (the 3-channel candidate behind the stem conv) ----------------
// The GEMM formulation would run an N=64-wide tile for Ci=3 columns and multiply stride^2-1 out of stride^2 taps by
// structural zeros.  Here one thread owns one input pixel and all CI channels, walks only the taps that hit the
// output grid, and streams dout with 128-bit loads; lanes of a warp are mapped to pixels of the same stride-parity
// class so the tap loop is warp-uniform and the weight loads are broadcasts.
// Weights of the taps that can hit this block's image row are staged once in shared memory as [src][tap][ko][ci]
// (12 consecutive floats per 4 output channels -> three broadcast LDS.128 feed 48 FMAs); each thread owns PX pixels of
// one stride-parity class so every weight fetched from shared memory is reused PX times.
constexpr int SC_PX = 4;
constexpr int SC_KCH = 4;   // 16-byte chunks of output channels per warp and tap (Co <= 64)
template <int CI>
__global__ void __launch_bounds__(128) dgrad_small_ci_kernel(GemmArgs a, int n_r, int smem_floats, int vec) {
  pdl_prologue();
  extern __shared__ __align__(16) float wsm[];            // [nsrc][n_r * S][Co][CI], then the reduction scratch
  const ConvGeom g = a.g;
  const int img = blockIdx.z, h = blockIdx.y;
  const int lane = threadIdx.x & 31, kq = threadIdx.x >> 5;  // warp = quarter of the output-channel range
  const int Wc = (g.W + g.stride - 1) / g.stride;
  // valid filter rows for this image row: r = r0 + t * stride, p = p0 - t
  const int hb = h + g.pad;
  const int r0 = hb % g.stride, p0 = hb / g.stride;
  const int taps = n_r * g.S;
  for (int e = threadIdx.x; e < g.Co * CI; e += 128) {     // (ko, c) fixed per thread; no divisions in the copy loops
    const int ko = e / CI, c = e - ko * CI;
    for (int src = 0; src < a.nsrc; ++src)
      for (int tr = 0; tr < n_r; ++tr) {
        const int r = r0 + tr * g.stride;
        for (int s = 0; s < g.S; ++s) {
          float* dst = wsm + ((src * taps + tr * g.S + s) * g.Co + ko) * CI + c;
          if (r < g.R) {
            const float* gp = a.wgt[src] + ((long long)ko * (g.R * g.S) + r * g.S + s) * g.Ci + c;
            asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((uint32_t)__cvta_generic_to_shared(dst)), "l"(gp) : "memory");
          } else {
            *dst = 0.f;
          }
        }
      }
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncthreads();
  float* red = wsm + smem_floats;  // reduction scratch behind the weights: [4][32][SC_PX * CI]
  {
  const int Wcp = ((Wc + SC_PX - 1) / SC_PX) * SC_PX;     // per-class slot range padded so that a thread never straddles classes
  const int slot0 = (blockIdx.x * 32 + lane) * SC_PX;   // SC_PX consecutive slots of one class
  const int cls = slot0 / Wcp;
  const int kper = ((g.Co + 15) / 16) * 4;               // output channels per warp, multiple of 4
  const int ko_lo = kq * kper, ko_hi = min(g.Co, ko_lo + kper);
  float acc[SC_PX][CI];
#pragma unroll
  for (int px = 0; px < SC_PX; ++px)
#pragma unroll
    for (int c = 0; c < CI; ++c) acc[px][c] = 0.f;
  int wpix[SC_PX];
  bool pvalid[SC_PX];
#pragma unroll
  for (int px = 0; px < SC_PX; ++px) {
    const int idx = slot0 + px - cls * Wcp;
    wpix[px] = idx * g.stride + cls;
    pvalid[px] = cls < g.stride && idx < Wc && wpix[px] < g.W;
  }
  if (cls < g.stride) {
    const int xb = cls + g.pad;
    const int s0 = xb % g.stride;                          // valid filter columns: s = s0 + u * stride, same for the whole class
    for (int src = 0; src < a.nsrc; ++src) {
      const float* __restrict__ dout = a.act[src];
      for (int tr = 0; tr < n_r; ++tr) {
        const int r = r0 + tr * g.stride, p = p0 - tr;
        if (r >= g.R || p < 0 || p >= g.Ho) continue;
        for (int s = s0; s < g.S; s += g.stride) {
          const float* wt = wsm + ((long long)(src * taps + tr * g.S + s) * g.Co) * CI;
          const float* dp[SC_PX];
          bool ok[SC_PX];
#pragma unroll
          for (int px = 0; px < SC_PX; ++px) {
            const int wp = wpix[px] + g.pad - s;
            const int q = wp / g.stride;
            ok[px] = pvalid[px] && wp >= 0 && q < g.Wo;
            dp[px] = dout + ((long long)(img * g.Ho + p) * g.Wo + (ok[px] ? q : 0)) * g.Co;
          }
          // the warp's slice of output channels is at most SC_KCH * 4 wide: issue every dout load of this tap first
          float4 dv[SC_KCH][SC_PX];
#pragma unroll
          for (int kc = 0; kc < SC_KCH; ++kc) {
            const int ko = ko_lo + 4 * kc;
#pragma unroll
            for (int px = 0; px < SC_PX; ++px) {
              dv[kc][px] = make_float4(0.f, 0.f, 0.f, 0.f);
              if (ok[px] && ko < ko_hi) {
                if (vec) dv[kc][px] = __ldg(reinterpret_cast<const float4*>(dp[px] + ko));
                else {
                  float t4[4] = {0.f, 0.f, 0.f, 0.f};
                  for (int j = 0; j < 4; ++j)
                    if (ko + j < g.Co) t4[j] = __ldg(dp[px] + ko + j);
                  dv[kc][px] = make_float4(t4[0], t4[1], t4[2], t4[3]);
                }
              }
            }
          }
#pragma unroll
          for (int kc = 0; kc < SC_KCH; ++kc) {
            const int ko = ko_lo + 4 * kc;
            if (ko >= ko_hi) break;
            float wv[4 * CI];
#pragma unroll
            for (int e = 0; e < 4 * CI; ++e) wv[e] = (ko + e / CI < g.Co) ? wt[ko * CI + e] : 0.f;
#pragma unroll
            for (int px = 0; px < SC_PX; ++px) {
              const float dd[4] = {dv[kc][px].x, dv[kc][px].y, dv[kc][px].z, dv[kc][px].w};
#pragma unroll
              for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int c = 0; c < CI; ++c) acc[px][c] = fmaf(dd[j], wv[j * CI + c], acc[px][c]);
            }
          }
        }
      }
    }
  }
  // sum the four output-channel quarters through shared memory
  __syncthreads();
#pragma unroll
  for (int px = 0; px < SC_PX; ++px)
#pragma unroll
    for (int c = 0; c < CI; ++c) red[(kq * 32 + lane) * (SC_PX * CI) + px * CI + c] = acc[px][c];
  __syncthreads();
  if (kq == 0) {
#pragma unroll
  for (int px = 0; px < SC_PX; ++px) {
    if (!pvalid[px]) continue;
    float* op = a.out + img * a.x_sN + (long long)(h * g.W + wpix[px]) * a.x_sP;
#pragma unroll
    for (int c = 0; c < CI; ++c) {
      const int e = px * CI + c;
      const float v = ((red[lane * (SC_PX * CI) + e] + red[(32 + lane) * (SC_PX * CI) + e]) + red[(64 + lane) * (SC_PX * CI) + e]) +
                      red[(96 + lane) * (SC_PX * CI) + e];
      float* q = op + (long long)c * a.x_sC;
      *q = a.accumulate ? *q + v : v;
    }
  }
  }
 }
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

bool dgrad_small_ci_fits(const GemmArgs& a) {
  const ConvGeom& g = a.g;
  return a.mode == GEMM_DGRAD && g.Ci <= 4 && g.Co <= 16 * SC_KCH && g.H <= 65535 && g.N <= 65535 &&
         (size_t)a.nsrc * ((g.R + g.stride - 1) / g.stride) * g.S * g.Co * g.Ci * 4 <= 200 * 1024;
}

GemmPlan dgrad_small_ci_plan(const GemmArgs& a) {
  bool vec = a.g.Co % 4 == 0;
  for (int q = 0; q < a.nsrc; ++q) vec = vec && aligned16(a.act[q]);
  GemmPlan p;
  p.family = GEMM_FAM_DGRAD_SMALL_CI; p.mode = a.mode; p.nsrc = a.nsrc;
  p.tile_rows = 32 * SC_PX; p.tile_width = a.g.Ci; p.vec = vec ? 1 : 0;
  return p;
}

int launch_dgrad_small_ci(const GemmArgs& a, const GemmPlan& p, cudaStream_t stream) {
  const ConvGeom& g = a.g;
  const int Wc = (g.W + g.stride - 1) / g.stride;
  const int n_r = (g.R + g.stride - 1) / g.stride;   // filter rows that can hit one image row
  const int wfloats = a.nsrc * n_r * g.S * g.Co * g.Ci;
  const int rfloats = 4 * 32 * SC_PX * g.Ci;
  const int smem_floats = (wfloats + 3) & ~3;   // weights, then the reduction scratch
  const size_t smem = (size_t)(smem_floats + rfloats) * sizeof(float);
  if (smem > 200 * 1024) { set_error("dgrad_small_ci: filter too large for shared memory"); return -4; }
  const int Wcp = ((Wc + SC_PX - 1) / SC_PX) * SC_PX;
  dim3 grid(ceil_div((long long)Wcp * g.stride, 32 * SC_PX), g.H, g.N), block(128);
#define BRE_LAUNCH_SC(CI_)                                                                                              \
  do {                                                                                                                  \
    static size_t cap = 0;                                                                                              \
    if (smem > 48 * 1024 && smem > cap) {                                                                               \
      BRE_CUDA_CHECK(cudaFuncSetAttribute(dgrad_small_ci_kernel<CI_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
      cap = smem;                                                                                                       \
    }                                                                                                                   \
    BRE_KLAUNCH((dgrad_small_ci_kernel<CI_>), grid, block, smem, stream, a, n_r, smem_floats, p.vec);                                   \
  } while (0)
  switch (g.Ci) {
    case 1: BRE_LAUNCH_SC(1); break;
    case 2: BRE_LAUNCH_SC(2); break;
    case 3: BRE_LAUNCH_SC(3); break;
    default: BRE_LAUNCH_SC(4); break;
  }
#undef BRE_LAUNCH_SC
  BRE_CHECK_LAUNCH();
  return 0;
}

GemmPlan simt_plan(const GemmArgs& a) {
  const ConvGeom& g = a.g;
  int M, Nc, K;
  gemm_dims(a, M, Nc, K);
  bool ptr_ok = true;
  for (int s = 0; s < a.nsrc; ++s) ptr_ok = ptr_ok && aligned16(a.act[s]) && aligned16(a.wgt[s]);
  const bool x_vec = (a.x_sC == 1) && (g.Ci % 4 == 0) && (a.x_sP % 4 == 0) && (a.x_sN % 4 == 0);
  bool vecA, vecB, vecOut;
  if (a.mode == GEMM_FPROP) {
    vecA = ptr_ok && x_vec;
    vecB = ptr_ok && (K % 4 == 0);
    vecOut = aligned16(a.out) && (Nc % 4 == 0);
  } else if (a.mode == GEMM_DGRAD) {
    vecA = ptr_ok && (g.Co % 4 == 0);
    vecB = ptr_ok && (g.Ci % 4 == 0);
    vecOut = aligned16(a.out) && x_vec;
  } else {
    vecA = ptr_ok && (g.Co % 4 == 0);
    vecB = ptr_ok && x_vec;
    vecOut = aligned16(a.out) && (Nc % 4 == 0);
  }
  const int total = ceil_div(K, IG_BK) * a.nsrc;
  const long long tiles = (long long)ceil_div(M, IG_BM) * ceil_div(Nc, IG_BN);
  int splits = 1;
  if (tiles < 2 * kNumSMs) {
    splits = ceil_div(2 * kNumSMs, tiles);
    const int max_by_k = total / 4 > 0 ? total / 4 : 1;
    if (splits > max_by_k) splits = max_by_k;
  }
  if (splits > total) splits = total;
  if (splits > 1 && (a.ws == nullptr || a.counters == nullptr)) splits = 1;
  if (splits > 1 && tiles * splits > a.ws_tiles) splits = (int)(a.ws_tiles / tiles) > 1 ? (int)(a.ws_tiles / tiles) : 1;
  GemmPlan p;
  p.family = GEMM_FAM_SIMT; p.mode = a.mode; p.nsrc = a.nsrc;
  p.tile_rows = IG_BM; p.tile_width = IG_BN; p.stages = 2;
  p.total_kblocks = total; p.kblocks_per_split = ceil_div(total, splits);
  p.splits = ceil_div(total, p.kblocks_per_split);  // no empty splits
  p.vec = (vecA ? 1 : 0) | (vecB ? 2 : 0) | (vecOut ? 4 : 0);
  return p;
}

int launch_igemm_simt(const GemmArgs& a, const GemmPlan& p, cudaStream_t stream) {
  Dims d;
  gemm_dims(a, d.M, d.Nc, d.K);
  d.steps_per_src = ceil_div(d.K, IG_BK);
  d.total_steps = p.total_kblocks;
  d.steps_per_split = p.kblocks_per_split;
  d.vecA = p.vec & 1; d.vecB = (p.vec >> 1) & 1; d.vecOut = (p.vec >> 2) & 1;
  const int tm = ceil_div(d.M, IG_BM), tn = ceil_div(d.Nc, IG_BN);
  if (tn > 65535 || p.splits > 65535) { set_error("igemm: grid too large"); return -1; }
  dim3 grid(tm, tn, p.splits), block(IG_THREADS);
  if (a.mode == GEMM_FPROP) BRE_KLAUNCH((igemm_simt_kernel<GEMM_FPROP>), grid, block, 0, stream, a, d);
  else if (a.mode == GEMM_DGRAD) BRE_KLAUNCH((igemm_simt_kernel<GEMM_DGRAD>), grid, block, 0, stream, a, d);
  else BRE_KLAUNCH((igemm_simt_kernel<GEMM_WGRAD>), grid, block, 0, stream, a, d);
  BRE_CHECK_LAUNCH();
  return 0;
}

thread_local GemmPlan g_last_plan;

}  // namespace

const GemmPlan& last_gemm_plan() { return g_last_plan; }

const GemmSwitches& gemm_switches() {
  static const GemmSwitches sw = [] {
    auto getenv_or = [](const char* name, int dflt) { const char* e = getenv(name); return e ? atoi(e) : dflt; };
    GemmSwitches s;
    s.tc_tma = getenv_or("BRE_TC_TMA", 1);
    s.tc_strided_tma = getenv_or("BRE_TC_STRIDED_TMA", 1);
    s.tc_narrow = getenv_or("BRE_TC_NARROW", 1);
    s.tc_stream = getenv_or("BRE_TC_STREAM", 1);
    s.tc_stages = getenv_or("BRE_TC_STAGES", 0);
    s.tc_shortk_stages = getenv_or("BRE_TC_SHORTK_STAGES", 2);
    s.tc_max_splits = getenv_or("BRE_TC_MAX_SPLITS", 0);
    s.tc_target_ctas = getenv_or("BRE_TC_TARGET_CTAS", 0);
    s.tc_proxy_fence = getenv_or("BRE_TC_PROXY_FENCE", 0);
    s.tc_prefetch = getenv_or("BRE_TC_PREFETCH", 1);
    s.tc_producers = getenv_or("BRE_TC_PRODUCERS", 2);
    if (s.tc_producers < 1 || s.tc_producers > 4) s.tc_producers = 2;
    s.linear_small = getenv_or("BRE_LINEAR_SMALL", 1);
    s.linear_small_rows = getenv_or("BRE_LINEAR_SMALL_ROWS", 0);
    s.linear_tall = getenv_or("BRE_LINEAR_TALL", 1);
    return s;
  }();
  return sw;
}

// The family order of every GEMM, for all back ends: the tall-K linear dgrad, the small-row linear kernels where they are
// preferred, the tensor cores where they cover the shape, then the fp32 kernels -- the small-row linear kernels, the small-channel
// dgrad, the SIMT implicit GEMM.
GemmPlan plan_gemm(const GemmArgs& a, int backend) {
  if (linear_tall_supported(a)) return linear_tall_plan(a);
  if (backend != 1 && linear_small_preferred(a)) return linear_small_plan(a);
  if (backend != 0 && igemm_tc_supported(a)) return tc_plan(a, true);
  if (backend == 1) return GemmPlan();
  if (gemm_switches().linear_small && a.g.N <= 16 && linear_small_supported(a)) return linear_small_plan(a);
  if (dgrad_small_ci_fits(a)) return dgrad_small_ci_plan(a);
  return simt_plan(a);
}

int launch_gemm(const GemmArgs& a, int backend, cudaStream_t stream) {
  int M, Nc, K;
  gemm_dims(a, M, Nc, K);
  if (M <= 0 || Nc <= 0 || K <= 0 || a.nsrc < 1 || a.nsrc > 2) { set_error("igemm: empty problem or bad nsrc"); return -1; }
  GemmPlan p = plan_gemm(a, backend);
  int rc;
  switch (p.family) {
    case GEMM_FAM_LINEAR_TALL: rc = launch_linear_tall(a, p, stream); break;
    case GEMM_FAM_LINEAR_SMALL: rc = launch_linear_small(a, p, stream); break;
    case GEMM_FAM_TC: rc = launch_igemm_tc(a, p, stream); break;
    case GEMM_FAM_DGRAD_SMALL_CI: rc = launch_dgrad_small_ci(a, p, stream); break;
    case GEMM_FAM_SIMT: rc = launch_igemm_simt(a, p, stream); break;
    default: set_error("tensor-core back end does not cover this shape"); return -4;
  }
  g_last_plan = p;
  return rc;
}

}  // namespace bre
