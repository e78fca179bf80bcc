// Candidate augmentations on the device (SURVEY section 8 f-4; reference attacks/auxiliaries/augmentations.py, applied in the closure
// at optimization_based_attack.py:149-153).  The candidate x passes through a short pipeline of *linear* views before the model sees
// it; the closure's gradient is pulled back through the transposed pipeline.  Supported steps (the ones that keep the shape):
//   discrete_shift  (Jitter :9-18)            torch.roll by two random offsets in [-lim, lim), one draw per forward, whole batch
//   flip            (Flip :57-64)             horizontal flip with probability p, one draw per forward
//   colorjitter     (ColorJitter :70-89)      (x - mean[n, c]) / std[n, c], constants drawn once per attacker
//   continuous_shift (RandomTransform :141-205) grid_sample (align_corners = True; bilinear, nearest or bicubic; zeros, border or
//                                             reflection padding) on the grid g(i, j) = (lin[j] + sx[n], lin[i] + sy[n]),
//                                             lin = linspace(-1, 1, S), per-image random shifts of at most shift / (S - 1), each
//                                             coordinate negated per image by the fliplr / flipud grid flips; padding "circular" maps
//                                             g -> ((g + 1) mod 1) - 1 and samples with zeros padding as the reference does (which samples
//                                             the top-left quadrant twice per axis -- reproduced).  The grid is separable, so every output
//                                             row / column reads at most 4 taps of its axis (cs_taps), and the pull-back is two 1-D gathers.
// Shape-changing stages (each a stage of its own, see AugStage): RESAMPLE = a window resized bilinearly (Zoom :34-40, CenterZoom :43-55,
// Focus :20-31), BLUR = binomial depthwise convolution (AntiAlias :198-226).  Their pull-backs are fixed-order gathers (no atomics).
// Random draws come from Philox keyed by (seed, iteration, step), so the forward view and the transposed pull-back of one
// iteration see the same draws without any host round trip; `bre_augment_*` take the draws explicitly (parity tests).
#include <math.h>

#include "../../include/breaching_b200.h"
#include "common.cuh"
#include "augment.cuh"

namespace bre {
namespace {

__device__ __forceinline__ void philox4(uint64_t seed, uint32_t a, uint32_t b, uint32_t c, uint32_t (&out)[4]) {
  uint32_t ctr[4] = {a, b, c, 0x85EBCA6Bu};
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, ctr[0]), lo0 = 0xD2511F53u * ctr[0];
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, ctr[2]), lo1 = 0xCD9E8D57u * ctr[2];
    const uint32_t n0 = hi1 ^ ctr[1] ^ k0, n1 = lo1, n2 = hi0 ^ ctr[3] ^ k1, n3 = lo0;
    ctr[0] = n0; ctr[1] = n1; ctr[2] = n2; ctr[3] = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  out[0] = ctr[0]; out[1] = ctr[1]; out[2] = ctr[2]; out[3] = ctr[3];
}
__device__ __forceinline__ float u01(uint32_t v) { return ((float)(v >> 8) + 0.5f) * (1.0f / 16777216.0f); }

// one thread block: the draws of this iteration, every stage -> draws[stage] in global memory (read by the view / pull-back kernels).
// A PIXEL stage draws with its plan's seed (the first one with the pipeline's seed: a pipeline of one PIXEL stage draws exactly what a
// single plan drew); a focus stage draws its window corner from Philox(seed, iteration, 0x10000 + stage).
__global__ void aug_draw_kernel(AugPipeline pipe, const Scalars* sc, AugDraws* draws, int N) {
  pdl_prologue();
  const int it = sc != nullptr ? sc->it : 0;
  for (int k = 0; k < pipe.n_stages; ++k) {
    const AugStage& st = pipe.st[k];
    AugDraws* d = draws + k;
    if (st.kind == AUG_STAGE_RESAMPLE && st.focus) {
      if (threadIdx.x == 0) {      // Focus (:27-31): pert = (rand(2) * 2 - 1) * std; corner = (pert + in // 2 - size // 2).long().clamp
        uint32_t r[4];
        philox4(pipe.seed, (uint32_t)it, 0x10000u + (uint32_t)k, 0u, r);
        const float py = (u01(r[0]) * 2.f - 1.f) * st.focus_std, px = (u01(r[1]) * 2.f - 1.f) * st.focus_std;
        int y0 = (int)((py + (float)(st.Hi / 2)) - (float)(st.wh / 2)), x0 = (int)((px + (float)(st.Wi / 2)) - (float)(st.ww / 2));
        y0 = y0 < 0 ? 0 : (y0 > st.Hi - st.wh ? st.Hi - st.wh : y0);
        x0 = x0 < 0 ? 0 : (x0 > st.Wi - st.ww ? st.Wi - st.ww : x0);
        d->o1[0] = y0; d->o2[0] = x0;
      }
      continue;
    }
    if (st.kind != AUG_STAGE_PIXEL) continue;
    const AugPlan& plan = pipe.plan[k];
    for (int s = threadIdx.x; s < plan.n_steps; s += blockDim.x) {
      uint32_t r[4];
      philox4(plan.seed, (uint32_t)it, (uint32_t)s, 0u, r);
      if (plan.kind[s] == AUG_SHIFT) {
        const int lim = (int)plan.p0[s];
        d->o1[s] = lim > 0 ? (int)(r[0] % (uint32_t)(2 * lim)) - lim : 0;   // randint(-lim, lim)
        d->o2[s] = lim > 0 ? (int)(r[1] % (uint32_t)(2 * lim)) - lim : 0;
      } else if (plan.kind[s] == AUG_FLIP) {
        d->o1[s] = u01(r[0]) < plan.p0[s] ? 1 : 0;
      }
    }
    // continuous shift: two uniforms per image, and the grid flips from the third and fourth word (randgen[:, 2:4] > 0.5)
    for (int n = threadIdx.x; n < N; n += blockDim.x) {
      uint32_t r[4];
      philox4(plan.seed, (uint32_t)it, 0xC0FFEEu, (uint32_t)n, r);
      d->sx[n] = u01(r[0]);
      d->sy[n] = u01(r[1]);
      d->flr[n] = plan.cs_fliplr && u01(r[2]) > 0.5f;
      d->fud[n] = plan.cs_flipud && u01(r[3]) > 0.5f;
    }
  }
}

// index map of the permutation steps: output pixel (i, j) reads input pixel (y, x)
__device__ __forceinline__ void map_back(const AugPlan& plan, const AugDraws& d, int H, int W, int i, int j, int& y, int& x) {
  y = i; x = j;
  for (int s = plan.n_steps - 1; s >= 0; --s) {
    if (plan.kind[s] == AUG_FLIP) { if (d.o1[s]) x = W - 1 - x; }
    else if (plan.kind[s] == AUG_SHIFT) {         // out[i, j] = in[(i - o1) mod H, (j - o2) mod W]
      y = ((y - d.o1[s]) % H + H) % H;
      x = ((x - d.o2[s]) % W + W) % W;
    }
  }
}
__device__ __forceinline__ void map_forward(const AugPlan& plan, const AugDraws& d, int H, int W, int y, int x, int& i, int& j) {
  i = y; j = x;
  for (int s = 0; s < plan.n_steps; ++s) {
    if (plan.kind[s] == AUG_SHIFT) { i = ((i + d.o1[s]) % H + H) % H; j = ((j + d.o2[s]) % W + W) % W; }
    else if (plan.kind[s] == AUG_FLIP) { if (d.o1[s]) j = W - 1 - j; }
  }
}

// continuous shift along one axis of extent S: the taps of output index o for the uniform u and flip bit of its image, following
// ATen's grid sampler (GridSampler.h) with align_corners = True.  The coordinate is computed in double: the fp32 weights are then the
// float64 reference's rounded once.  bilinear / nearest: the unnormalised coordinate is clipped (border) or reflected about 0 and
// S - 1 and clipped (reflection), then sampled, and taps outside [0, S) read zero; nearest rounds half to even.  bicubic: four taps
// floor - 1 .. floor + 2 of the raw coordinate with the cubic-convolution weights (A = -0.75), each tap index passed through the
// padding rule on its own (several taps may land on one pixel).  idx = -1: a tap that reads zero.
struct CsTaps { short idx[4]; float w[4]; };

__device__ __forceinline__ double cs_reflect(double p, int S) {       // reflect_coordinates(p, 0, 2 (S - 1)), then clip
  if (S <= 1) return 0.0;
  const double span = (double)(S - 1);
  p = fabs(p);
  const double extra = fmod(p, span);
  const double r = ((long long)floor(p / span)) % 2 == 0 ? extra : span - extra;
  return fmin(fmax(r, 0.0), span);
}
__device__ __forceinline__ int cs_bound(int i, int S, int padding) {   // an integer tap under the padding rule (-1: zero)
  if (padding == AUG_CS_BORDER) return i < 0 ? 0 : (i > S - 1 ? S - 1 : i);
  if (padding == AUG_CS_REFLECTION) {
    if (S <= 1) return 0;
    const int period = 2 * (S - 1);
    int m = (i < 0 ? -i : i) % period;
    return m > S - 1 ? period - m : m;
  }
  return i >= 0 && i < S ? i : -1;
}
__device__ __forceinline__ double cubic1(double x) { const double A = -0.75; return ((A + 2.0) * x - (A + 3.0)) * x * x + 1.0; }
__device__ __forceinline__ double cubic2(double x) { const double A = -0.75; return ((A * x - 5.0 * A) * x + 8.0 * A) * x - 4.0 * A; }

__device__ CsTaps cs_taps(const AugPlan& plan, float u, int flip, int o, int S) {
  const double lin = S > 1 ? -1.0 + 2.0 * (double)o / (double)(S - 1) : -1.0;
  double g = lin + ((double)u - 0.5) * 2.0 * ((double)plan.cs_shift / (double)(S - 1));
  if (flip) g = -g;
  if (plan.cs_circular) g = (g + 1.0) - floor(g + 1.0) - 1.0;        // python's (g + 1) % 1 - 1
  double pos = (g + 1.0) / 2.0 * (double)(S - 1);                    // grid_sampler_unnormalize, align_corners = True
  CsTaps t;
#pragma unroll
  for (int k = 0; k < 4; ++k) { t.idx[k] = -1; t.w[k] = 0.f; }
  if (plan.cs_mode == AUG_CS_BICUBIC) {
    const double fl = floor(pos), f = pos - fl;
    const double c[4] = {cubic2(f + 1.0), cubic1(f), cubic1(1.0 - f), cubic2(2.0 - f)};
#pragma unroll
    for (int k = 0; k < 4; ++k) { t.idx[k] = (short)cs_bound((int)fl - 1 + k, S, plan.cs_padding); t.w[k] = (float)c[k]; }
    return t;
  }
  if (plan.cs_padding == AUG_CS_BORDER) pos = fmin(fmax(pos, 0.0), (double)(S - 1));
  else if (plan.cs_padding == AUG_CS_REFLECTION) pos = cs_reflect(pos, S);
  if (plan.cs_mode == AUG_CS_NEAREST) {
    const double r = rint(pos);
    t.idx[0] = (short)(r >= 0.0 && r < (double)S ? (int)r : -1); t.w[0] = 1.f;
    return t;
  }
  const double fl = floor(pos), f = pos - fl;
  const int i0 = (int)fl;
  t.idx[0] = (short)(i0 >= 0 && i0 < S ? i0 : -1);           t.w[0] = (float)(1.0 - f);
  t.idx[1] = (short)(i0 + 1 >= 0 && i0 + 1 < S ? i0 + 1 : -1); t.w[1] = (float)f;
  return t;
}

// forward view: permutation steps, then (optionally) the continuous shift, then the colour affine.  blockIdx.y = image; with the
// continuous shift the block first tabulates the taps of its image's rows and columns in shared memory ([H] then [W]).
__global__ void __launch_bounds__(256) aug_view_kernel(const float* __restrict__ x, float* __restrict__ out, int C, int H, int W,
                                                       AugPlan plan, const AugDraws* __restrict__ draws) {
  extern __shared__ CsTaps taps[];
  pdl_prologue();
  const int n = blockIdx.y;
  const long long per = (long long)C * H * W;
  const AugDraws& d = *draws;   // read through the pointer (uniform addresses: served by the L1 / constant path)
  if (plan.cs_enabled) {
    for (int k = threadIdx.x; k < H + W; k += blockDim.x)
      taps[k] = k < H ? cs_taps(plan, d.sy[n], d.fud[n], k, H) : cs_taps(plan, d.sx[n], d.flr[n], k - H, W);
    __syncthreads();
  }
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < per; e += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(e % W);
    const long long t = e / W;
    const int i = (int)(t % H);
    const int c = (int)(t / H);
    const float* src = x + ((long long)n * C + c) * H * W;
    float v;
    if (plan.cs_enabled) {   // the continuous shift is the outermost spatial step: sample the permuted image
      const CsTaps& ty = taps[i];
      const CsTaps& tx = taps[H + j];
      v = 0.f;
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) {
          const int yy = ty.idx[a], xx = tx.idx[b];
          if (yy >= 0 && xx >= 0 && ty.w[a] != 0.f && tx.w[b] != 0.f) {
            int sy, sx;
            map_back(plan, d, H, W, yy, xx, sy, sx);
            v = fmaf(ty.w[a] * tx.w[b], src[(long long)sy * W + sx], v);
          }
        }
    } else {
      int sy, sx;
      map_back(plan, d, H, W, i, j, sy, sx);
      v = src[(long long)sy * W + sx];
    }
    if (plan.cj_scale != nullptr) v = fmaf(v, plan.cj_scale[n * C + c], plan.cj_shift[n * C + c]);
    out[(long long)n * per + e] = v;
  }
}

// pull-back without continuous shift: gx[y, x] = scale * g[forward(y, x)]
__global__ void __launch_bounds__(256) aug_pull_perm_kernel(const float* __restrict__ g, float* __restrict__ gx, int N, int C, int H, int W,
                                                            AugPlan plan, const AugDraws* __restrict__ draws) {
  pdl_prologue();
  const long long total = (long long)N * C * H * W;
  const AugDraws& d = *draws;   // read through the pointer (uniform addresses: served by the L1 / constant path)
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int xq = (int)(e % W);
    long long t = e / W;
    const int yq = (int)(t % H); t /= H;
    const int c = (int)(t % C);
    const int n = (int)(t / C);
    int i, j;
    map_forward(plan, d, H, W, yq, xq, i, j);
    float v = g[(((long long)n * C + c) * H + i) * W + j];
    if (plan.cj_scale != nullptr) v *= plan.cj_scale[n * C + c];
    gx[e] = v;
  }
}

// pull-back through the continuous shift, separable and deterministic (no atomics): first along x, then along y.
//   tmp[n, c, i, xx] = sum_j wx(j -> xx) g[n, c, i, j]          out[n, c, yy, xx] = sum_i wy(i -> yy) tmp[n, c, i, xx]
// wx(j -> xx) sums the taps of output j that land on xx (bicubic taps may fold onto one pixel).  blockIdx.y = image; the block
// tabulates its image's taps of the axis with the same cs_taps as the view, so both see bitwise the same weights.  Every thread walks
// the output index of its axis in order (O(S) per element; the warp reads one table entry at a time, a shared-memory broadcast).
__global__ void __launch_bounds__(256) aug_pull_cs_kernel(const float* __restrict__ g, float* __restrict__ out, int C, int H, int W,
                                                          AugPlan plan, const AugDraws* __restrict__ draws, int axis) {
  extern __shared__ CsTaps taps[];
  pdl_prologue();
  const int n = blockIdx.y;
  const int S = axis == 0 ? W : H;
  for (int k = threadIdx.x; k < S; k += blockDim.x)
    taps[k] = axis == 0 ? cs_taps(plan, draws->sx[n], draws->flr[n], k, S) : cs_taps(plan, draws->sy[n], draws->fud[n], k, S);
  __syncthreads();
  const long long per = (long long)C * H * W;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < per; e += (long long)gridDim.x * blockDim.x) {
    const int xq = (int)(e % W);
    const int yq = (int)((e / W) % H);
    const float* plane = g + (long long)n * per + (e - ((long long)yq * W + xq));
    const int q = axis == 0 ? xq : yq;
    float acc = 0.f;
    for (int o = 0; o < S; ++o) {
      const CsTaps& t = taps[o];
      float w = 0.f;
#pragma unroll
      for (int k = 0; k < 4; ++k) w += t.idx[k] == q ? t.w[k] : 0.f;
      if (w != 0.f) acc = fmaf(w, axis == 0 ? plane[(long long)yq * W + o] : plane[(long long)o * W + xq], acc);
    }
    out[(long long)n * per + e] = acc;
  }
}

// RESAMPLE view: the window [y0, y0 + wh) x [x0, x0 + ww) of every plane, resized bilinearly to Ho x Wo (F.interpolate, bilinear,
// align_corners = False; zoom: window = image, centerzoom / focus: a fixed / drawn corner; wh = Ho makes the copy exact)
__device__ __forceinline__ void resample_corner(const AugStage& st, const AugDraws* d, int& y0, int& x0) {
  y0 = st.y0; x0 = st.x0;
  if (st.focus) { y0 = d->o1[0]; x0 = d->o2[0]; }
}
__global__ void __launch_bounds__(256) aug_resample_view_kernel(const float* __restrict__ x, float* __restrict__ out, int planes, AugStage st,
                                                                const AugDraws* __restrict__ draws) {
  pdl_prologue();
  int y0, x0;
  resample_corner(st, draws, y0, x0);
  const float sh = (float)st.wh / (float)st.Ho, sw = (float)st.ww / (float)st.Wo;
  const long long total = (long long)planes * st.Ho * st.Wo;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int ox = (int)(e % st.Wo);
    const long long t = e / st.Wo;
    const int oy = (int)(t % st.Ho);
    const long long pl = t / st.Ho;
    int a0, a1, b0, b1; float ly, lx;
    bilinear_src(oy, sh, st.wh, a0, a1, ly);
    bilinear_src(ox, sw, st.ww, b0, b1, lx);
    const float* p = x + pl * st.Hi * st.Wi + (long long)y0 * st.Wi + x0;
    const float top = (1.f - lx) * p[(long long)a0 * st.Wi + b0] + lx * p[(long long)a0 * st.Wi + b1];
    const float bot = (1.f - lx) * p[(long long)a1 * st.Wi + b0] + lx * p[(long long)a1 * st.Wi + b1];
    out[e] = (1.f - ly) * top + ly * bot;
  }
}

// weight of window index q in the bilinear stencil of output index o (both neighbours land on q at the clamped last index)
__device__ __forceinline__ float bilinear_weight(int o, float scale, int in, int q) {
  int i0, i1; float l;
  bilinear_src(o, scale, in, i0, i1, l);
  return (i0 == q ? 1.f - l : 0.f) + (i1 == q ? l : 0.f);
}
// the output indices whose stencil can touch window index q: source coordinates in [q - 1, q + 1), widened by two on each side
// (the membership test is exact, the range only has to contain it)
__device__ __forceinline__ void bilinear_range(int q, float scale, int out, int& lo, int& hi) {
  lo = (int)floorf(((float)q - 0.5f) / scale - 0.5f) - 2;
  hi = (int)ceilf(((float)q + 1.5f) / scale - 0.5f) + 2;
  lo = lo < 0 ? 0 : lo;
  hi = hi > out - 1 ? out - 1 : hi;
}
// RESAMPLE pull-back, separable in two fixed-order gathers (no atomics; each bilinear weight is evaluated once per gathered term):
//   axis 0: tmp[pl, oy, qx] = sum_ox wx(ox -> qx) g[pl, oy, ox]                  (qx in the window, tmp is [planes, Ho, ww])
//   axis 1: gx[pl, y, x]   = sum_oy wy(oy -> y - y0) tmp[pl, oy, x - x0]           (zero outside the window)
__global__ void __launch_bounds__(256) aug_resample_pull_kernel(const float* __restrict__ g, float* __restrict__ out, int planes, AugStage st,
                                                                const AugDraws* __restrict__ draws, int axis) {
  pdl_prologue();
  int y0, x0;
  resample_corner(st, draws, y0, x0);
  const float sh = (float)st.wh / (float)st.Ho, sw = (float)st.ww / (float)st.Wo;
  const int rows = axis == 0 ? st.Ho : st.Hi, cols = axis == 0 ? st.ww : st.Wi;
  const long long total = (long long)planes * rows * cols;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(e % cols);
    const long long t = e / cols;
    const int r = (int)(t % rows);
    const long long pl = t / rows;
    float acc = 0.f;
    if (axis == 0) {
      const float* row = g + (pl * st.Ho + r) * st.Wo;
      int lo, hi;
      bilinear_range(c, sw, st.Wo, lo, hi);
      for (int ox = lo; ox <= hi; ++ox) {
        const float w = bilinear_weight(ox, sw, st.ww, c);
        if (w != 0.f) acc = fmaf(w, row[ox], acc);
      }
    } else {
      const int qy = r - y0, qx = c - x0;
      if (qy >= 0 && qy < st.wh && qx >= 0 && qx < st.ww) {
        const float* col = g + pl * st.Ho * st.ww + qx;
        int lo, hi;
        bilinear_range(qy, sh, st.Ho, lo, hi);
        for (int oy = lo; oy <= hi; ++oy) {
          const float w = bilinear_weight(oy, sh, st.wh, qy);
          if (w != 0.f) acc = fmaf(w, col[(long long)oy * st.ww], acc);
        }
      }
    }
    out[e] = acc;
  }
}

// BLUR (AntiAlias :198-226): depthwise conv2d with the normalised outer product of the binomial row of `width`, zero padding
// width // 2, `stride`.  The weights c[a] / 2^(width - 1) are dyadic: their products are the reference's filter exactly.
__device__ __forceinline__ float binomial_weight(int width, int a) {
  float c = 1.f;                                      // C(width - 1, a), exact in fp32 for width <= 7
  for (int i = 0; i < a; ++i) c = c * (float)(width - 1 - i) / (float)(i + 1);
  return ldexpf(c, -(width - 1));
}
__global__ void __launch_bounds__(256) aug_blur_view_kernel(const float* __restrict__ x, float* __restrict__ out, int planes, AugStage st) {
  pdl_prologue();
  const int pad = st.width / 2;
  const long long total = (long long)planes * st.Ho * st.Wo;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int ox = (int)(e % st.Wo);
    const long long t = e / st.Wo;
    const int oy = (int)(t % st.Ho);
    const long long pl = t / st.Ho;
    const float* p = x + pl * st.Hi * st.Wi;
    float acc = 0.f;
    for (int a = 0; a < st.width; ++a) {
      const int y = oy * st.stride - pad + a;
      if (y < 0 || y >= st.Hi) continue;
      float row = 0.f;
      for (int b = 0; b < st.width; ++b) {
        const int xx = ox * st.stride - pad + b;
        if (xx >= 0 && xx < st.Wi) row = fmaf(binomial_weight(st.width, b), p[(long long)y * st.Wi + xx], row);
      }
      acc = fmaf(binomial_weight(st.width, a), row, acc);
    }
    out[e] = acc;
  }
}
// BLUR pull-back: input pixel (y, x) gathers the view gradients of the outputs (oy, ox) with oy * stride - pad + a = y, in order of a, b
__global__ void __launch_bounds__(256) aug_blur_pull_kernel(const float* __restrict__ g, float* __restrict__ gx, int planes, AugStage st) {
  pdl_prologue();
  const int pad = st.width / 2;
  const long long total = (long long)planes * st.Hi * st.Wi;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int xq = (int)(e % st.Wi);
    const long long t = e / st.Wi;
    const int yq = (int)(t % st.Hi);
    const long long pl = t / st.Hi;
    const float* p = g + pl * st.Ho * st.Wo;
    float acc = 0.f;
    for (int a = 0; a < st.width; ++a) {
      const int ny = yq + pad - a;
      if (ny < 0 || ny % st.stride != 0 || ny / st.stride >= st.Ho) continue;
      const int oy = ny / st.stride;
      float row = 0.f;
      for (int b = 0; b < st.width; ++b) {
        const int nx = xq + pad - b;
        if (nx < 0 || nx % st.stride != 0 || nx / st.stride >= st.Wo) continue;
        row = fmaf(binomial_weight(st.width, b), p[(long long)oy * st.Wo + nx / st.stride], row);
      }
      acc = fmaf(binomial_weight(st.width, a), row, acc);
    }
    gx[e] = acc;
  }
}

inline int grid_for(long long n) {
  long long b = (n + 255) / 256;
  const long long cap = (long long)kNumSMs * 16;
  return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

}  // namespace

int launch_aug_draws(const AugPipeline& pipe, const Scalars* sc, AugDraws* draws, int N, cudaStream_t s) {
  if (N > AUG_MAX_BATCH) { set_error("augmentations: batch larger than AUG_MAX_BATCH"); return -4; }
  BRE_KLAUNCH(aug_draw_kernel, 1, 64, 0, s, pipe, sc, draws, N);
  BRE_CHECK_LAUNCH();
  return 0;
}
// the continuous-shift kernels run one grid row per image (blockIdx.y), about as many blocks in all as grid_for gives the batch
inline dim3 grid_per_image(int N, long long per) {
  const int bx = grid_for((long long)N * per) / N;
  return dim3(bx < 1 ? 1 : bx, N);
}
int launch_aug_view(const float* x, float* out, int N, int C, int H, int W, const AugPlan& plan, const AugDraws* draws, cudaStream_t s) {
  const size_t smem = plan.cs_enabled ? (size_t)(H + W) * sizeof(CsTaps) : 0;
  BRE_KLAUNCH(aug_view_kernel, grid_per_image(N, (long long)C * H * W), 256, smem, s, x, out, C, H, W, plan, draws);
  BRE_CHECK_LAUNCH();
  return 0;
}
// gx <- pull-back of g (g is clobbered when the continuous shift is enabled: it serves as the intermediate); tmp: same size
int launch_aug_pull(float* g, float* tmp, float* gx, int N, int C, int H, int W, const AugPlan& plan, const AugDraws* draws, cudaStream_t s) {
  const int grid = grid_for((long long)N * C * H * W);
  const float* src = g;
  if (plan.cs_enabled) {
    const dim3 gi = grid_per_image(N, (long long)C * H * W);
    BRE_KLAUNCH(aug_pull_cs_kernel, gi, 256, (size_t)W * sizeof(CsTaps), s, (const float*)g, tmp, C, H, W, plan, draws, 0);
    BRE_KLAUNCH(aug_pull_cs_kernel, gi, 256, (size_t)H * sizeof(CsTaps), s, (const float*)tmp, g, C, H, W, plan, draws, 1);
  }
  BRE_KLAUNCH(aug_pull_perm_kernel, grid, 256, 0, s, src, gx, N, C, H, W, plan, draws);
  BRE_CHECK_LAUNCH();
  return 0;
}

int launch_aug_resample(const float* x, float* out, int N, const AugStage& st, const AugDraws* draws, bool transpose, float* tmp, cudaStream_t s) {
  const int planes = N * st.C;
  if (!transpose) BRE_KLAUNCH(aug_resample_view_kernel, grid_for((long long)planes * st.Ho * st.Wo), 256, 0, s, x, out, planes, st, draws);
  else {
    BRE_KLAUNCH(aug_resample_pull_kernel, grid_for((long long)planes * st.Ho * st.ww), 256, 0, s, x, (float*)tmp, planes, st, draws, 0);
    BRE_KLAUNCH(aug_resample_pull_kernel, grid_for((long long)planes * st.Hi * st.Wi), 256, 0, s, (const float*)tmp, out, planes, st, draws, 1);
  }
  BRE_CHECK_LAUNCH();
  return 0;
}
int launch_aug_blur(const float* x, float* out, int N, const AugStage& st, bool transpose, cudaStream_t s) {
  const int planes = N * st.C;
  if (!transpose) BRE_KLAUNCH(aug_blur_view_kernel, grid_for((long long)planes * st.Ho * st.Wo), 256, 0, s, x, out, planes, st);
  else BRE_KLAUNCH(aug_blur_pull_kernel, grid_for((long long)planes * st.Hi * st.Wi), 256, 0, s, x, out, planes, st);
  BRE_CHECK_LAUNCH();
  return 0;
}

}  // namespace bre

using namespace bre;

// ---- stand-alone entry points with explicit draws (parity tests against the reference modules) -----------------------------------
static int fill_plan(AugPlan* plan, AugDraws* d, int32_t n_steps, const int32_t* kinds, const int32_t* o1, const int32_t* o2, float cs_shift,
                     int32_t cs_circular, int32_t cs_mode, int32_t cs_padding, const float* sx, const float* sy, const int32_t* flr,
                     const int32_t* fud, int32_t N, int32_t H, int32_t W, const float* cj_scale, const float* cj_shift) {
  if (n_steps < 0 || n_steps > AUG_MAX_STEPS || N > AUG_MAX_BATCH) { set_error("bre_augment: too many steps / images"); return BRE_ERR_INVALID; }
  if (cs_mode < AUG_CS_BILINEAR || cs_mode > AUG_CS_BICUBIC || cs_padding < AUG_CS_ZEROS || cs_padding > AUG_CS_REFLECTION ||
      (cs_circular && cs_padding != AUG_CS_ZEROS)) {
    set_error("bre_augment: unknown continuous_shift mode / padding (circular wraps the grid and pads with zeros)"); return BRE_ERR_INVALID;
  }
  if (sx != nullptr && (H > AUG_CS_MAX_SIDE || W > AUG_CS_MAX_SIDE)) { set_error("bre_augment: continuous_shift on a side over 1024"); return BRE_ERR_UNSUPPORTED; }
  memset(plan, 0, sizeof(*plan));
  memset(d, 0, sizeof(*d));
  plan->n_steps = n_steps;
  for (int s = 0; s < n_steps; ++s) { plan->kind[s] = kinds[s]; d->o1[s] = o1[s]; d->o2[s] = o2 ? o2[s] : 0; }
  plan->cs_enabled = sx != nullptr; plan->cs_shift = cs_shift; plan->cs_circular = cs_circular;
  plan->cs_mode = cs_mode; plan->cs_padding = cs_padding;
  for (int n = 0; n < N && sx != nullptr; ++n) {
    d->sx[n] = sx[n]; d->sy[n] = sy[n];
    d->flr[n] = flr != nullptr && flr[n] != 0; d->fud[n] = fud != nullptr && fud[n] != 0;
  }
  plan->cj_scale = cj_scale; plan->cj_shift = cj_shift;
  return 0;
}

extern "C" int bre_augment_view(const float* x, float* out, int32_t N, int32_t C, int32_t H, int32_t W, int32_t n_steps, const int32_t* kinds,
                                const int32_t* o1, const int32_t* o2, float cs_shift, int32_t cs_circular, const float* sx, const float* sy,
                                const float* cj_scale, const float* cj_shift, int32_t transpose, float* scratch, void* stream) {
  return bre_augment_view_ex(x, out, N, C, H, W, n_steps, kinds, o1, o2, cs_shift, cs_circular, BRE_CS_BILINEAR, BRE_CS_ZEROS, sx, sy, nullptr,
                             nullptr, cj_scale, cj_shift, transpose, scratch, stream);
}

extern "C" int bre_augment_view_ex(const float* x, float* out, int32_t N, int32_t C, int32_t H, int32_t W, int32_t n_steps, const int32_t* kinds,
                                   const int32_t* o1, const int32_t* o2, float cs_shift, int32_t cs_circular, int32_t cs_mode, int32_t cs_padding,
                                   const float* sx, const float* sy, const int32_t* fliplr, const int32_t* flipud, const float* cj_scale,
                                   const float* cj_shift, int32_t transpose, float* scratch, void* stream) {
  if (!x || !out || N <= 0 || C <= 0 || H <= 0 || W <= 0 || (sx != nullptr) != (sy != nullptr)) { set_error("bre_augment_view: bad arguments"); return BRE_ERR_INVALID; }
  AugPlan plan; AugDraws host;
  const int frc = fill_plan(&plan, &host, n_steps, kinds, o1, o2, cs_shift, cs_circular, cs_mode, cs_padding, sx, sy, fliplr, flipud, N, H, W,
                            cj_scale, cj_shift);
  if (frc != 0) return frc;
  cudaStream_t s = (cudaStream_t)stream;
  AugDraws* dev = nullptr;
  BRE_CUDA_CHECK(cudaMallocAsync((void**)&dev, sizeof(AugDraws), s));
  BRE_CUDA_CHECK(cudaMemcpyAsync(dev, &host, sizeof(AugDraws), cudaMemcpyHostToDevice, s));
  int rc = 0;
  if (!transpose) rc = launch_aug_view(x, out, N, C, H, W, plan, dev, s);
  else {
    if (plan.cs_enabled && !scratch) { set_error("bre_augment_view: the transposed continuous shift needs a scratch buffer"); rc = BRE_ERR_INVALID; }
    else rc = launch_aug_pull(const_cast<float*>(x), scratch, out, N, C, H, W, plan, dev, s);
  }
  cudaStreamSynchronize(s);
  cudaFreeAsync(dev, s);
  return rc;
}

extern "C" int bre_augment_resample(const float* x, float* out, int32_t N, int32_t C, int32_t Hi, int32_t Wi, int32_t y0, int32_t x0,
                                    int32_t wh, int32_t ww, int32_t Ho, int32_t Wo, int32_t transpose, void* stream) {
  if (!x || !out || N <= 0 || C <= 0 || Hi <= 0 || Wi <= 0 || Ho <= 0 || Wo <= 0 || wh <= 0 || ww <= 0 || y0 < 0 || x0 < 0 || y0 + wh > Hi ||
      x0 + ww > Wi) { set_error("bre_augment_resample: bad arguments (the window must lie inside the input)"); return BRE_ERR_INVALID; }
  AugStage st;
  memset(&st, 0, sizeof(st));
  st.kind = AUG_STAGE_RESAMPLE; st.C = C; st.Hi = Hi; st.Wi = Wi; st.Ho = Ho; st.Wo = Wo; st.y0 = y0; st.x0 = x0; st.wh = wh; st.ww = ww;
  cudaStream_t s = (cudaStream_t)stream;
  float* tmp = nullptr;             // the pull-back's intermediate [N, C, Ho, ww]
  if (transpose) BRE_CUDA_CHECK(cudaMallocAsync((void**)&tmp, (size_t)N * C * Ho * ww * sizeof(float), s));
  const int rc = launch_aug_resample(x, out, N, st, nullptr, transpose != 0, tmp, s);
  BRE_CUDA_CHECK(cudaStreamSynchronize(s));
  if (tmp) cudaFreeAsync(tmp, s);
  return rc;
}

extern "C" int bre_augment_blur(const float* x, float* out, int32_t N, int32_t C, int32_t Hi, int32_t Wi, int32_t width, int32_t stride,
                                int32_t transpose, void* stream) {
  if (!x || !out || N <= 0 || C <= 0 || Hi <= 0 || Wi <= 0 || width < 1 || width > 7 || stride < 1) {
    set_error("bre_augment_blur: bad arguments (width 1..7, stride >= 1)"); return BRE_ERR_INVALID;
  }
  AugStage st;
  memset(&st, 0, sizeof(st));
  st.kind = AUG_STAGE_BLUR; st.C = C; st.Hi = Hi; st.Wi = Wi; st.width = width; st.stride = stride;
  st.Ho = (Hi + 2 * (width / 2) - width) / stride + 1; st.Wo = (Wi + 2 * (width / 2) - width) / stride + 1;
  const int rc = launch_aug_blur(x, out, N, st, transpose != 0, (cudaStream_t)stream);
  BRE_CUDA_CHECK(cudaStreamSynchronize((cudaStream_t)stream));
  return rc;
}
