// Non-GEMM layer kernels (see layers.cuh).  All HBM-bound: coalesced along the channel dimension of the
// NHWC activations (32 consecutive channels = one 128-byte line per warp row), grid sized from the SM count.
#include <stdlib.h>

#include "layers.cuh"

#include <float.h>

namespace bre {

namespace {

constexpr int kEwThreads = 256;

inline int ew_grid(long long n) {
  long long b = (n + kEwThreads - 1) / kEwThreads;
  const long long cap = (long long)kNumSMs * 16;
  return (int)(b < cap ? (b > 0 ? b : 1) : cap);
}

// 128-bit kernels: every channel count of the conv nets is a multiple of 4 (BRE_VEC_EW=0 falls back to the scalar kernels)
inline bool vec_ok(int C) {
  static const bool env = [] { const char* e = getenv("BRE_VEC_EW"); return e ? atoi(e) != 0 : true; }();
  return env && C % 4 == 0 && C >= 4;
}

// ---- BN constants -------------------------------------------------------------------------------
__global__ void bn_prepare_kernel(const float* __restrict__ gamma, const float* __restrict__ beta,
                                  const float* __restrict__ rm, const float* __restrict__ rv, float eps, int C,
                                  float* scale, float* shift, float* inv, float* nrm) {
  pdl_prologue();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float iv = 1.0f / sqrtf(rv[c] + eps);
  inv[c] = iv;
  nrm[c] = -rm[c] * iv;
  scale[c] = gamma[c] * iv;
  shift[c] = beta[c] - gamma[c] * rm[c] * iv;
}

// ---- fused BN + residual + ReLU forward ------------------------------------------------------------
__global__ void bnact_fwd_kernel(const float* __restrict__ in, const float* __restrict__ res, float* __restrict__ out,
                                 long long total, int C, bool has_bn, bool relu, BnConsts bn, bool round_out) {
  pdl_prologue();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    float u = in[i];
    // eval-mode BN as ATen applies it: x * alpha + beta', alpha = gamma * invstd, beta' = beta - mean * alpha
    if (has_bn) u = fmaf(u, __ldg(bn.scale + c), __ldg(bn.shift + c));
    if (res != nullptr) u += res[i];
    u = relu ? fmaxf(u, 0.f) : u;
    out[i] = round_out ? tf32_rna(u) : u;
  }
}

// ---- (32 channels) x (pixel slab) reductions ------------------------------------------------------
// Block (32, 8); blockIdx.x = channel group, blockIdx.y = slab.  Returns per-thread partial sums reduced over
// threadIdx.y into row 0, then the last-arriving block of a channel group reduces the slabs in fixed order.
template <int NV>
__device__ __forceinline__ bool slab_reduce(float (&v)[NV], float* partials, int* counters, int Cpad, float (&total)[NV], bool defer = false) {
  __shared__ float sm[NV][8][33];
  __shared__ int s_last;
  const int x = threadIdx.x, y = threadIdx.y;
#pragma unroll
  for (int k = 0; k < NV; ++k) sm[k][y][x] = v[k];
  __syncthreads();
  const int c = blockIdx.x * 32 + x;
  if (y == 0) {
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      float s = 0.f;
#pragma unroll
      for (int yy = 0; yy < 8; ++yy) s += sm[k][yy][x];
      partials[((long long)blockIdx.y * Cpad + c) * NV + k] = s;
    }
  }
  if (defer) return false;   // the slabs are summed later by one batched kernel for all layers (launch_bn_grad_finalize)
  __threadfence();
  __syncthreads();
  if (x == 0 && y == 0) {
    const int prev = atomicAdd(counters + blockIdx.x, 1);
    s_last = (prev == (int)gridDim.y - 1);
    if (s_last) counters[blockIdx.x] = 0;
  }
  __syncthreads();
  if (!s_last) return false;
  __threadfence();
  if (y == 0) {
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      float s = 0.f;
      for (int base = 0; base < (int)gridDim.y; base += 16) {   // 16 independent loads per round trip, summed in slab order
        float r[16];
#pragma unroll
        for (int u = 0; u < 16; ++u) r[u] = base + u < (int)gridDim.y ? __ldcg(partials + ((long long)(base + u) * Cpad + c) * NV + k) : 0.f;
#pragma unroll
        for (int u = 0; u < 16; ++u) s += r[u];
      }
      total[k] = s;
    }
  }
  return y == 0;
}

inline void slab_grid(long long P, int C, dim3& grid, dim3& block, long long& pps) {
  const int cg = ceil_div(C, 32);
  long long slabs = (2LL * kNumSMs + cg - 1) / cg;
  const long long max_slabs = (P + 7) / 8;
  if (slabs > max_slabs) slabs = max_slabs;
  if (slabs < 1) slabs = 1;
  if (slabs > 4096) slabs = 4096;
  pps = (P + slabs - 1) / slabs;
  slabs = (P + pps - 1) / pps;
  grid = dim3(cg, (unsigned)slabs);
  block = dim3(32, 8);
}

__global__ void bnact_bwd_kernel(BnActBwdArgs a, long long pps, int Cpad) {
  pdl_prologue();
  const int c = blockIdx.x * 32 + threadIdx.x;
  const bool cv = c < a.C;
  const long long p0 = blockIdx.y * pps;
  const long long p1 = (p0 + pps < a.P) ? p0 + pps : a.P;
  float v[2] = {0.f, 0.f};
  float inv = 0.f, nrm = 0.f, scale = 1.f;
  if (cv && a.has_bn) { inv = __ldg(a.bn.inv + c); nrm = __ldg(a.bn.nrm + c); scale = __ldg(a.bn.scale + c); }
  if (cv) {
    for (long long p = p0 + threadIdx.y; p < p1; p += 8) {
      const long long o = p * a.C + c;
      float du = a.dout[o];
      if (a.relu && !(a.out[o] > 0.f)) du = 0.f;
      float di = du;
      if (a.has_bn) {
        const float xhat = fmaf(a.in[o], inv, nrm);
        v[0] = fmaf(du, xhat, v[0]);
        v[1] += du;
        di = scale * du;
      }
      if (a.din != nullptr) {
        if (a.acc_in) di += a.din[o];
        a.din[o] = a.round_din ? tf32_rna(di) : di;
      }
      if (a.dres != nullptr) a.dres[o] = a.acc_res ? a.dres[o] + du : du;
    }
  }
  if (!a.has_bn || a.g_gamma == nullptr) return;  // uniform across the grid
  float tot[2];
  if (slab_reduce<2>(v, a.partials, a.counters, Cpad, tot, a.defer != 0) && cv) {
    a.g_gamma[c] = tot[0];
    a.g_beta[c] = tot[1];
  }
}

__global__ void bnact_tan_fwd_kernel(BnActTanFwdArgs a, long long total) {
  pdl_prologue();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % a.C);
    float u = a.tin != nullptr ? a.tin[i] : 0.f;
    if (a.has_bn) {
      const float xhat = fmaf(a.in[i], __ldg(a.bn.inv + c), __ldg(a.bn.nrm + c));
      u = fmaf(__ldg(a.bn.scale + c), u, fmaf(__ldg(a.v_gamma + c), xhat, __ldg(a.v_beta + c)));
    }
    if (a.tres != nullptr) u += a.tres[i];
    if (a.relu && !(a.out[i] > 0.f)) u = 0.f;
    a.tout[i] = a.round_out ? tf32_rna(u) : u;
  }
}

__global__ void bnact_tan_bwd_kernel(BnActTanBwdArgs a, long long total) {
  pdl_prologue();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % a.C);
    float tdu = a.tdout[i];
    float du = a.dout[i];
    if (a.relu && !(a.out[i] > 0.f)) { tdu = 0.f; du = 0.f; }
    float tdi = tdu;
    if (a.has_bn) {
      tdi = fmaf(__ldg(a.bn.scale + c), tdu, __ldg(a.v_gamma + c) * __ldg(a.bn.inv + c) * du);
      if (a.di_cm != nullptr) tdi += fmaf(__ldg(a.di_cv + c), a.in[i] - __ldg(a.di_mean + c), __ldg(a.di_cm + c));
    }
    if (a.tdin != nullptr) {
      if (a.acc_in) tdi += a.tdin[i];
      a.tdin[i] = a.round_din ? tf32_rna(tdi) : tdi;
    }
    if (a.tdres != nullptr) a.tdres[i] = a.acc_res ? a.tdres[i] + tdu : tdu;
  }
}

// slab-mapped variant of the tangent backward that also reduces the tangents of the BN parameter gradients
__global__ void bnact_tan_bwd_g_kernel(BnActTanBwdArgs a, long long pps, int Cpad) {
  pdl_prologue();
  const int c = blockIdx.x * 32 + threadIdx.x;
  const bool cv = c < a.C;
  const long long p0 = blockIdx.y * pps;
  const long long p1 = (p0 + pps < a.P) ? p0 + pps : a.P;
  float v[2] = {0.f, 0.f};
  float inv = 0.f, nrm = 0.f, scale = 1.f, vg = 0.f;
  if (cv) { inv = __ldg(a.bn.inv + c); nrm = __ldg(a.bn.nrm + c); scale = __ldg(a.bn.scale + c); vg = __ldg(a.v_gamma + c); }
  // DeepInversion adjoint at the BN input (the last local step of a FedAvg evaluation): not part of the parameter tangents
  const bool di = a.di_cm != nullptr;
  float di_m = 0.f, di_v = 0.f, di_mean = 0.f;
  if (cv && di) { di_m = __ldg(a.di_cm + c); di_v = __ldg(a.di_cv + c); di_mean = __ldg(a.di_mean + c); }
  if (cv) {
    for (long long p = p0 + threadIdx.y; p < p1; p += 8) {
      const long long o = p * a.C + c;
      float tdu = a.tdout[o], du = a.dout[o];
      if (a.relu && !(a.out[o] > 0.f)) { tdu = 0.f; du = 0.f; }
      const float xhat = fmaf(a.in[o], inv, nrm);
      const float tz = a.tin != nullptr ? a.tin[o] : 0.f;
      v[0] += fmaf(tdu, xhat, du * tz * inv);
      v[1] += tdu;
      float tdi = fmaf(scale, tdu, vg * inv * du);
      if (di) tdi += fmaf(di_v, a.in[o] - di_mean, di_m);
      if (a.tdin != nullptr) {
        if (a.acc_in) tdi += a.tdin[o];
        a.tdin[o] = a.round_din ? tf32_rna(tdi) : tdi;
      }
      if (a.tdres != nullptr) a.tdres[o] = a.acc_res ? a.tdres[o] + tdu : tdu;
    }
  }
  float tot[2];
  if (slab_reduce<2>(v, a.partials, a.counters, Cpad, tot) && cv) {
    a.tg_gamma[c] = tot[0];
    a.tg_beta[c] = tot[1];
  }
}

__global__ void axpby_kernel(const float* __restrict__ x, const float* __restrict__ y, float alpha, float* __restrict__ out, long long n4) {
  pdl_prologue();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(x) + i), b = __ldg(reinterpret_cast<const float4*>(y) + i);
    reinterpret_cast<float4*>(out)[i] = make_float4(fmaf(alpha, b.x, a.x), fmaf(alpha, b.y, a.y), fmaf(alpha, b.z, a.z), fmaf(alpha, b.w, a.w));
  }
}

// round-to-nearest (ties away) of fp32 values to the TF32 grid, in place: the tensor core drops the 13 low mantissa bits of
// kind::tf32 operands (truncation), so operands rounded beforehand are multiplied as if converted with cvt.rna.tf32
__global__ void round_tf32_kernel(const float* src, float* dst, long long n4) {
  pdl_prologue();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(src)[i];
    reinterpret_cast<float4*>(dst)[i] = make_float4(tf32_rna(v.x), tf32_rna(v.y), tf32_rna(v.z), tf32_rna(v.w));
  }
}

__global__ void channel_sum_kernel(const float* __restrict__ x, long long P, int C, float* out, float* partials,
                                   int* counters, long long pps, int Cpad) {
  pdl_prologue();
  const int c = blockIdx.x * 32 + threadIdx.x;
  const long long p0 = blockIdx.y * pps;
  const long long p1 = (p0 + pps < P) ? p0 + pps : P;
  float v[1] = {0.f};
  if (c < C)
    for (long long p = p0 + threadIdx.y; p < p1; p += 8) v[0] += x[p * C + c];
  float tot[1];
  if (slab_reduce<1>(v, partials, counters, Cpad, tot) && c < C) out[c] = tot[0];
}

__global__ void channel_stats_kernel(const float* __restrict__ x, long long P, int C, float* mean, float* var,
                                     float* partials, int* counters, long long pps, int Cpad) {
  pdl_prologue();
  const int c = blockIdx.x * 32 + threadIdx.x;
  const long long p0 = blockIdx.y * pps;
  const long long p1 = (p0 + pps < P) ? p0 + pps : P;
  // shifted sums (shift = first element of the channel) keep E[x^2] - E[x]^2 well conditioned in fp32
  const float sh = c < C ? x[c] : 0.f;
  float v[2] = {0.f, 0.f};
  if (c < C)
    for (long long p = p0 + threadIdx.y; p < p1; p += 8) {
      const float t = x[p * C + c] - sh;
      v[0] += t;
      v[1] = fmaf(t, t, v[1]);
    }
  float tot[2];
  if (slab_reduce<2>(v, partials, counters, Cpad, tot) && c < C) {
    const float m = tot[0] / (float)P;
    mean[c] = m + sh;
    var[c] = fmaxf(tot[1] / (float)P - m * m, 0.f);
  }
}


// ======================================================================================================================
// 128-bit variants of the BN / residual / ReLU sweeps (C % 4 == 0, which every conv net here satisfies).  The scalar kernels
// above move 4 bytes per thread and instruction, far from the HBM rate on the batch-8 tensors of config 3; these move 16 bytes per thread with several independent loads in flight.
// Same expressions, element by element.
// ======================================================================================================================
__device__ __forceinline__ float4 ld4(const float* p, long long i4) { return __ldg(reinterpret_cast<const float4*>(p) + i4); }
__device__ __forceinline__ float4 ldrw4(const float* p, long long i4) { return reinterpret_cast<const float4*>(p)[i4]; }   // buffers this kernel also writes
__device__ __forceinline__ float4 ldc4(const float* p, int c4) { return __ldg(reinterpret_cast<const float4*>(p) + c4); }
__device__ __forceinline__ void st4(float* p, long long i4, float4 v) { reinterpret_cast<float4*>(p)[i4] = v; }
__device__ __forceinline__ float4 rna4(float4 v) { return make_float4(tf32_rna(v.x), tf32_rna(v.y), tf32_rna(v.z), tf32_rna(v.w)); }
#define BRE_F4(expr_x, expr_y, expr_z, expr_w) make_float4(expr_x, expr_y, expr_z, expr_w)

__global__ void __launch_bounds__(256) bnact_fwd_vec_kernel(const float* __restrict__ in, const float* __restrict__ res, float* __restrict__ out,
                                                            long long total4, int C4, bool has_bn, bool relu, BnConsts bn, bool round_out) {
  pdl_prologue();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total4; i += (long long)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % C4);
    float4 u = ld4(in, i);
    if (has_bn) {
      const float4 sc = ldc4(bn.scale, c4), sh = ldc4(bn.shift, c4);
      u = BRE_F4(fmaf(u.x, sc.x, sh.x), fmaf(u.y, sc.y, sh.y), fmaf(u.z, sc.z, sh.z), fmaf(u.w, sc.w, sh.w));
    }
    if (res != nullptr) { const float4 r = ld4(res, i); u.x += r.x; u.y += r.y; u.z += r.z; u.w += r.w; }
    if (relu) u = BRE_F4(fmaxf(u.x, 0.f), fmaxf(u.y, 0.f), fmaxf(u.z, 0.f), fmaxf(u.w, 0.f));
    st4(out, i, round_out ? rna4(u) : u);
  }
}

__global__ void __launch_bounds__(256) bnact_tan_fwd_vec_kernel(BnActTanFwdArgs a, long long total4, int C4) {
  pdl_prologue();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total4; i += (long long)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % C4);
    float4 u = a.tin != nullptr ? ld4(a.tin, i) : make_float4(0.f, 0.f, 0.f, 0.f);
    if (a.has_bn) {
      const float4 z = ld4(a.in, i), inv = ldc4(a.bn.inv, c4), nrm = ldc4(a.bn.nrm, c4), sc = ldc4(a.bn.scale, c4);
      const float4 vg = ldc4(a.v_gamma, c4), vb = ldc4(a.v_beta, c4);
      u.x = fmaf(sc.x, u.x, fmaf(vg.x, fmaf(z.x, inv.x, nrm.x), vb.x));
      u.y = fmaf(sc.y, u.y, fmaf(vg.y, fmaf(z.y, inv.y, nrm.y), vb.y));
      u.z = fmaf(sc.z, u.z, fmaf(vg.z, fmaf(z.z, inv.z, nrm.z), vb.z));
      u.w = fmaf(sc.w, u.w, fmaf(vg.w, fmaf(z.w, inv.w, nrm.w), vb.w));
    }
    if (a.tres != nullptr) { const float4 r = ld4(a.tres, i); u.x += r.x; u.y += r.y; u.z += r.z; u.w += r.w; }
    if (a.relu) {
      const float4 o = ld4(a.out, i);
      if (!(o.x > 0.f)) u.x = 0.f;
      if (!(o.y > 0.f)) u.y = 0.f;
      if (!(o.z > 0.f)) u.z = 0.f;
      if (!(o.w > 0.f)) u.w = 0.f;
    }
    st4(a.tout, i, a.round_out ? rna4(u) : u);
  }
}

__global__ void __launch_bounds__(256) bnact_tan_bwd_vec_kernel(BnActTanBwdArgs a, long long total4, int C4) {
  pdl_prologue();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total4; i += (long long)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % C4);
    float4 tdu = ld4(a.tdout, i), du = ld4(a.dout, i);
    if (a.relu) {
      const float4 o = ld4(a.out, i);
      if (!(o.x > 0.f)) { tdu.x = 0.f; du.x = 0.f; }
      if (!(o.y > 0.f)) { tdu.y = 0.f; du.y = 0.f; }
      if (!(o.z > 0.f)) { tdu.z = 0.f; du.z = 0.f; }
      if (!(o.w > 0.f)) { tdu.w = 0.f; du.w = 0.f; }
    }
    float4 tdi = tdu;
    if (a.has_bn) {
      const float4 sc = ldc4(a.bn.scale, c4), vg = ldc4(a.v_gamma, c4), inv = ldc4(a.bn.inv, c4);
      tdi = BRE_F4(fmaf(sc.x, tdu.x, vg.x * inv.x * du.x), fmaf(sc.y, tdu.y, vg.y * inv.y * du.y), fmaf(sc.z, tdu.z, vg.z * inv.z * du.z),
                   fmaf(sc.w, tdu.w, vg.w * inv.w * du.w));
      if (a.di_cm != nullptr) {
        const float4 z = ld4(a.in, i), cv = ldc4(a.di_cv, c4), mn = ldc4(a.di_mean, c4), cm = ldc4(a.di_cm, c4);
        tdi.x += fmaf(cv.x, z.x - mn.x, cm.x); tdi.y += fmaf(cv.y, z.y - mn.y, cm.y);
        tdi.z += fmaf(cv.z, z.z - mn.z, cm.z); tdi.w += fmaf(cv.w, z.w - mn.w, cm.w);
      }
    }
    if (a.tdin != nullptr) {
      if (a.acc_in) { const float4 o = ldrw4(a.tdin, i); tdi.x += o.x; tdi.y += o.y; tdi.z += o.z; tdi.w += o.w; }
      st4(a.tdin, i, a.round_din ? rna4(tdi) : tdi);
    }
    if (a.tdres != nullptr) {
      float4 r = tdu;
      if (a.acc_res) { const float4 o = ldrw4(a.tdres, i); r.x += o.x; r.y += o.y; r.z += o.z; r.w += o.w; }
      st4(a.tdres, i, r);
    }
  }
}

// ---- (LX float4 columns) x (pixel slab) reductions: block of 256 threads = LX x LY, blockIdx.x = column group, blockIdx.y = slab --
// Per thread NV x 4 partial sums; rows of the block are summed in shared memory in fixed order, then the last-arriving block of a
// column group sums the slabs in fixed order (deterministic, like slab_reduce).
template <int NV>
__device__ __forceinline__ bool slab_reduce4(float (&v)[NV][4], int LX, int LY, float* partials, int* counters, int Cpad, int C,
                                             float (&total)[NV][4], bool defer = false) {
  __shared__ float sm4[NV * 4][257];
  __shared__ int s_last4;
  const int tid = threadIdx.x, lx = tid % LX;
#pragma unroll
  for (int k = 0; k < NV; ++k)
#pragma unroll
    for (int j = 0; j < 4; ++j) sm4[k * 4 + j][tid] = v[k][j];
  __syncthreads();
  const int c0 = (blockIdx.x * LX + lx) * 4;
  if (tid < LX && c0 < C) {
#pragma unroll
    for (int k = 0; k < NV; ++k)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float s = 0.f;
        for (int y = 0; y < LY; ++y) s += sm4[k * 4 + j][y * LX + lx];
        partials[((long long)blockIdx.y * Cpad + c0 + j) * NV + k] = s;
      }
  }
  if (defer) return false;   // summed over the slabs later, batched over all layers (launch_bn_grad_finalize)
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    const int prev = atomicAdd(counters + blockIdx.x, 1);
    s_last4 = (prev == (int)gridDim.y - 1);
    if (s_last4) counters[blockIdx.x] = 0;
  }
  __syncthreads();
  if (!s_last4) return false;
  __threadfence();
  // all 256 threads: one (quantity, channel) sum over the slabs each, in slab order (fixed), then handed to the column's owner
  __shared__ float tot4[NV][128];
  const int cols = LX * 4;
  for (int idx = tid; idx < cols * NV; idx += 256) {
    const int k = idx / cols, col = idx - k * cols;
    const int c = blockIdx.x * cols + col;
    // slabs in batches of 32 independent loads (one L2 round trip per batch instead of one per few slabs), summed in slab order
    float sum = 0.f;
    if (c < C) {
      const int ns = (int)gridDim.y;
      for (int base = 0; base < ns; base += 32) {
        float r[32];
#pragma unroll
        for (int u = 0; u < 32; ++u) r[u] = base + u < ns ? __ldcg(partials + ((long long)(base + u) * Cpad + c) * NV + k) : 0.f;
#pragma unroll
        for (int u = 0; u < 32; ++u) sum += r[u];
      }
    }
    tot4[k][col] = sum;
  }
  __syncthreads();
  if (tid < LX && c0 < C) {
#pragma unroll
    for (int k = 0; k < NV; ++k)
#pragma unroll
      for (int j = 0; j < 4; ++j) total[k][j] = tot4[k][lx * 4 + j];
    return true;
  }
  return false;
}

inline void slab_grid4(long long P, int C, dim3& grid, int& LX, int& LY, long long& pps, int waves = 2, long long target_blocks = 0) {
  const int C4 = C / 4;
  LX = C4 < 32 ? C4 : 32;
  while (256 % LX != 0) --LX;          // C4 = 16, 32, 64 ... in practice; keep LX a divisor of 256 for odd widths
  LY = 256 / LX;
  const int cg = ceil_div(C4, LX);
  // `waves` x kNumSMs blocks: 2 when the last block of a column group sums the slabs itself (a longer tail per slab), 4 when the slabs are
  // summed by a later batched kernel (deferred BN gradients, batched statistics)
  // (a batched launch over many tensors passes this tensor's share of the whole grid as `target_blocks` instead)
  const long long want = target_blocks > 0 ? target_blocks : (long long)waves * kNumSMs;
  long long slabs = (want + cg - 1) / cg;
  const long long max_slabs = (P + LY - 1) / LY;
  if (slabs > max_slabs) slabs = max_slabs;
  const long long cap = kSlabPartialFloats / (2LL * cg * LX * 4);   // partials: slabs x Cpad x (<= 2 quantities)
  if (slabs > cap) slabs = cap;
  if (slabs < 1) slabs = 1;
  pps = (P + slabs - 1) / slabs;
  slabs = (P + pps - 1) / pps;
  grid = dim3(cg, (unsigned)slabs);
}

__global__ void __launch_bounds__(256, 2) bnact_bwd_vec_kernel(BnActBwdArgs a, long long pps, int Cpad, int LX, int LY) {
  pdl_prologue();
  const int lx = threadIdx.x % LX, ly = threadIdx.x / LX;
  const int c4 = blockIdx.x * LX + lx, C4 = a.C / 4;
  const bool cv = c4 < C4;
  const long long p0 = blockIdx.y * pps;
  const long long p1 = (p0 + pps < a.P) ? p0 + pps : a.P;
  float v[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
  float4 inv = make_float4(0.f, 0.f, 0.f, 0.f), nrm = inv, scale = make_float4(1.f, 1.f, 1.f, 1.f);
  if (cv && a.has_bn) { inv = ldc4(a.bn.inv, c4); nrm = ldc4(a.bn.nrm, c4); scale = ldc4(a.bn.scale, c4); }
  if (cv) {
    // four pixel rows per trip, every load issued before the first use: the block count only gives ~16 warps per SM, and the stores
    // (which the compiler must assume to alias the loads) would otherwise serialise one row per memory round trip
    constexpr int U = 4;
    const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long long p = p0 + ly; p < p1; p += (long long)LY * U) {
      float4 du[U], y[U], z[U], qi[U], qr[U];
      bool ok[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long pp = p + (long long)u * LY;
        ok[u] = pp < p1;
        const long long o = pp * C4 + c4;
        du[u] = ok[u] ? ld4(a.dout, o) : zero4;
        y[u] = (ok[u] && a.relu) ? ld4(a.out, o) : make_float4(1.f, 1.f, 1.f, 1.f);
        z[u] = (ok[u] && a.has_bn) ? ld4(a.in, o) : zero4;
        qi[u] = (ok[u] && a.din != nullptr && a.acc_in) ? ldrw4(a.din, o) : zero4;
        qr[u] = (ok[u] && a.dres != nullptr && a.acc_res) ? ldrw4(a.dres, o) : zero4;
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (!ok[u]) continue;
        const long long o = (p + (long long)u * LY) * C4 + c4;
        float4 d = du[u];
        if (a.relu) {
          if (!(y[u].x > 0.f)) d.x = 0.f;
          if (!(y[u].y > 0.f)) d.y = 0.f;
          if (!(y[u].z > 0.f)) d.z = 0.f;
          if (!(y[u].w > 0.f)) d.w = 0.f;
        }
        float4 di = d;
        if (a.has_bn) {
          v[0][0] = fmaf(d.x, fmaf(z[u].x, inv.x, nrm.x), v[0][0]); v[0][1] = fmaf(d.y, fmaf(z[u].y, inv.y, nrm.y), v[0][1]);
          v[0][2] = fmaf(d.z, fmaf(z[u].z, inv.z, nrm.z), v[0][2]); v[0][3] = fmaf(d.w, fmaf(z[u].w, inv.w, nrm.w), v[0][3]);
          v[1][0] += d.x; v[1][1] += d.y; v[1][2] += d.z; v[1][3] += d.w;
          di = BRE_F4(scale.x * d.x, scale.y * d.y, scale.z * d.z, scale.w * d.w);
        }
        if (a.din != nullptr) {
          di.x += qi[u].x; di.y += qi[u].y; di.z += qi[u].z; di.w += qi[u].w;
          st4(a.din, o, a.round_din ? rna4(di) : di);
        }
        if (a.dres != nullptr) st4(a.dres, o, BRE_F4(d.x + qr[u].x, d.y + qr[u].y, d.z + qr[u].z, d.w + qr[u].w));
      }
    }
  }
  if (!a.has_bn || a.g_gamma == nullptr) return;  // uniform across the grid
  float tot[2][4];
  if (slab_reduce4<2>(v, LX, LY, a.partials, a.counters, Cpad, a.C, tot, a.defer != 0)) {
    st4(a.g_gamma, c4, make_float4(tot[0][0], tot[0][1], tot[0][2], tot[0][3]));
    st4(a.g_beta, c4, make_float4(tot[1][0], tot[1][1], tot[1][2], tot[1][3]));
  }
}

__global__ void __launch_bounds__(256) channel_stats_vec_kernel(const float* __restrict__ x, long long P, int C, float* mean, float* var,
                                                                float* partials, int* counters, long long pps, int Cpad, int LX, int LY) {
  pdl_prologue();
  const int lx = threadIdx.x % LX, ly = threadIdx.x / LX;
  const int c4 = blockIdx.x * LX + lx, C4 = C / 4;
  const long long p0 = blockIdx.y * pps;
  const long long p1 = (p0 + pps < P) ? p0 + pps : P;
  // shifted sums (shift = first element of the channel) keep E[x^2] - E[x]^2 well conditioned in fp32
  const float4 sh = c4 < C4 ? ldc4(x, c4) : make_float4(0.f, 0.f, 0.f, 0.f);
  float v[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
  if (c4 < C4) {
    constexpr int U = 8;   // eight independent 128-bit loads in flight per thread
    for (long long p = p0 + ly; p < p1; p += (long long)LY * U) {
      float4 t[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long pp = p + (long long)u * LY;
        t[u] = pp < p1 ? ld4(x, pp * C4 + c4) : sh;   // (a padded row contributes x - shift = 0 to both sums)
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const float a0 = t[u].x - sh.x, a1 = t[u].y - sh.y, a2 = t[u].z - sh.z, a3 = t[u].w - sh.w;
        v[0][0] += a0; v[0][1] += a1; v[0][2] += a2; v[0][3] += a3;
        v[1][0] = fmaf(a0, a0, v[1][0]); v[1][1] = fmaf(a1, a1, v[1][1]); v[1][2] = fmaf(a2, a2, v[1][2]); v[1][3] = fmaf(a3, a3, v[1][3]);
      }
    }
  }
  float tot[2][4];
  if (slab_reduce4<2>(v, LX, LY, partials, counters, Cpad, C, tot)) {
    const float shv[4] = {sh.x, sh.y, sh.z, sh.w};
    float m[4], vr[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float mj = tot[0][j] / (float)P;
      m[j] = mj + shv[j];
      vr[j] = fmaxf(tot[1][j] / (float)P - mj * mj, 0.f);
    }
    st4(mean, c4, make_float4(m[0], m[1], m[2], m[3]));
    st4(var, c4, make_float4(vr[0], vr[1], vr[2], vr[3]));
  }
}

// ---- per-channel statistics of many tensors in one launch (DeepInversion: every BN input of the forward pass) --------------------
// 53 separate slab reductions (ResNet-50) each pay a fixed two-phase overhead; batched: one launch writes the slab partials
// of all layers (blockIdx.x -> (layer, channel group, slab) through a prefix table), one launch turns them into mean / variance.
__global__ void __launch_bounds__(256) channel_stats_batched_kernel(const StatSlot* __restrict__ table, int n_layers) {
  pdl_prologue();
  __shared__ float sm4[8][257];
  int layer = 0;
  while (layer + 1 < n_layers && (int)blockIdx.x >= table[layer + 1].first_block) ++layer;
  const StatSlot e = table[layer];
  const int local = (int)blockIdx.x - e.first_block;
  const int bx = local % e.cg, by = local / e.cg;
  const int LX = e.LX, LY = e.LY, C4 = e.C / 4;
  const int tid = threadIdx.x, lx = tid % LX, ly = tid / LX;
  const int c4 = bx * LX + lx;
  const long long p0 = by * e.pps;
  const long long p1 = (p0 + e.pps < e.P) ? p0 + e.pps : e.P;
  const float4 sh = c4 < C4 ? ldc4(e.x, c4) : make_float4(0.f, 0.f, 0.f, 0.f);   // shift = first element of the channel (conditioning)
  float v[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
  if (c4 < C4) {
    constexpr int U = 8;
    for (long long p = p0 + ly; p < p1; p += (long long)LY * U) {
      float4 t[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long pp = p + (long long)u * LY;
        t[u] = pp < p1 ? ld4(e.x, pp * C4 + c4) : sh;
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const float a0 = t[u].x - sh.x, a1 = t[u].y - sh.y, a2 = t[u].z - sh.z, a3 = t[u].w - sh.w;
        v[0][0] += a0; v[0][1] += a1; v[0][2] += a2; v[0][3] += a3;
        v[1][0] = fmaf(a0, a0, v[1][0]); v[1][1] = fmaf(a1, a1, v[1][1]); v[1][2] = fmaf(a2, a2, v[1][2]); v[1][3] = fmaf(a3, a3, v[1][3]);
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 2; ++k)
#pragma unroll
    for (int j = 0; j < 4; ++j) sm4[k * 4 + j][tid] = v[k][j];
  __syncthreads();
  const int c0 = c4 * 4;
  if (tid < LX && c0 < e.C) {
#pragma unroll
    for (int k = 0; k < 2; ++k)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float sum = 0.f;
        for (int y = 0; y < LY; ++y) sum += sm4[k * 4 + j][y * LX + lx];
        e.partials[((long long)by * e.Cpad + c0 + j) * 2 + k] = sum;
      }
  }
}

__global__ void __launch_bounds__(256) channel_stats_batched_finalize_kernel(const StatSlot* __restrict__ table, int n_layers) {
  pdl_prologue();
  int layer = 0;
  while (layer + 1 < n_layers && (int)blockIdx.x >= table[layer + 1].first_group) ++layer;
  const StatSlot e = table[layer];
  const int c = ((int)blockIdx.x - e.first_group) * 256 + threadIdx.x;
  if (c >= e.C) return;
  float s0 = 0.f, s1 = 0.f;
  for (int base = 0; base < e.slabs; base += 16) {
    float r0[16], r1[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const bool ok = base + u < e.slabs;
      const float* q = e.partials + ((long long)(base + u) * e.Cpad + c) * 2;
      r0[u] = ok ? __ldcg(q) : 0.f;
      r1[u] = ok ? __ldcg(q + 1) : 0.f;
    }
#pragma unroll
    for (int u = 0; u < 16; ++u) { s0 += r0[u]; s1 += r1[u]; }
  }
  const float sh = e.x[c];
  const float m = s0 / (float)e.P;
  e.mean[c] = m + sh;
  e.var[c] = fmaxf(s1 / (float)e.P - m * m, 0.f);
}

// ---- deferred, batched finalisation of the BN parameter gradients ---------------------------------------------------------------
// Every bnact_bwd launch used to end with a serial tail: atomic ticket, the last block of each channel group re-reads the slab
// partials and sums them (on the critical path of the backward sweep 20-53 times per iteration).  With
// `defer` the kernels stop after writing their partials; one launch at the end of the sweep sums the slabs of *all* layers (one
// block per 32 channels of a layer, fixed summation order) -- the gradients of gamma / beta are only read by the matching reduction.
__global__ void __launch_bounds__(1024) bn_grad_finalize_kernel(const BnGradSlot* __restrict__ table, int n_layers) {
  // block = 32 channels x 2 quantities (64 adjacent floats of a slab row: coalesced) x 16 interleaved slices of the slab list; the
  // slices are folded in a fixed order.
  __shared__ float part[16][64];
  pdl_prologue();
  int layer = 0;
  while (layer + 1 < n_layers && (int)blockIdx.x >= table[layer + 1].first_block) ++layer;
  const BnGradSlot e = table[layer];
  const int group = (int)blockIdx.x - e.first_block;
  const int q = threadIdx.x & 63, slice = threadIdx.x >> 6;
  const int c = group * 32 + (q >> 1), k = q & 1;
  float sum = 0.f;
  if (c < e.C) {
    const float* __restrict__ src = e.partials + (long long)c * 2 + k;
    const long long pitch = (long long)e.Cpad * 2;
    int sl = slice;
    for (; sl + 48 < e.slabs; sl += 64) {
      const float v0 = __ldcg(src + sl * pitch), v1 = __ldcg(src + (sl + 16) * pitch), v2 = __ldcg(src + (sl + 32) * pitch), v3 = __ldcg(src + (sl + 48) * pitch);
      sum += v0; sum += v1; sum += v2; sum += v3;
    }
    for (; sl < e.slabs; sl += 16) sum += __ldcg(src + sl * pitch);
  }
  part[slice][q] = sum;
  __syncthreads();
  if (slice == 0 && c < e.C) {
    float t = 0.f;
#pragma unroll
    for (int u = 0; u < 16; ++u) t += part[u][q];
    (k == 0 ? e.g_gamma : e.g_beta)[c] = t;
  }
}

// ---- train-mode BatchNorm (rules in layers.cuh) -------------------------------------------------------------
__global__ void bn_train_prepare_kernel(const float* mean, const float* var, const float* gamma, const float* beta, float eps, int C,
                                        float* scale, float* shift, float* inv, float* nrm) {
  pdl_prologue();
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < C; c += gridDim.x * blockDim.x) {
    const float iv = 1.0f / sqrtf(var[c] + eps);
    const float nr = -mean[c] * iv;
    inv[c] = iv; nrm[c] = nr;
    scale[c] = gamma[c] * iv;
    shift[c] = fmaf(gamma[c], nr, beta[c]);
  }
}

__global__ void bn_train_bwd_kernel(BnTrainArgs a, long long total) {
  pdl_prologue();
  const float invP = 1.0f / (float)a.P;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % a.C);
    float du = a.dout[i];
    if (a.relu && !(a.out[i] > 0.f)) du = 0.f;
    const float xh = fmaf(a.in[i], __ldg(a.inv + c), __ldg(a.nrm + c));
    float di = __ldg(a.scale + c) * (du - __ldg(a.sum_du + c) * invP - xh * __ldg(a.sum_duxh + c) * invP);
    if (a.acc) di += a.dst[i];
    a.dst[i] = a.round_out ? tf32_rna(di) : di;
    if (a.keep_du != nullptr && i < a.C) { a.keep_du[i] = a.sum_du[i]; a.keep_duxh[i] = a.sum_duxh[i]; }
  }
}

__global__ void bn_train_tan_stats_kernel(BnTrainArgs a, float* m1, float* m2, float* partials, int* counters, long long pps, int Cpad) {
  pdl_prologue();
  const int c = blockIdx.x * 32 + threadIdx.x;
  const bool cv = c < a.C;
  const long long p0 = blockIdx.y * pps;
  const long long p1 = (p0 + pps < a.P) ? p0 + pps : a.P;
  float v[2] = {0.f, 0.f};
  if (cv) {
    const float inv = __ldg(a.inv + c), nrm = __ldg(a.nrm + c);
    for (long long p = p0 + threadIdx.y; p < p1; p += 8) {
      const long long o = p * a.C + c;
      const float xd = a.xd[o];
      v[0] += xd;
      v[1] = fmaf(fmaf(a.in[o], inv, nrm), xd, v[1]);
    }
  }
  float tot[2];
  if (slab_reduce<2>(v, partials, counters, Cpad, tot) && cv) {
    m1[c] = tot[0] / (float)a.P;
    m2[c] = tot[1] / (float)a.P;
  }
}

__global__ void bn_train_tan_fwd_kernel(BnTrainArgs a, long long total) {
  pdl_prologue();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % a.C);
    const float xh = fmaf(a.in[i], __ldg(a.inv + c), __ldg(a.nrm + c));
    float u = fmaf(__ldg(a.v_gamma + c), xh, __ldg(a.v_beta + c)) +
              __ldg(a.scale + c) * (a.xd[i] - __ldg(a.m1 + c) - xh * __ldg(a.m2 + c));
    if (a.tres != nullptr) u += a.tres[i];
    if (a.relu && !(a.out[i] > 0.f)) u = 0.f;
    a.dst[i] = a.round_out ? tf32_rna(u) : u;
  }
}

__global__ void bn_train_tanbwd_stats_kernel(BnTrainArgs a, float* b1, float* b2, float* partials, int* counters, long long pps, int Cpad) {
  pdl_prologue();
  const int c = blockIdx.x * 32 + threadIdx.x;
  const bool cv = c < a.C;
  const long long p0 = blockIdx.y * pps;
  const long long p1 = (p0 + pps < a.P) ? p0 + pps : a.P;
  float v[2] = {0.f, 0.f};
  if (cv) {
    const float inv = __ldg(a.inv + c), nrm = __ldg(a.nrm + c), m1 = __ldg(a.m1 + c), m2 = __ldg(a.m2 + c);
    for (long long p = p0 + threadIdx.y; p < p1; p += 8) {
      const long long o = p * a.C + c;
      float du = a.dout[o], tdu = a.tdout[o];
      if (a.relu && !(a.out[o] > 0.f)) { du = 0.f; tdu = 0.f; }
      const float xh = fmaf(a.in[o], inv, nrm);
      const float xhd = inv * (a.xd[o] - m1 - xh * m2);
      v[0] += tdu;
      v[1] += fmaf(tdu, xh, du * xhd);
    }
  }
  float tot[2];
  if (slab_reduce<2>(v, partials, counters, Cpad, tot) && cv) {
    b1[c] = tot[0] / (float)a.P;
    b2[c] = tot[1] / (float)a.P;
    if (a.tg_beta != nullptr) { a.tg_beta[c] = tot[0]; a.tg_gamma[c] = tot[1]; }
  }
}

__global__ void bn_train_tan_bwd_kernel(BnTrainArgs a, long long total) {
  pdl_prologue();
  const float invP = 1.0f / (float)a.P;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % a.C);
    float du = a.dout[i], tdu = a.tdout[i];
    if (a.relu && !(a.out[i] > 0.f)) { du = 0.f; tdu = 0.f; }
    const float inv = __ldg(a.inv + c), scale = __ldg(a.scale + c), m2 = __ldg(a.m2 + c);
    const float xh = fmaf(a.in[i], inv, __ldg(a.nrm + c));
    const float xhd = inv * (a.xd[i] - __ldg(a.m1 + c) - xh * m2);
    const float a1 = __ldg(a.sum_du + c) * invP, a2 = __ldg(a.sum_duxh + c) * invP;
    const float w = du - a1 - xh * a2;
    const float wd = tdu - __ldg(a.b1 + c) - xhd * a2 - xh * __ldg(a.b2 + c);
    float tdi = (__ldg(a.v_gamma + c) * inv - scale * inv * m2) * w + scale * wd;
    if (a.dst != nullptr) {
      if (a.acc) tdi += a.dst[i];
      a.dst[i] = a.round_out ? tf32_rna(tdi) : tdi;
    }
    if (a.dres != nullptr) a.dres[i] = a.acc_res ? a.dres[i] + tdu : tdu;
  }
}

// ---- pooling ---------------------------------------------------------------------------------------
__global__ void maxpool_fwd_kernel(const float* __restrict__ in, float* __restrict__ out, int* __restrict__ idx, PoolGeom g,
                                   long long total) {
  pdl_prologue();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % g.C);
    long long t = i / g.C;
    const int q = (int)(t % g.Wo); t /= g.Wo;
    const int p = (int)(t % g.Ho);
    const int n = (int)(t / g.Ho);
    const int h0 = p * g.stride - g.pad, w0 = q * g.stride - g.pad;
    float best = -FLT_MAX * 2.f;  // -inf
    int bi = -1;
    for (int r = 0; r < g.k; ++r) {
      const int h = h0 + r;
      if (h < 0 || h >= g.H) continue;
      for (int s = 0; s < g.k; ++s) {
        const int w = w0 + s;
        if (w < 0 || w >= g.W) continue;
        const float v = in[((long long)(n * g.H + h) * g.W + w) * g.C + c];
        if (v > best || v != v || bi < 0) { best = v; bi = h * g.W + w; }
      }
    }
    out[i] = best;
    idx[i] = bi;
  }
}

__global__ void maxpool_bwd_kernel(const float* __restrict__ dout, const int* __restrict__ idx, float* __restrict__ din, bool acc,
                                   PoolGeom g, long long total) {
  pdl_prologue();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % g.C);
    long long t = i / g.C;
    const int w = (int)(t % g.W); t /= g.W;
    const int h = (int)(t % g.H);
    const int n = (int)(t / g.H);
    const int me = h * g.W + w;
    int p_lo = h + g.pad - g.k + 1; p_lo = p_lo > 0 ? (p_lo + g.stride - 1) / g.stride : 0;
    int q_lo = w + g.pad - g.k + 1; q_lo = q_lo > 0 ? (q_lo + g.stride - 1) / g.stride : 0;
    int p_hi = (h + g.pad) / g.stride; if (p_hi > g.Ho - 1) p_hi = g.Ho - 1;
    int q_hi = (w + g.pad) / g.stride; if (q_hi > g.Wo - 1) q_hi = g.Wo - 1;
    float s = 0.f;
    for (int p = p_lo; p <= p_hi; ++p)
      for (int q = q_lo; q <= q_hi; ++q) {
        const long long o = ((long long)(n * g.Ho + p) * g.Wo + q) * g.C + c;
        if (idx[o] == me) s += dout[o];
      }
    din[i] = acc ? din[i] + s : s;
  }
}

// 128-bit forms of the three pooling kernels (C % 4 == 0, 16-byte aligned tensors, < 2^31 elements): a thread owns four adjacent
// channels of one pixel, so the index arithmetic is paid once per 16 bytes and every access is a full-width load / store.  The
// scalar kernels above spend most of their time in 64-bit divisions.
__device__ __forceinline__ void take_max(float v, int at, float& best, int& bi) {
  if (v > best || v != v || bi < 0) { best = v; bi = at; }
}
__global__ void __launch_bounds__(kEwThreads) maxpool_fwd_vec_kernel(const float4* __restrict__ in, float4* __restrict__ out, int4* __restrict__ idx,
                                                                     PoolGeom g, int total4) {
  pdl_prologue();
  const int C4 = g.C >> 2;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += gridDim.x * blockDim.x) {
    const int c4 = i % C4;
    int t = i / C4;
    const int q = t % g.Wo; t /= g.Wo;
    const int p = t % g.Ho;
    const int n = t / g.Ho;
    const int h0 = p * g.stride - g.pad, w0 = q * g.stride - g.pad;
    float4 best = make_float4(-FLT_MAX * 2.f, -FLT_MAX * 2.f, -FLT_MAX * 2.f, -FLT_MAX * 2.f);  // -inf
    int4 bi = make_int4(-1, -1, -1, -1);
    for (int r = 0; r < g.k; ++r) {
      const int h = h0 + r;
      if (h < 0 || h >= g.H) continue;
      for (int s = 0; s < g.k; ++s) {
        const int w = w0 + s;
        if (w < 0 || w >= g.W) continue;
        const int at = h * g.W + w;
        const float4 v = in[(long long)(n * g.H * g.W + at) * C4 + c4];
        take_max(v.x, at, best.x, bi.x); take_max(v.y, at, best.y, bi.y);
        take_max(v.z, at, best.z, bi.z); take_max(v.w, at, best.w, bi.w);
      }
    }
    out[i] = best;
    idx[i] = bi;
  }
}

template <bool ACC>
__global__ void __launch_bounds__(kEwThreads) maxpool_bwd_vec_kernel(const float4* __restrict__ dout, const int4* __restrict__ idx,
                                                                     float4* __restrict__ din, PoolGeom g, int total4) {
  pdl_prologue();
  const int C4 = g.C >> 2;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += gridDim.x * blockDim.x) {
    const int c4 = i % C4;
    int t = i / C4;
    const int w = t % g.W; t /= g.W;
    const int h = t % g.H;
    const int n = t / g.H;
    const int me = h * g.W + w;
    int p_lo = h + g.pad - g.k + 1; p_lo = p_lo > 0 ? (p_lo + g.stride - 1) / g.stride : 0;
    int q_lo = w + g.pad - g.k + 1; q_lo = q_lo > 0 ? (q_lo + g.stride - 1) / g.stride : 0;
    int p_hi = (h + g.pad) / g.stride; if (p_hi > g.Ho - 1) p_hi = g.Ho - 1;
    int q_hi = (w + g.pad) / g.stride; if (q_hi > g.Wo - 1) q_hi = g.Wo - 1;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int p = p_lo; p <= p_hi; ++p)
      for (int q = q_lo; q <= q_hi; ++q) {
        const long long o = (long long)((n * g.Ho + p) * g.Wo + q) * C4 + c4;
        const int4 ix = idx[o];
        const float4 d = dout[o];
        if (ix.x == me) s.x += d.x;
        if (ix.y == me) s.y += d.y;
        if (ix.z == me) s.z += d.z;
        if (ix.w == me) s.w += d.w;
      }
    if (ACC) { const float4 o = din[i]; s.x += o.x; s.y += o.y; s.z += o.z; s.w += o.w; }
    din[i] = s;
  }
}

__global__ void __launch_bounds__(kEwThreads) maxpool_gather_vec_kernel(const float* __restrict__ tin, const int4* __restrict__ idx,
                                                                        float4* __restrict__ tout, PoolGeom g, int total4) {
  pdl_prologue();
  const int C4 = g.C >> 2;
  const int per = C4 * g.Ho * g.Wo;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += gridDim.x * blockDim.x) {
    const int c = (i % C4) * 4;
    const long long base = (long long)(i / per) * g.H * g.W;
    const int4 ix = idx[i];
    float4 v;
    v.x = tin[(base + ix.x) * g.C + c];
    v.y = tin[(base + ix.y) * g.C + c + 1];
    v.z = tin[(base + ix.z) * g.C + c + 2];
    v.w = tin[(base + ix.w) * g.C + c + 3];
    tout[i] = v;
  }
}

inline bool pool_vec_ok(const PoolGeom& g, const void* a, const void* b, const void* c) {
  const long long big = (long long)g.N * g.H * g.W * g.C;
  return vec_ok(g.C) && big < (1LL << 31) && ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c)) & 15) == 0;
}

__global__ void maxpool_gather_kernel(const float* __restrict__ tin, const int* __restrict__ idx, float* __restrict__ tout,
                                      PoolGeom g, long long total) {
  pdl_prologue();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % g.C);
    const long long n = i / ((long long)g.C * g.Ho * g.Wo);
    tout[i] = tin[(n * g.H * g.W + idx[i]) * g.C + c];
  }
}

__global__ void avgpool_fwd_kernel(const float* __restrict__ in, float* __restrict__ out, int N, int HW, int C) {
  pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * C) return;
  const int n = i / C, c = i - n * C;
  float s = 0.f;
  for (int p = 0; p < HW; ++p) s += in[((long long)n * HW + p) * C + c];
  out[i] = s / (float)HW;
}

__global__ void avgpool_bwd_kernel(const float* __restrict__ dout, float* __restrict__ din, bool acc, long long total, int HW, int C) {
  pdl_prologue();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long n = i / ((long long)C * HW);
    const float v = dout[n * C + c] / (float)HW;
    din[i] = acc ? din[i] + v : v;
  }
}

// ---- softmax cross-entropy -------------------------------------------------------------------------
// Softmax cross-entropy, mean over N.  Targets: class indices, or -- joint data / label optimisation
// (optimization_with_label_attack.py:154: `labels.softmax(dim=-1)` handed to the loss) -- class probabilities q [N, C].
__global__ void ce_fwd_kernel(const float* __restrict__ logits, const long long* __restrict__ labels, const float* __restrict__ q, int N,
                              int C, float* p, float* loss_n, float* dlogits) {
  pdl_prologue();
  __shared__ double scratch[32];
  __shared__ float s_max, s_sum;
  const int n = blockIdx.x;
  const float* z = logits + (long long)n * C;
  float mx = -FLT_MAX;
  for (int c = threadIdx.x; c < C; c += blockDim.x) mx = fmaxf(mx, z[c]);
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  __shared__ float wmax[32];
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
  for (int c = threadIdx.x; c < C; c += blockDim.x) part += (double)expf(z[c] - mx);
  const double tot = block_sum(part, scratch);
  if (threadIdx.x == 0) s_sum = (float)tot;
  __syncthreads();
  const float sum = s_sum;
  const float invN = 1.0f / (float)N;
  if (q != nullptr) {
    const float lse = mx + logf(sum);
    double lpart = 0.0;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      const float pc = expf(z[c] - mx) / sum, qc = q[(long long)n * C + c];
      p[(long long)n * C + c] = pc;
      dlogits[(long long)n * C + c] = (pc - qc) * invN;
      lpart -= (double)qc * (double)(z[c] - lse);
    }
    const double ltot = block_sum(lpart, scratch);
    if (threadIdx.x == 0) loss_n[n] = (float)ltot;
    return;
  }
  const int y = (int)labels[n];
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float pc = expf(z[c] - mx) / sum;
    p[(long long)n * C + c] = pc;
    dlogits[(long long)n * C + c] = (pc - (c == y ? 1.f : 0.f)) * invN;
  }
  if (threadIdx.x == 0) loss_n[n] = -(z[y] - mx - logf(sum));
}

// d(objective)/d(target probabilities): the matching term sees q only through dL/dq = -log_softmax(z) / N, whose tangent in
// the weight direction v is -(zdot - <p, zdot>) / N; the task-loss regulariser adds task_reg * dL/dq itself.
__global__ void ce_label_grad_kernel(const float* __restrict__ logits, const float* __restrict__ p, const float* __restrict__ zdot, int N,
                                     int C, float task_reg, float* __restrict__ out) {
  pdl_prologue();
  __shared__ double scratch[32];
  __shared__ float s_dot, s_lse;
  const int n = blockIdx.x;
  const float* z = logits + (long long)n * C;
  const float* pp = p + (long long)n * C;
  const float* zz = zdot + (long long)n * C;
  double part = 0.0;
  for (int c = threadIdx.x; c < C; c += blockDim.x) part += (double)pp[c] * (double)zz[c];
  const double tot = block_sum(part, scratch);
  if (threadIdx.x == 0) s_dot = (float)tot;
  __syncthreads();
  if (task_reg != 0.f) {   // log-sum-exp of the row (uniform branch)
    float mx = -FLT_MAX;
    for (int c = threadIdx.x; c < C; c += blockDim.x) mx = fmaxf(mx, z[c]);
    __shared__ float wmax[32];
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = mx;
    __syncthreads();
    mx = wmax[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) mx = fmaxf(mx, wmax[w]);
    double spart = 0.0;
    for (int c = threadIdx.x; c < C; c += blockDim.x) spart += (double)expf(z[c] - mx);
    const double stot = block_sum(spart, scratch);
    if (threadIdx.x == 0) s_lse = mx + logf((float)stot);
    __syncthreads();
  }
  const float dot = s_dot, invN = 1.0f / (float)N;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float v = -(zz[c] - dot) * invN;
    if (task_reg != 0.f) v -= task_reg * (z[c] - s_lse) * invN;
    out[(long long)n * C + c] = v;
  }
}

__global__ void ce_tan_bwd_kernel(const float* __restrict__ p, const float* __restrict__ zdot, int N, int C, float* tdl) {
  pdl_prologue();
  __shared__ double scratch[32];
  __shared__ float s_dot;
  const int n = blockIdx.x;
  const float* pp = p + (long long)n * C;
  const float* zz = zdot + (long long)n * C;
  double part = 0.0;
  for (int c = threadIdx.x; c < C; c += blockDim.x) part += (double)pp[c] * (double)zz[c];
  const double tot = block_sum(part, scratch);
  if (threadIdx.x == 0) s_dot = (float)tot;
  __syncthreads();
  const float dot = s_dot, invN = 1.0f / (float)N;
  for (int c = threadIdx.x; c < C; c += blockDim.x) tdl[(long long)n * C + c] = pp[c] * (zz[c] - dot) * invN;
}

// the tangent seed plus coef * (p - onehot(y)) / N: the task-loss term of the last local step of a FedAvg evaluation, which
// enters that step's tangent-backward stream scaled by -1/lr (DESIGN.md section 3.1).  ROUND: output on the TF32 grid.
template <bool ROUND>
__global__ void ce_tan_bwd_seed_kernel(const float* __restrict__ p, const float* __restrict__ zdot, const long long* __restrict__ labels,
                                       int N, int C, float coef, float* tdl) {
  pdl_prologue();
  __shared__ double scratch[32];
  __shared__ float s_dot;
  const int n = blockIdx.x;
  const float* pp = p + (long long)n * C;
  const float* zz = zdot + (long long)n * C;
  double part = 0.0;
  for (int c = threadIdx.x; c < C; c += blockDim.x) part += (double)pp[c] * (double)zz[c];
  const double tot = block_sum(part, scratch);
  if (threadIdx.x == 0) s_dot = (float)tot;
  __syncthreads();
  const float dot = s_dot, invN = 1.0f / (float)N;
  const int y = (int)labels[n];
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float t = fmaf(coef, (pp[c] - (c == y ? 1.f : 0.f)) * invN, pp[c] * (zz[c] - dot) * invN);
    tdl[(long long)n * C + c] = ROUND ? tf32_rna(t) : t;
  }
}

// ---- layout ----------------------------------------------------------------------------------------
__global__ void permute_kernel(const float* __restrict__ src, float* __restrict__ dst, int O, int I, int HW, bool inverse,
                               long long total) {
  pdl_prologue();
  // index space of the OHWI side (coalesced writes forward, coalesced reads inverse)
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ic = (int)(i % I);
    long long t = i / I;
    const int hw = (int)(t % HW);
    const long long o = t / HW;
    const long long j = (o * I + ic) * HW + hw;  // OIHW side
    if (!inverse) dst[i] = src[j]; else dst[j] = src[i];
  }
}

__global__ void axpy_kernel(const float* __restrict__ x, float* __restrict__ y, float alpha, long long n) {
  pdl_prologue();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    y[i] = fmaf(alpha, x[i], y[i]);
}

}  // namespace

int launch_bn_prepare(const float* gamma, const float* beta, const float* rm, const float* rv, float eps, int C,
                      float* scale, float* shift, float* inv, float* nrm, cudaStream_t s) {
  BRE_KLAUNCH(bn_prepare_kernel, ceil_div(C, 128), 128, 0, s, gamma, beta, rm, rv, eps, C, scale, shift, inv, nrm);
  BRE_CHECK_LAUNCH();
  return 0;
}

int launch_bnact_fwd(const float* in, const float* res, float* out, long long P, int C, bool has_bn, bool relu,
                     BnConsts bn, bool round_out, cudaStream_t s) {
  const long long total = P * C;
  if (vec_ok(C)) {
    BRE_KLAUNCH(bnact_fwd_vec_kernel, ew_grid(total / 4), kEwThreads, 0, s, in, res, out, total / 4, C / 4, has_bn, relu, bn, round_out);
    BRE_CHECK_LAUNCH();
    return 0;
  }
  BRE_KLAUNCH(bnact_fwd_kernel, ew_grid(total), kEwThreads, 0, s, in, res, out, total, C, has_bn, relu, bn, round_out);
  BRE_CHECK_LAUNCH();
  return 0;
}

// fills the geometry fields of a StatSlot (x, partials, mean, var and the block / group offsets are the caller's); false if the
// 128-bit path does not apply to this channel count
bool channel_stats_plan(long long P, int C, StatSlot* slot, long long target_blocks) {
  if (!vec_ok(C)) return false;
  dim3 grid;
  int LX, LY;
  long long pps;
  slab_grid4(P, C, grid, LX, LY, pps, 4, target_blocks);
  slot->P = P; slot->pps = pps; slot->C = C; slot->LX = LX; slot->LY = LY; slot->cg = (int)grid.x; slot->slabs = (int)grid.y;
  slot->Cpad = (int)(grid.x * LX * 4);
  return true;
}
int launch_channel_stats_batched(const StatSlot* table_dev, int n_layers, int total_blocks, int total_groups, cudaStream_t s) {
  BRE_KLAUNCH(channel_stats_batched_kernel, total_blocks, 256, 0, s, table_dev, n_layers);
  BRE_KLAUNCH(channel_stats_batched_finalize_kernel, total_groups, 256, 0, s, table_dev, n_layers);
  BRE_CHECK_LAUNCH();
  return 0;
}

void bnact_bwd_plan(long long P, int C, int* slabs, int* Cpad) {   // geometry of a *deferred* launch_bnact_bwd
  dim3 grid, block;
  long long pps;
  if (vec_ok(C)) {
    int LX, LY;
    slab_grid4(P, C, grid, LX, LY, pps, 4);
    *Cpad = (int)(grid.x * LX * 4);
  } else {
    slab_grid(P, C, grid, block, pps);
    *Cpad = (int)(grid.x * 32);
  }
  *slabs = (int)grid.y;
}

int launch_bn_grad_finalize(const BnGradSlot* table_dev, int n_layers, int total_blocks, cudaStream_t s) {
  if (n_layers <= 0 || total_blocks <= 0) return 0;
  BRE_KLAUNCH(bn_grad_finalize_kernel, total_blocks, 1024, 0, s, table_dev, n_layers);
  BRE_CHECK_LAUNCH();
  return 0;
}

int launch_bnact_bwd(const BnActBwdArgs& a, cudaStream_t s) {
  dim3 grid, block;
  long long pps;
  if (vec_ok(a.C)) {
    int LX, LY;
    slab_grid4(a.P, a.C, grid, LX, LY, pps, a.defer ? 4 : 2);
    BRE_KLAUNCH(bnact_bwd_vec_kernel, grid, 256, 0, s, a, pps, (int)(grid.x * LX * 4), LX, LY);
    BRE_CHECK_LAUNCH();
    return 0;
  }
  slab_grid(a.P, a.C, grid, block, pps);
  BRE_KLAUNCH(bnact_bwd_kernel, grid, block, 0, s, a, pps, grid.x * 32);
  BRE_CHECK_LAUNCH();
  return 0;
}

int launch_bnact_tan_fwd(const BnActTanFwdArgs& a, cudaStream_t s) {
  const long long total = a.P * a.C;
  if (vec_ok(a.C)) {
    BRE_KLAUNCH(bnact_tan_fwd_vec_kernel, ew_grid(total / 4), kEwThreads, 0, s, a, total / 4, a.C / 4);
    BRE_CHECK_LAUNCH();
    return 0;
  }
  BRE_KLAUNCH(bnact_tan_fwd_kernel, ew_grid(total), kEwThreads, 0, s, a, total);
  BRE_CHECK_LAUNCH();
  return 0;
}

int launch_axpby(const float* x, const float* y, float alpha, float* out, long long n, cudaStream_t s) {
  if (n % 4 != 0) { set_error("axpby: length must be a multiple of 4"); return -1; }
  BRE_KLAUNCH(axpby_kernel, ew_grid(n / 4), kEwThreads, 0, s, x, y, alpha, out, n / 4);
  return 0;
}

int launch_round_tf32(const float* src, float* dst, long long n, cudaStream_t s) {
  if (n % 4 != 0) { set_error("round_tf32: length must be a multiple of 4"); return -1; }
  BRE_KLAUNCH(round_tf32_kernel, ew_grid(n / 4), kEwThreads, 0, s, src, dst, n / 4);
  return 0;
}

int launch_bnact_tan_bwd(const BnActTanBwdArgs& a, cudaStream_t s) {
  if (a.has_bn && a.tg_gamma != nullptr) {
    dim3 grid, block;
    long long pps;
    slab_grid(a.P, a.C, grid, block, pps);
    BRE_KLAUNCH(bnact_tan_bwd_g_kernel, grid, block, 0, s, a, pps, (int)(grid.x * 32));
    return 0;
  }
  const long long total = a.P * a.C;
  if (vec_ok(a.C)) {
    BRE_KLAUNCH(bnact_tan_bwd_vec_kernel, ew_grid(total / 4), kEwThreads, 0, s, a, total / 4, a.C / 4);
    BRE_CHECK_LAUNCH();
    return 0;
  }
  BRE_KLAUNCH(bnact_tan_bwd_kernel, ew_grid(total), kEwThreads, 0, s, a, total);
  BRE_CHECK_LAUNCH();
  return 0;
}

int launch_bn_train_prepare(const float* mean, const float* var, const float* gamma, const float* beta, float eps, int C, float* scale,
                            float* shift, float* inv, float* nrm, cudaStream_t s) {
  BRE_KLAUNCH(bn_train_prepare_kernel, ceil_div(C, 128), 128, 0, s, mean, var, gamma, beta, eps, C, scale, shift, inv, nrm);
  return 0;
}
int launch_bn_train_bwd(const BnTrainArgs& a, cudaStream_t s) {
  const long long total = a.P * a.C;
  BRE_KLAUNCH(bn_train_bwd_kernel, ew_grid(total), kEwThreads, 0, s, a, total);
  return 0;
}
int launch_bn_train_tan_stats(const BnTrainArgs& a, float* m1, float* m2, float* partials, int* counters, cudaStream_t s) {
  dim3 grid, block;
  long long pps;
  slab_grid(a.P, a.C, grid, block, pps);
  BRE_KLAUNCH(bn_train_tan_stats_kernel, grid, block, 0, s, a, m1, m2, partials, counters, pps, (int)(grid.x * 32));
  return 0;
}
int launch_bn_train_tan_fwd(const BnTrainArgs& a, cudaStream_t s) {
  const long long total = a.P * a.C;
  BRE_KLAUNCH(bn_train_tan_fwd_kernel, ew_grid(total), kEwThreads, 0, s, a, total);
  return 0;
}
int launch_bn_train_tanbwd_stats(const BnTrainArgs& a, float* b1, float* b2, float* partials, int* counters, cudaStream_t s) {
  dim3 grid, block;
  long long pps;
  slab_grid(a.P, a.C, grid, block, pps);
  BRE_KLAUNCH(bn_train_tanbwd_stats_kernel, grid, block, 0, s, a, b1, b2, partials, counters, pps, (int)(grid.x * 32));
  return 0;
}
int launch_bn_train_tan_bwd(const BnTrainArgs& a, cudaStream_t s) {
  const long long total = a.P * a.C;
  BRE_KLAUNCH(bn_train_tan_bwd_kernel, ew_grid(total), kEwThreads, 0, s, a, total);
  return 0;
}

int launch_channel_sum(const float* x, long long P, int C, float* out, float* partials, int* counters, cudaStream_t s) {
  dim3 grid, block;
  long long pps;
  slab_grid(P, C, grid, block, pps);
  BRE_KLAUNCH(channel_sum_kernel, grid, block, 0, s, x, P, C, out, partials, counters, pps, grid.x * 32);
  BRE_CHECK_LAUNCH();
  return 0;
}

int launch_channel_stats(const float* x, long long P, int C, float* mean, float* var, float* partials, int* counters,
                         cudaStream_t s) {
  dim3 grid, block;
  long long pps;
  if (vec_ok(C)) {
    int LX, LY;
    slab_grid4(P, C, grid, LX, LY, pps);
    BRE_KLAUNCH(channel_stats_vec_kernel, grid, 256, 0, s, x, P, C, mean, var, partials, counters, pps, (int)(grid.x * LX * 4), LX, LY);
    BRE_CHECK_LAUNCH();
    return 0;
  }
  slab_grid(P, C, grid, block, pps);
  BRE_KLAUNCH(channel_stats_kernel, grid, block, 0, s, x, P, C, mean, var, partials, counters, pps, grid.x * 32);
  BRE_CHECK_LAUNCH();
  return 0;
}

int launch_maxpool_fwd(const float* in, float* out, int* idx, PoolGeom g, cudaStream_t s) {
  const long long total = (long long)g.N * g.Ho * g.Wo * g.C;
  if (pool_vec_ok(g, in, out, idx)) {
    BRE_KLAUNCH(maxpool_fwd_vec_kernel, ew_grid(total / 4), kEwThreads, 0, s, reinterpret_cast<const float4*>(in), reinterpret_cast<float4*>(out),
                reinterpret_cast<int4*>(idx), g, (int)(total / 4));
    BRE_CHECK_LAUNCH();
    return 0;
  }
  BRE_KLAUNCH(maxpool_fwd_kernel, ew_grid(total), kEwThreads, 0, s, in, out, idx, g, total);
  BRE_CHECK_LAUNCH();
  return 0;
}
int launch_maxpool_bwd(const float* dout, const int* idx, float* din, bool acc, PoolGeom g, cudaStream_t s) {
  const long long total = (long long)g.N * g.H * g.W * g.C;
  if (pool_vec_ok(g, dout, idx, din)) {
    const float4* d4 = reinterpret_cast<const float4*>(dout);
    const int4* i4 = reinterpret_cast<const int4*>(idx);
    if (acc) BRE_KLAUNCH(maxpool_bwd_vec_kernel<true>, ew_grid(total / 4), kEwThreads, 0, s, d4, i4, reinterpret_cast<float4*>(din), g, (int)(total / 4));
    else BRE_KLAUNCH(maxpool_bwd_vec_kernel<false>, ew_grid(total / 4), kEwThreads, 0, s, d4, i4, reinterpret_cast<float4*>(din), g, (int)(total / 4));
    BRE_CHECK_LAUNCH();
    return 0;
  }
  BRE_KLAUNCH(maxpool_bwd_kernel, ew_grid(total), kEwThreads, 0, s, dout, idx, din, acc, g, total);
  BRE_CHECK_LAUNCH();
  return 0;
}
int launch_maxpool_gather(const float* tin, const int* idx, float* tout, PoolGeom g, cudaStream_t s) {
  const long long total = (long long)g.N * g.Ho * g.Wo * g.C;
  if (pool_vec_ok(g, tin, idx, tout)) {
    BRE_KLAUNCH(maxpool_gather_vec_kernel, ew_grid(total / 4), kEwThreads, 0, s, tin, reinterpret_cast<const int4*>(idx), reinterpret_cast<float4*>(tout), g,
                (int)(total / 4));
    BRE_CHECK_LAUNCH();
    return 0;
  }
  BRE_KLAUNCH(maxpool_gather_kernel, ew_grid(total), kEwThreads, 0, s, tin, idx, tout, g, total);
  BRE_CHECK_LAUNCH();
  return 0;
}
int launch_avgpool_fwd(const float* in, float* out, int N, int HW, int C, cudaStream_t s) {
  BRE_KLAUNCH(avgpool_fwd_kernel, ceil_div((long long)N * C, 128), 128, 0, s, in, out, N, HW, C);
  BRE_CHECK_LAUNCH();
  return 0;
}
int launch_avgpool_bwd(const float* dout, float* din, bool acc, int N, int HW, int C, cudaStream_t s) {
  const long long total = (long long)N * HW * C;
  BRE_KLAUNCH(avgpool_bwd_kernel, ew_grid(total), kEwThreads, 0, s, dout, din, acc, total, HW, C);
  BRE_CHECK_LAUNCH();
  return 0;
}

int launch_ce_fwd(const float* logits, const long long* labels, const float* q, int N, int C, float* p, float* loss_n,
                  float* dlogits, cudaStream_t s) {
  BRE_KLAUNCH(ce_fwd_kernel, N, 256, 0, s, logits, labels, q, N, C, p, loss_n, dlogits);
  BRE_CHECK_LAUNCH();
  return 0;
}
int launch_ce_label_grad(const float* logits, const float* p, const float* zdot, int N, int C, float task_reg, float* out, cudaStream_t s) {
  BRE_KLAUNCH(ce_label_grad_kernel, N, 256, 0, s, logits, p, zdot, N, C, task_reg, out);
  BRE_CHECK_LAUNCH();
  return 0;
}
int launch_ce_tan_bwd_seeded(const float* p, const float* zdot, const long long* labels, int N, int C, float coef, float* tdlogits,
                             bool round_out, cudaStream_t s) {
  if (round_out) BRE_KLAUNCH(ce_tan_bwd_seed_kernel<true>, N, 256, 0, s, p, zdot, labels, N, C, coef, tdlogits);
  else BRE_KLAUNCH(ce_tan_bwd_seed_kernel<false>, N, 256, 0, s, p, zdot, labels, N, C, coef, tdlogits);
  BRE_CHECK_LAUNCH();
  return 0;
}
int launch_ce_tan_bwd(const float* p, const float* zdot, int N, int C, float* tdlogits, cudaStream_t s) {
  BRE_KLAUNCH(ce_tan_bwd_kernel, N, 256, 0, s, p, zdot, N, C, tdlogits);
  BRE_CHECK_LAUNCH();
  return 0;
}

int launch_permute(const float* src, float* dst, int O, int I, int HW, bool inverse, cudaStream_t s) {
  const long long total = (long long)O * I * HW;
  BRE_KLAUNCH(permute_kernel, ew_grid(total), kEwThreads, 0, s, src, dst, O, I, HW, inverse, total);
  BRE_CHECK_LAUNCH();
  return 0;
}
int launch_axpy(const float* x, float* y, float alpha, long long n, cudaStream_t s) {
  BRE_KLAUNCH(axpy_kernel, ew_grid(n), kEwThreads, 0, s, x, y, alpha, n);
  BRE_CHECK_LAUNCH();
  return 0;
}

}  // namespace bre
