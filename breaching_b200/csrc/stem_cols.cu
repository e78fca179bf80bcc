// The convolution fed by the candidate (ResNet stem 7x7/2 on 3 channels, first 3x3 conv of the ConvNets) on the tensor cores.
//
// With 3 input channels the implicit-GEMM k-blocks cannot come from a tensor map (one pixel is 12 bytes), so this layer would
// run on the fp32 SIMT kernels.  Here the candidate is unfolded once per forward into a column matrix
//     xcol[m = (n, p, q)][k = (r, s, c)]   (K = R*S*Ci zero-padded to a multiple of 64, values on the TF32 grid)
// and the four contractions of the layer become plain 1x1 "convolutions" over xcol that the tensor-core kernel covers:
//     F / TF :  fprop  xcol . Wcol^T , xcol . Vcol^T          B :  wgrad  dout^T . xcol  -> Gcol
//     TB     :  dgrad  [td | d] . [Wcol ; Vcol] -> dcol[m][k], folded back onto the NCHW candidate gradient by col2im
// (an explicit GEMM + col2im is the textbook form of a strided dgrad: every input pixel gathers the <= ceil(R/stride)^2 column
// entries that touched it -- no atomics, fixed summation order).  Wcol / Vcol are the zero-padded [Co][K] copies of the OHWI
// weight / direction, Gcol is unpadded back into the gradient arena.
#include "layers.cuh"

namespace bre {
namespace {

struct ColGeom { int N, C, H, W, Ho, Wo, R, S, stride, pad, K, Kp; };

// xcol[m][k4 .. k4+3]: one thread per 16-byte granule
__global__ void __launch_bounds__(256) stem_im2col_kernel(const float* __restrict__ x, float* __restrict__ xcol, ColGeom g, long long total,
                                                          int round_out) {
  pdl_prologue();
  const int gran = g.Kp >> 2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long m = i / gran;
    const int k0 = (int)(i - m * gran) << 2;
    const int HoWo = g.Ho * g.Wo;
    const int n = (int)(m / HoWo), rem = (int)(m - (long long)n * HoWo);
    const int p = rem / g.Wo, q = rem - p * g.Wo;
    const int y0 = p * g.stride - g.pad, x0 = q * g.stride - g.pad;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = k0 + j;
      float val = 0.f;
      if (k < g.K) {
        const int rs = k / g.C, c = k - rs * g.C;
        const int r = rs / g.S, s = rs - r * g.S;
        const int yy = y0 + r, xx = x0 + s;
        if (yy >= 0 && yy < g.H && xx >= 0 && xx < g.W) val = __ldg(x + (((long long)n * g.C + c) * g.H + yy) * g.W + xx);
      }
      v[j] = round_out ? tf32_rna(val) : val;
    }
    *reinterpret_cast<float4*>(xcol + m * g.Kp + k0) = make_float4(v[0], v[1], v[2], v[3]);
  }
}

// Same unfold with the k -> (r, s, c) decode done once per block into shared memory (Kp <= 256: the 7x7x3 stem pads to 192, a
// 3x3x3 first conv to 64) and 32-bit index arithmetic: the generic kernel above spends its time in the per-element divisions.
__global__ void __launch_bounds__(256) stem_im2col_lut_kernel(const float* __restrict__ x, float* __restrict__ xcol, ColGeom g, int total, int round_out) {
  __shared__ int tap_off[256];   // c * H * W + r * W + s
  __shared__ int tap_rs[256];    // r | s << 8, -1 for the zero padding of K
  pdl_launch_dependents();
  for (int k = threadIdx.x; k < g.Kp; k += blockDim.x) {
    if (k < g.K) {
      const int rs = k / g.C, c = k - rs * g.C;
      const int r = rs / g.S, sx = rs - r * g.S;
      tap_off[k] = (c * g.H + r) * g.W + sx;
      tap_rs[k] = r | (sx << 8);
    } else {
      tap_off[k] = 0;
      tap_rs[k] = -1;
    }
  }
  __syncthreads();
  pdl_wait();
  const int gran = g.Kp >> 2, HoWo = g.Ho * g.Wo, plane = g.C * g.H * g.W;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int m = i / gran;
    const int k0 = (i - m * gran) << 2;
    const int n = m / HoWo, rem = m - n * HoWo;
    const int p = rem / g.Wo, q = rem - p * g.Wo;
    const int y0 = p * g.stride - g.pad, x0 = q * g.stride - g.pad;
    const float* __restrict__ base = x + (long long)n * plane + y0 * g.W + x0;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int t = tap_rs[k0 + j];
      float val = 0.f;
      if (t >= 0) {
        const int yy = y0 + (t & 255), xx = x0 + (t >> 8);
        if (yy >= 0 && yy < g.H && xx >= 0 && xx < g.W) val = __ldg(base + tap_off[k0 + j]);
      }
      v[j] = round_out ? tf32_rna(val) : val;
    }
    reinterpret_cast<float4*>(xcol)[i] = make_float4(v[0], v[1], v[2], v[3]);
  }
}

// grad[n][c][y][x] = sum over taps (r, s) with (y + pad - r) % stride == 0, (x + pad - s) % stride == 0 of dcol[(n, p, q)][(r, s, c)]
__global__ void __launch_bounds__(256) stem_col2im_kernel(const float* __restrict__ dcol, float* __restrict__ grad, ColGeom g, long long total) {
  pdl_prologue();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int xx = (int)(i % g.W);
    const long long t = i / g.W;
    const int yy = (int)(t % g.H);
    const int n = (int)(t / g.H);
    float acc[4] = {0.f, 0.f, 0.f, 0.f};     // C <= 4
    const int yb = yy + g.pad, xb = xx + g.pad;
    for (int r = yb % g.stride; r < g.R; r += g.stride) {
      const int p = (yb - r) / g.stride;
      if (p < 0 || p >= g.Ho) continue;
      for (int s = xb % g.stride; s < g.S; s += g.stride) {
        const int q = (xb - s) / g.stride;
        if (q < 0 || q >= g.Wo) continue;
        const float* src = dcol + (((long long)n * g.Ho + p) * g.Wo + q) * g.Kp + (r * g.S + s) * g.C;
#pragma unroll
        for (int c = 0; c < 4; ++c)
          if (c < g.C) acc[c] += __ldg(src + c);
      }
    }
    for (int c = 0; c < g.C; ++c) grad[(((long long)n * g.C + c) * g.H + yy) * g.W + xx] = acc[c];
  }
}

// dst[co][k] = k < K ? src[co * K + k] : 0   (forward) ;   dst[co * K + k] = src[co][k]   (inverse)
__global__ void __launch_bounds__(256) stem_pad_rows_kernel(const float* __restrict__ src, float* __restrict__ dst, int Co, int K, int Kp,
                                                            int inverse, int round_out) {
  pdl_prologue();
  const long long total = (long long)Co * (inverse ? K : Kp);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    if (inverse) {
      const int co = (int)(i / K), k = (int)(i - (long long)co * K);
      dst[i] = src[(long long)co * Kp + k];
    } else {
      const int co = (int)(i / Kp), k = (int)(i - (long long)co * Kp);
      const float v = k < K ? src[(long long)co * K + k] : 0.f;
      dst[i] = round_out ? tf32_rna(v) : v;
    }
  }
}

inline int grid_for(long long n) {
  long long b = (n + 255) / 256;
  const long long cap = (long long)kNumSMs * 16;
  return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

}  // namespace

int launch_stem_im2col(const float* x, float* xcol, int N, int C, int H, int W, int Ho, int Wo, int R, int S, int stride, int pad, int Kp,
                       bool round_out, cudaStream_t s) {
  const ColGeom g{N, C, H, W, Ho, Wo, R, S, stride, pad, R * S * C, Kp};
  const long long total = (long long)N * Ho * Wo * (Kp / 4);
  if (Kp <= 256 && R < 256 && S < 256 && total < (1LL << 31) && (long long)N * C * H * W < (1LL << 31)) {
    BRE_KLAUNCH(stem_im2col_lut_kernel, grid_for(total), 256, 0, s, x, xcol, g, (int)total, round_out ? 1 : 0);
    BRE_CHECK_LAUNCH();
    return 0;
  }
  BRE_KLAUNCH(stem_im2col_kernel, grid_for(total), 256, 0, s, x, xcol, g, total, round_out ? 1 : 0);
  BRE_CHECK_LAUNCH();
  return 0;
}
int launch_stem_col2im(const float* dcol, float* grad, int N, int C, int H, int W, int Ho, int Wo, int R, int S, int stride, int pad, int Kp,
                       cudaStream_t s) {
  if (C > 4) { set_error("stem col2im: at most 4 input channels"); return -4; }
  const ColGeom g{N, C, H, W, Ho, Wo, R, S, stride, pad, R * S * C, Kp};
  const long long total = (long long)N * H * W;
  BRE_KLAUNCH(stem_col2im_kernel, grid_for(total), 256, 0, s, dcol, grad, g, total);
  BRE_CHECK_LAUNCH();
  return 0;
}
int launch_stem_pad_rows(const float* src, float* dst, int Co, int K, int Kp, bool inverse, bool round_out, cudaStream_t s) {
  BRE_KLAUNCH(stem_pad_rows_kernel, grid_for((long long)Co * Kp), 256, 0, s, src, dst, Co, K, Kp, inverse ? 1 : 0, round_out ? 1 : 0);
  BRE_CHECK_LAUNCH();
  return 0;
}

}  // namespace bre
