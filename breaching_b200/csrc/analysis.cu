// Reconstruction-quality metrics on the device (SURVEY section 8 f-3): the step right after the hot path.  The reference
// de-normalises both batches, clamps them to [0, 1] and takes per-example mean squared errors (analysis/analysis.py:228-242);
// PSNR = 10 log10(factor^2 / mse) per example follows on the host from those N numbers (analysis/metrics.py:108-130).
#include "../../include/breaching_b200.h"
#include "common.cuh"
#include "augment.cuh"

namespace bre {
namespace {

constexpr int MSE_THREADS = 256;

struct MseArgs {
  const float* rec; const float* ref;
  long long per_example;   // C * HW
  int C; int HW;
  float mean[8], stdv[8];  // per channel (C <= 8), identity when has_norm == 0
  int has_norm, clamp;
};

// grid (B, N): block (b, n) sums its strided share of example n; partials[n * B + b]
__global__ void __launch_bounds__(MSE_THREADS) mse_partial_kernel(MseArgs a, double* __restrict__ partials) {
  __shared__ double scratch[32];
  const int n = blockIdx.y;
  const float* __restrict__ r = a.rec + (long long)n * a.per_example;
  const float* __restrict__ t = a.ref + (long long)n * a.per_example;
  double sum = 0.0;
  for (long long i = (long long)blockIdx.x * MSE_THREADS + threadIdx.x; i < a.per_example; i += (long long)gridDim.x * MSE_THREADS) {
    float u = r[i], v = t[i];
    if (a.has_norm) {
      const int c = (int)(i / a.HW);
      u = fmaf(u, a.stdv[c], a.mean[c]);
      v = fmaf(v, a.stdv[c], a.mean[c]);
    }
    if (a.clamp) { u = fminf(fmaxf(u, 0.f), 1.f); v = fminf(fmaxf(v, 0.f), 1.f); }
    const float d = u - v;
    sum += (double)(d * d);
  }
  const double bs = block_sum(sum, scratch);
  if (threadIdx.x == 0) partials[(long long)n * gridDim.x + blockIdx.x] = bs;
}

// one block per example: fixed-order sum of its B partials -> mean
__global__ void __launch_bounds__(MSE_THREADS) mse_final_kernel(const double* __restrict__ partials, int B, long long per_example,
                                                                double* __restrict__ mse) {
  __shared__ double scratch[32];
  double s = 0.0;
  for (int b = threadIdx.x; b < B; b += MSE_THREADS) s += partials[(long long)blockIdx.x * B + b];
  s = block_sum(s, scratch);
  if (threadIdx.x == 0) mse[blockIdx.x] = s / (double)per_example;
}

}  // namespace
}  // namespace bre

using namespace bre;

extern "C" int bre_image_mse(const float* rec, const float* ref, int32_t N, int32_t C, int32_t HW, const float* mean, const float* stdv,
                             int32_t clamp01, double* mse_host, void* stream) {
  if (!rec || !ref || !mse_host || N <= 0 || C <= 0 || HW <= 0) { set_error("bre_image_mse: bad arguments"); return BRE_ERR_INVALID; }
  if ((mean != nullptr) != (stdv != nullptr)) { set_error("bre_image_mse: mean and std go together"); return BRE_ERR_INVALID; }
  if (mean != nullptr && C > 8) { set_error("bre_image_mse: at most 8 normalised channels"); return BRE_ERR_UNSUPPORTED; }
  cudaStream_t s = (cudaStream_t)stream;
  MseArgs a;
  memset(&a, 0, sizeof(a));
  a.rec = rec; a.ref = ref; a.C = C; a.HW = HW; a.per_example = (long long)C * HW; a.clamp = clamp01 != 0;
  a.has_norm = mean != nullptr;
  for (int c = 0; c < C && a.has_norm; ++c) { a.mean[c] = mean[c]; a.stdv[c] = stdv[c]; }
  long long want = (a.per_example + MSE_THREADS * 8 - 1) / (MSE_THREADS * 8);
  const long long cap = (long long)kNumSMs * 4 / N > 1 ? (long long)kNumSMs * 4 / N : 1;
  const int B = (int)(want < 1 ? 1 : (want > cap ? cap : want));
  double *partials = nullptr, *mse_dev = nullptr;
  BRE_CUDA_CHECK(cudaMallocAsync((void**)&partials, sizeof(double) * (size_t)B * N, s));
  BRE_CUDA_CHECK(cudaMallocAsync((void**)&mse_dev, sizeof(double) * (size_t)N, s));
  mse_partial_kernel<<<dim3(B, N), MSE_THREADS, 0, s>>>(a, partials);
  mse_final_kernel<<<N, MSE_THREADS, 0, s>>>(partials, B, a.per_example, mse_dev);
  cudaError_t err = cudaGetLastError();
  if (err == cudaSuccess) err = cudaMemcpyAsync(mse_host, mse_dev, sizeof(double) * (size_t)N, cudaMemcpyDeviceToHost, s);
  if (err == cudaSuccess) err = cudaStreamSynchronize(s);
  cudaFreeAsync(partials, s);
  cudaFreeAsync(mse_dev, s);
  if (err != cudaSuccess) { set_error(std::string("bre_image_mse failed: ") + cudaGetErrorString(err)); return BRE_ERR_CUDA; }
  return BRE_OK;
}

// ---- bilinear resize of NCHW batches (MultiScaleOptimizationAttacker, multiscale_optimization_attack.py:45-69) ---------------------
// F.interpolate(mode="bilinear", align_corners=False): the index rule bilinear_src (augment.cuh), shared with the RESAMPLE stage.
namespace bre {
namespace {
__global__ void __launch_bounds__(256) resize_bilinear_kernel(const float* __restrict__ src, float* __restrict__ dst, int planes, int Hi, int Wi,
                                                              int Ho, int Wo, float sh, float sw) {
  const long long total = (long long)planes * Ho * Wo;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(i % Wo);
    const long long t = i / Wo;
    const int y = (int)(t % Ho);
    const long long pl = t / Ho;
    int y0, y1, x0, x1; float ly, lx;
    bilinear_src(y, sh, Hi, y0, y1, ly);
    bilinear_src(x, sw, Wi, x0, x1, lx);
    const float* p = src + pl * Hi * Wi;
    const float top = (1.f - lx) * p[(long long)y0 * Wi + x0] + lx * p[(long long)y0 * Wi + x1];
    const float bot = (1.f - lx) * p[(long long)y1 * Wi + x0] + lx * p[(long long)y1 * Wi + x1];
    dst[i] = (1.f - ly) * top + ly * bot;
  }
}
}  // namespace
}  // namespace bre

extern "C" int bre_resize_bilinear(const float* src, float* dst, int32_t N, int32_t C, int32_t Hi, int32_t Wi, int32_t Ho, int32_t Wo,
                                   void* stream) {
  if (!src || !dst || N <= 0 || C <= 0 || Hi <= 0 || Wi <= 0 || Ho <= 0 || Wo <= 0) { set_error("bre_resize_bilinear: bad arguments"); return BRE_ERR_INVALID; }
  const long long total = (long long)N * C * Ho * Wo;
  long long blocks = (total + 255) / 256;
  if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
  resize_bilinear_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(src, dst, N * C, Hi, Wi, Ho, Wo, (float)Hi / (float)Ho, (float)Wi / (float)Wo);
  const cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess) { set_error(std::string("bre_resize_bilinear failed: ") + cudaGetErrorString(err)); return BRE_ERR_CUDA; }
  return BRE_OK;
}
