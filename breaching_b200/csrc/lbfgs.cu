// L-BFGS kernels (see lbfgs.cuh).  Every scalar is fp64 and stays on the device; cross-block sums are fixed-order (per-block
// partials summed in block order), so two launches on the same inputs give the same bits.
#include <algorithm>

#include "lbfgs.cuh"
#include "objective.cuh"

namespace bre {

namespace {

constexpr int kThreads = 256;
constexpr int kMaxSlots = BRE_LBFGS_MAX_HISTORY + 1;
constexpr int kVecMaxBlocks = kNumSMs * 4;

// block-wide sums of N doubles; totals in v[] of thread 0.  scratch: (blockDim / 32) * N doubles
template <int N>
__device__ __forceinline__ void block_sums(double (&v)[N], double* scratch) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int q = 0; q < N; ++q) v[q] = warp_sum(v[q]);
  __syncthreads();   // earlier readers of scratch are done
  if (lane == 0) {
#pragma unroll
    for (int q = 0; q < N; ++q) scratch[warp * N + q] = v[q];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int q = 0; q < N; ++q) {
      double t = 0.0;
      for (int w = 0; w < nw; ++w) t += scratch[w * N + q];
      v[q] = t;
    }
  }
}

__device__ __forceinline__ float block_max(float v, float* scratch) {   // valid in thread 0
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if (lane == 0) scratch[warp] = v;
  __syncthreads();
  if (threadIdx.x == 0)
    for (int w = 0; w < nw; ++w) v = fmaxf(v, scratch[w]);
  return v;
}

// last block of a grid to arrive (after writing its partials); the counter is re-armed for the next launch
__device__ __forceinline__ bool last_block(int* counter, int* s_last) {
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const int prev = atomicAdd(counter, 1);
    *s_last = prev == (int)gridDim.x - 1;
    if (*s_last) *counter = 0;
  }
  __syncthreads();
  if (!*s_last) return false;
  __threadfence();
  return true;
}

__device__ __forceinline__ double* vec_partials(const LbfgsView& v) { return v.partials + (long long)v.gram_blocks * (5 * v.R + 4); }

// 1. the ring pass.  Candidate pair y = g - prev_g, s = t d into the spare slot p; per block (a contiguous chunk of the vector) the
// partial dot products [5 j + q] for each live slot j: s_p.y_j, s_j.y_p, y_p.y_j, s_j.g, y_j.g, and [5 R + q]: s_p.y_p, y_p.y_p,
// s_p.g, y_p.g.
__global__ void __launch_bounds__(kThreads) lbfgs_gram_kernel(LbfgsView v) {
  pdl_prologue();
  __shared__ double scratch[(kThreads / 32) * 5];
  const bre_lbfgs_scalars* st = v.st;
  if (st->total_iters == 0) return;   // the optimiser's first iteration has no previous direction
  const int R = v.R, first = st->first, m = st->count, p = (first + m) % R;
  const long long n = v.n, chunk = (n + gridDim.x - 1) / gridDim.x, lo = blockIdx.x * chunk, hi = min(n, lo + chunk);
  float* sp = v.S + (long long)p * n;
  float* yp = v.Y + (long long)p * n;
  const float t = (float)st->t;
  double* out = v.partials + (long long)blockIdx.x * (5 * R + 4);
  double a[4] = {0.0, 0.0, 0.0, 0.0};
  for (long long i = lo + threadIdx.x; i < hi; i += kThreads) {
    const float gi = v.g[i], y = gi - v.prev_g[i], s = t * v.d[i];
    yp[i] = y;
    sp[i] = s;
    a[0] += (double)s * y; a[1] += (double)y * y; a[2] += (double)s * gi; a[3] += (double)y * gi;
  }
  block_sums(a, scratch);
  if (threadIdx.x == 0)
    for (int q = 0; q < 4; ++q) out[5 * R + q] = a[q];
  for (int k = 0; k < m; ++k) {
    const int j = (first + k) % R;
    const float* Sj = v.S + (long long)j * n;
    const float* Yj = v.Y + (long long)j * n;
    double b[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
    for (long long i = lo + threadIdx.x; i < hi; i += kThreads) {   // sp / yp: written above by this thread
      const float s = sp[i], y = yp[i], gi = v.g[i], sj = Sj[i], yj = Yj[i];
      b[0] += (double)s * yj; b[1] += (double)sj * y; b[2] += (double)y * yj; b[3] += (double)sj * gi; b[4] += (double)yj * gi;
    }
    block_sums(b, scratch);
    if (threadIdx.x == 0)
      for (int q = 0; q < 5; ++q) out[5 * j + q] = b[q];
  }
}

// 2. one CTA: the curvature test and push (Gram row / column of the new pair), then the two-loop recursion on the Gram matrices:
//   alpha_i = rho_i (s_i.q0 - sum_{j newer} alpha_j SY[i][j]),  q0 = -g
//   beta_i  = rho_i (h (y_i.q0 - sum_j alpha_j YY[i][j]) + sum_{k older} (alpha_k - beta_k) SY[k][i])
//   d = h q0 + sum_i (alpha_i - beta_i) s_i - h sum_j alpha_j y_j      (coefficients by age: [k] for s, [R + k] for y)
// which is torch's recursion in exact arithmetic.  Then the step length t of this inner iteration.
__global__ void __launch_bounds__(kThreads) lbfgs_recurrence_kernel(LbfgsView v, const float* lr_table, int n_lr, const Scalars* sc) {
  pdl_prologue();
  __shared__ double dots[5 * kMaxSlots + 4];
  __shared__ double al[kMaxSlots], be[kMaxSlots], z[kMaxSlots], sg[kMaxSlots], yg[kMaxSlots];
  __shared__ int slot[kMaxSlots];
  bre_lbfgs_scalars* st = v.st;
  const int R = v.R, K = 5 * R + 4, tid = threadIdx.x, lane = tid & 31;
  const bool first_iter = st->total_iters == 0;
  int first = st->first, m = st->count, pushed = 0;
  double h = st->h_diag, ys = 0.0;
  double *SY = v.SY(), *YY = v.YY(), *rho = v.rho(), *coef = v.coef();
  if (!first_iter) {
    for (int q = tid; q < K; q += blockDim.x) {
      const bool live = q >= 5 * R || (q / 5 - first + R) % R < m;
      double acc = 0.0;
      if (live)
        for (int b = 0; b < v.gram_blocks; ++b) acc += v.partials[(long long)b * K + q];
      dots[q] = acc;
    }
  }
  __syncthreads();
  if (first_iter) {
    first = 0; m = 0; h = 1.0;
  } else {
    ys = dots[5 * R];
    const double yy = dots[5 * R + 1];
    const int p = (first + m) % R;
    if (ys > v.k.curvature_min) {
      pushed = 1;
      for (int k = tid; k < m; k += blockDim.x) {
        const int j = (first + k) % R;
        SY[p * R + j] = dots[5 * j];
        SY[j * R + p] = dots[5 * j + 1];
        YY[p * R + j] = dots[5 * j + 2];
        YY[j * R + p] = dots[5 * j + 2];
      }
      if (tid == 0) { SY[p * R + p] = ys; YY[p * R + p] = yy; rho[p] = 1.0 / ys; }
      if (m == v.k.history) first = (first + 1) % R;
      else ++m;
      h = ys / yy;
    }
    for (int k = tid; k < m; k += blockDim.x) {
      const int j = (first + k) % R;
      slot[k] = j;
      const bool fresh = pushed && j == p;
      sg[k] = fresh ? dots[5 * R + 2] : dots[5 * j + 3];
      yg[k] = fresh ? dots[5 * R + 3] : dots[5 * j + 4];
    }
  }
  __syncthreads();   // the pushed Gram entries and the per-age tables are visible to the block
  if (tid < 32) {
    for (int k = m - 1; k >= 0; --k) {
      const int i = slot[k];
      double part = 0.0;
      for (int kk = k + 1 + lane; kk < m; kk += 32) part += al[kk] * SY[i * R + slot[kk]];
      part = warp_sum(part);
      if (lane == 0) al[k] = rho[i] * (-sg[k] - part);
      __syncwarp();
    }
  }
  __syncthreads();
  for (int k = tid; k < m; k += blockDim.x) {
    const int i = slot[k];
    double acc = 0.0;
    for (int kk = 0; kk < m; ++kk) acc += al[kk] * YY[i * R + slot[kk]];
    z[k] = acc;
  }
  __syncthreads();
  if (tid < 32) {
    for (int k = 0; k < m; ++k) {
      const int i = slot[k];
      double part = 0.0;
      for (int kk = lane; kk < k; kk += 32) part += (al[kk] - be[kk]) * SY[slot[kk] * R + i];
      part = warp_sum(part);
      if (lane == 0) be[k] = rho[i] * (h * (-yg[k] - z[k]) + part);
      __syncwarp();
    }
  }
  __syncthreads();
  for (int k = tid; k < m; k += blockDim.x) { coef[k] = al[k] - be[k]; coef[R + k] = -h * al[k]; }
  if (tid == 0) {
    st->first = first; st->count = m; st->h_diag = h; st->pushed = pushed; st->ys = ys;
    st->total_iters += 1; st->inner += 1; st->converged = 0;
    st->prev_loss = st->loss;
    if (lr_table != nullptr) {
      const int it = sc->it;
      const double lr = it < n_lr ? (double)lr_table[it] : 0.0;
      st->t = st->total_iters == 1 ? fmin(1.0, 1.0 / st->g_abs_sum) * lr : lr;
    }
  }
}

// 3. d = -h g + sum_k (cs_k S_k + cy_k Y_k) per element (fp64 accumulation), prev_g = g; g.d and max|d| reduced; the last block
// applies torch's `gtd > -tolerance_change` break and sets `eval` = whether the closure is evaluated again.
__global__ void __launch_bounds__(kThreads) lbfgs_dvec_kernel(LbfgsView v, unsigned long long eval, int use_handle) {
  pdl_prologue();
  __shared__ double cs[kMaxSlots], cy[kMaxSlots];
  __shared__ long long off[kMaxSlots];
  __shared__ double scratch[kThreads / 32];
  __shared__ float fscratch[kThreads / 32];
  __shared__ int s_last;
  bre_lbfgs_scalars* st = v.st;
  const int R = v.R, m = st->count, first = st->first;
  const double h = st->h_diag;
  const long long n = v.n;
  for (int k = threadIdx.x; k < m; k += blockDim.x) {
    cs[k] = v.coef()[k]; cy[k] = v.coef()[R + k]; off[k] = (long long)((first + k) % R) * n;
  }
  __syncthreads();
  double gd[1] = {0.0};
  float dmax = 0.f;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float gi = v.g[i];
    double acc = -h * (double)gi;
    for (int k = 0; k < m; ++k) acc += cs[k] * (double)v.S[off[k] + i] + cy[k] * (double)v.Y[off[k] + i];
    const float di = (float)acc;
    v.d[i] = di;
    v.prev_g[i] = gi;
    gd[0] += (double)gi * di;
    dmax = fmaxf(dmax, fabsf(di));
  }
  block_sums(gd, scratch);
  dmax = block_max(dmax, fscratch);
  double* part = vec_partials(v);
  if (threadIdx.x == 0) { part[2 * blockIdx.x] = gd[0]; part[2 * blockIdx.x + 1] = (double)dmax; }
  if (!last_block(v.counter, &s_last)) return;
  if (threadIdx.x != 0) return;
  double gtd = 0.0, dm = 0.0;
  for (int b = 0; b < (int)gridDim.x; ++b) { gtd += __ldcg(part + 2 * b); dm = fmax(dm, __ldcg(part + 2 * b + 1)); }
  st->gtd = gtd;
  st->d_max = dm;
  st->brk = gtd > -v.k.tol_change;
  if (use_handle) cudaGraphSetConditional(eval, !st->brk && st->inner != v.k.max_iter ? 1u : 0u);
}

// 4. x += t d (torch: x.add_(d, alpha=t)) over the segments
__global__ void __launch_bounds__(kThreads) lbfgs_step_kernel(LbfgsView v, LbfgsSegs seg) {
  pdl_prologue();
  if (v.st->brk) return;
  const float t = (float)v.st->t;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < v.n; i += (long long)gridDim.x * blockDim.x) {
    float* x = i < seg.n[0] ? seg.x[0] + i : seg.x[1] + (i - seg.n[0]);
    *x = fmaf(t, v.d[i], *x);
  }
}

// 5. the stop tests after the (possible) re-evaluation, in torch's order -> whether the inner loop goes on
__global__ void lbfgs_tail_kernel(LbfgsView v, unsigned long long loop) {
  pdl_prologue();
  const bre_lbfgs_scalars* st = v.st;
  const bre_lbfgs_consts& k = v.k;
  bool go = !st->brk && !(st->inner == k.max_iter || st->evals >= k.max_eval || st->converged);
  if (go && st->d_max * fabs(st->t) <= k.tol_change) go = false;
  if (go && fabs(st->loss - st->prev_loss) < k.tol_change) go = false;
  cudaGraphSetConditional(loop, go ? 1u : 0u);
}

__global__ void __launch_bounds__(kThreads) lbfgs_closure_tail_kernel(LbfgsView v, int first, Scalars* sc, float task_reg,
                                                                      unsigned long long loop, int use_handle) {
  pdl_prologue();
  __shared__ double scratch[kThreads / 32];
  __shared__ float fscratch[kThreads / 32];
  __shared__ int s_last;
  double gs[1] = {0.0};
  float gm = 0.f;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < v.n; i += (long long)gridDim.x * blockDim.x) {
    const float a = fabsf(v.g[i]);
    gs[0] += (double)a;
    gm = fmaxf(gm, a);
  }
  block_sums(gs, scratch);
  gm = block_max(gm, fscratch);
  double* part = vec_partials(v);
  if (threadIdx.x == 0) { part[2 * blockIdx.x] = gs[0]; part[2 * blockIdx.x + 1] = (double)gm; }
  if (!last_block(v.counter, &s_last)) return;
  if (threadIdx.x != 0) return;
  double sum = 0.0, mx = 0.0;
  for (int b = 0; b < (int)gridDim.x; ++b) { sum += __ldcg(part + 2 * b); mx = fmax(mx, __ldcg(part + 2 * b + 1)); }
  bre_lbfgs_scalars* st = v.st;
  const double loss = total_objective(sc, task_reg);
  st->loss = loss;
  st->g_max = mx;
  st->func_evals += 1;
  if (first) {
    st->first_loss = loss;
    st->first_terms[0] = sc->match; st->first_terms[1] = sc->task_loss; st->first_terms[2] = sc->tv;
    st->first_terms[3] = sc->norm; st->first_terms[4] = sc->di; st->first_terms[5] = sc->feat;
    st->evals = 1;
    st->inner = 0;
    st->brk = 0;
    st->g_abs_sum = sum;
    // torch returns right after the first closure when max|g| <= tolerance_grad; a non-finite loss ends the trial (commit_kernel)
    const bool run = !(mx <= v.k.tol_grad) && isfinite(loss) && !sc->stopped;
    if (use_handle) cudaGraphSetConditional(loop, run ? 1u : 0u);
  } else {
    st->evals += 1;
    st->converged = mx <= v.k.tol_grad;
  }
}

__global__ void __launch_bounds__(kThreads) lbfgs_finish_kernel(LbfgsView v, LbfgsSegs seg, Scalars* sc) {
  pdl_prologue();
  if (sc->stopped) return;
  const bre_lbfgs_scalars* st = v.st;
  const bool improved = (float)st->first_loss < (float)sc->fmin;   // the comparison commit_kernel makes with the same value
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    sc->match = st->first_terms[0]; sc->task_loss = st->first_terms[1]; sc->tv = st->first_terms[2];
    sc->norm = st->first_terms[3]; sc->di = st->first_terms[4]; sc->feat = st->first_terms[5];
  }
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < v.n; i += (long long)gridDim.x * blockDim.x) {
    if (i < seg.n[0]) {
      float x = seg.x[0][i];
      if (seg.boxed) {
        const int c = (int)((i / seg.HW) % seg.C);
        x = fmaxf(fminf(x, __ldg(seg.hi + c)), __ldg(seg.lo + c));
        seg.x[0][i] = x;
      }
      if (improved) seg.best[0][i] = x;
    } else if (improved) {
      const long long j = i - seg.n[0];
      seg.best[1][j] = seg.x[1][j];
    }
  }
}

inline int vec_grid(long long n) {
  const long long b = (n + kThreads - 1) / kThreads;
  return (int)std::max(1LL, std::min(b, (long long)kVecMaxBlocks));
}

}  // namespace

int lbfgs_gram_blocks(long long n) { return (int)std::max(1LL, std::min((n + 2047) / 2048, 2LL * kNumSMs)); }
long long lbfgs_partials_size(long long n, int history) { return (long long)lbfgs_gram_blocks(n) * (5 * (history + 1) + 4) + 2 * kVecMaxBlocks; }

int launch_lbfgs_closure_tail(const LbfgsView& v, bool first, Scalars* sc, float task_reg, unsigned long long loop, int use_handle,
                              cudaStream_t s) {
  BRE_KLAUNCH(lbfgs_closure_tail_kernel, vec_grid(v.n), kThreads, 0, s, v, first ? 1 : 0, sc, task_reg, loop, use_handle);
  BRE_CHECK_LAUNCH();
  return 0;
}

int launch_lbfgs_direction(const LbfgsView& v, const float* lr_table, int n_lr, const Scalars* sc, unsigned long long eval, int use_handle,
                           cudaStream_t s) {
  BRE_KLAUNCH(lbfgs_gram_kernel, v.gram_blocks, kThreads, 0, s, v);
  BRE_KLAUNCH(lbfgs_recurrence_kernel, 1, kThreads, 0, s, v, lr_table, n_lr, sc);
  BRE_KLAUNCH(lbfgs_dvec_kernel, vec_grid(v.n), kThreads, 0, s, v, eval, use_handle);
  BRE_CHECK_LAUNCH();
  return 0;
}

int launch_lbfgs_step(const LbfgsView& v, const LbfgsSegs& seg, cudaStream_t s) {
  BRE_KLAUNCH(lbfgs_step_kernel, vec_grid(v.n), kThreads, 0, s, v, seg);
  BRE_CHECK_LAUNCH();
  return 0;
}

int launch_lbfgs_tail(const LbfgsView& v, unsigned long long loop, cudaStream_t s) {
  BRE_KLAUNCH(lbfgs_tail_kernel, 1, 1, 0, s, v, loop);
  BRE_CHECK_LAUNCH();
  return 0;
}

int launch_lbfgs_finish(const LbfgsView& v, const LbfgsSegs& seg, Scalars* sc, cudaStream_t s) {
  BRE_KLAUNCH(lbfgs_finish_kernel, vec_grid(v.n), kThreads, 0, s, v, seg, sc);
  BRE_CHECK_LAUNCH();
  return 0;
}

}  // namespace bre

extern "C" int bre_lbfgs_direction(float* S, float* Y, double* gram, bre_lbfgs_scalars* state, const float* g, float* prev_g, float* d,
                                   int64_t n, const bre_lbfgs_consts* consts, void* stream) {
  using namespace bre;
  if (!S || !Y || !gram || !state || !g || !prev_g || !d || n <= 0 || !consts || consts->history < 1 ||
      consts->history > BRE_LBFGS_MAX_HISTORY) {
    set_error("bre_lbfgs_direction: bad arguments");
    return BRE_ERR_INVALID;
  }
  cudaStream_t s = (cudaStream_t)stream;
  LbfgsView v;
  v.n = n; v.R = consts->history + 1; v.k = *consts;
  v.S = S; v.Y = Y; v.g = const_cast<float*>(g); v.prev_g = prev_g; v.d = d; v.gram = gram; v.st = state;
  v.gram_blocks = lbfgs_gram_blocks(n);
  BRE_CUDA_CHECK(cudaMalloc((void**)&v.partials, lbfgs_partials_size(n, consts->history) * sizeof(double)));
  int rc = cudaMalloc((void**)&v.counter, sizeof(int)) == cudaSuccess ? 0 : BRE_ERR_CUDA;
  if (rc == 0 && cudaMemsetAsync(v.counter, 0, sizeof(int), s) != cudaSuccess) rc = BRE_ERR_CUDA;
  if (rc == 0) rc = launch_lbfgs_direction(v, nullptr, 0, nullptr, 0, 0, s);
  if (rc == 0 && cudaStreamSynchronize(s) != cudaSuccess) rc = BRE_ERR_CUDA;
  if (rc == BRE_ERR_CUDA) set_error("bre_lbfgs_direction: CUDA call failed");
  cudaFree(v.partials);
  if (v.counter) cudaFree(v.counter);
  return rc;
}
