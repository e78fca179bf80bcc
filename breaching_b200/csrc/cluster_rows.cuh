// Row-wise kernels over very wide rows (the 50 257-token vocabulary of BASELINE config 5): one *thread-block cluster* per row.
//
// With one CTA per row, 32 rows occupy 32 of 132 SMs and every reduction pass walks 200 KB per tensor serially.  Here the CS CTAs of a cluster (grid (rows, 1, CS), cluster along z) each
// take a contiguous segment of the row; the row reductions (max, sum, dot) are combined through distributed shared memory: every
// CTA publishes its partial in its own shared memory, one cluster barrier, then every CTA reads the CS partials with
// ld.shared::cluster in rank order -- the same total in every CTA, deterministic, no global scratch, no atomics.
// A launch without the cluster attribute is a cluster of one CTA: the same code path.
#pragma once
#include "common.cuh"

namespace bre {

constexpr int kRowClusterMax = 8;          // portable cluster size
constexpr int kRowThreads = 256;

__device__ __forceinline__ unsigned cluster_rank() { unsigned r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ unsigned cluster_size() { unsigned r; asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_barrier() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ double ld_cluster_f64(const double* local, unsigned rank) {
  const uint32_t saddr = (uint32_t)__cvta_generic_to_shared(local);
  uint32_t raddr;
  asm("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(raddr) : "r"(saddr), "r"(rank));
  double v;
  asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(v) : "r"(raddr) : "memory");
  return v;
}
__device__ __forceinline__ float ld_cluster_f32(const float* local, unsigned rank) {
  const uint32_t saddr = (uint32_t)__cvta_generic_to_shared(local);
  uint32_t raddr;
  asm("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(raddr) : "r"(saddr), "r"(rank));
  float v;
  asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(raddr) : "memory");
  return v;
}

// The row plan, one rule for the kernels and the host: a row of C elements on a cluster of cs CTAs is cut into segments of
// row_segment_len(C, cs) elements (4-element aligned starts so that float4 access stays possible); a segment of at most
// kSegCache elements per thread is cached in registers (row_seg_fits), a longer one is streamed from memory.
constexpr int kSegCache = 26;
__host__ __device__ __forceinline__ int row_segment_len(int C, int cs) { return (((C + cs - 1) / cs) + 3) & ~3; }
__host__ __device__ __forceinline__ bool row_seg_fits(int C, int cs) { return row_segment_len(C, cs) <= kSegCache * kRowThreads; }

// Segment [c0, c1) of a row of C elements served by this CTA.
__device__ __forceinline__ void row_segment(int C, int& c0, int& c1) {
  const int r = (int)cluster_rank();
  const int per = row_segment_len(C, (int)cluster_size());
  c0 = r * per < C ? r * per : C;
  c1 = c0 + per < C ? c0 + per : C;
}

// Workspace of the cluster-wide reductions of one kernel: one slot per reduction call site (slots are never reused, so one
// barrier per reduction suffices); `cluster_exit()` must be called by every thread before the kernel returns so that no CTA
// retires while a peer may still read its slots.
struct RowReduce {
  double slot[4];
  double scratch[32];
  double bcast;
};
enum RowOp { ROW_SUM = 0, ROW_MAX = 1 };

template <int OP>
__device__ __forceinline__ double row_allreduce(double v, RowReduce& ws, int slot) {
  // block reduction (all threads participate; blockDim.x == kRowThreads)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double u = __shfl_xor_sync(0xffffffffu, v, o);
    v = OP == ROW_SUM ? v + u : (u > v ? u : v);
  }
  __syncthreads();
  if (lane == 0) ws.scratch[warp] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = ws.scratch[0];
    for (int w = 1; w < kRowThreads / 32; ++w) t = OP == ROW_SUM ? t + ws.scratch[w] : (ws.scratch[w] > t ? ws.scratch[w] : t);
    ws.slot[slot] = t;
  }
  cluster_barrier();                       // every thread of every CTA of the cluster: partials published
  if (threadIdx.x == 0) {
    const unsigned n = cluster_size();
    double t = ld_cluster_f64(&ws.slot[slot], 0);
    for (unsigned r = 1; r < n; ++r) {
      const double u = ld_cluster_f64(&ws.slot[slot], r);
      t = OP == ROW_SUM ? t + u : (u > t ? u : t);
    }
    ws.bcast = t;
  }
  __syncthreads();
  const double out = ws.bcast;
  __syncthreads();
  return out;
}
__device__ __forceinline__ void cluster_exit() { cluster_barrier(); }

// ---- register-resident row segments ------------------------------------------------------------------------------------------------
// A CTA's segment of a 50 257-wide row is ~6 300 elements = 25 per thread.  The row kernels make two or three passes over it; with the
// plain loops every pass is a chain of dependent L2 round trips.  When the segment fits, each thread loads its elements once, all loads in flight together, and the passes run out of
// registers.  `seg_fits` depends only on the row width and the cluster size, so it is uniform over the cluster (the barriers inside the
// reductions need every CTA on the same path).
struct SegCache { float v[kSegCache]; };
__device__ __forceinline__ bool seg_fits(int C) { return row_seg_fits(C, (int)cluster_size()); }
__device__ __forceinline__ void seg_load(SegCache& s, const float* __restrict__ row, int c0, int c1, float fill) {
#pragma unroll
  for (int k = 0; k < kSegCache; ++k) {
    const int c = c0 + k * kRowThreads + (int)threadIdx.x;
    s.v[k] = c < c1 ? row[c] : fill;
  }
}

// (max, sum of exp(. - max)) of a row in ONE cluster-wide reduction: every thread brings the pair of its own elements, pairs are merged
// as (M, s exp(m - M) + s' exp(m' - M)) -- lanes, warps and CTAs in a fixed order.  Uses slots `slot` and `slot + 1`.
__device__ __forceinline__ void merge_softmax(float& m, double& s, float m2, double s2) {
  const float M = fmaxf(m, m2);
  s = s * (double)expf(m - M) + s2 * (double)expf(m2 - M);
  m = M;
}
__device__ __forceinline__ void row_allreduce_softmax(float& m, double& s, RowReduce& ws, int slot) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o);
    const double s2 = __shfl_xor_sync(0xffffffffu, s, o);
    merge_softmax(m, s, m2, s2);
  }
  __syncthreads();
  if (lane == 0) { ws.scratch[warp] = (double)m; ws.scratch[8 + warp] = s; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float tm = (float)ws.scratch[0];
    double ts = ws.scratch[8];
    for (int w = 1; w < kRowThreads / 32; ++w) merge_softmax(tm, ts, (float)ws.scratch[w], ws.scratch[8 + w]);
    ws.slot[slot] = (double)tm;
    ws.slot[slot + 1] = ts;
  }
  cluster_barrier();
  if (threadIdx.x == 0) {
    const unsigned n = cluster_size();
    float tm = (float)ld_cluster_f64(&ws.slot[slot], 0);
    double ts = ld_cluster_f64(&ws.slot[slot + 1], 0);
    for (unsigned r = 1; r < n; ++r) merge_softmax(tm, ts, (float)ld_cluster_f64(&ws.slot[slot], r), ld_cluster_f64(&ws.slot[slot + 1], r));
    ws.scratch[16] = (double)tm;
    ws.bcast = ts;
  }
  __syncthreads();
  m = (float)ws.scratch[16];
  s = ws.bcast;
  __syncthreads();
}
// the pair of one thread's cached elements (elements beyond the segment hold -FLT_MAX: exp underflows to 0)
__device__ __forceinline__ void seg_softmax_pair(const SegCache& z, float& m, double& s) {
  m = -3.402823466e+38f;
#pragma unroll
  for (int k = 0; k < kSegCache; ++k) m = fmaxf(m, z.v[k]);
  float acc = 0.f;
  double tot = 0.0;
#pragma unroll
  for (int k = 0; k < kSegCache; ++k) {
    acc += expf(z.v[k] - m);
    if ((k & 3) == 3) { tot += (double)acc; acc = 0.f; }   // short fp32 runs folded into the double total
  }
  s = tot + (double)acc;
}

// cluster size for rows of C elements: enough CTAs that a segment is a few thousand elements, at most the portable 8
inline int row_cluster_size(int C) {
  int cs = 1;
  while (cs < kRowClusterMax && C / (cs * 2) >= 2048) cs *= 2;
  return cs;
}

// launch helper: grid (rows, 1, cs), cluster (1, 1, cs), kRowThreads threads, PDL attribute like every other kernel
template <typename... KArgs, typename... Args>
inline cudaError_t launch_row_kernel(void (*kernel)(KArgs...), int rows, int C, cudaStream_t stream, Args... args) {
  const int cs = row_cluster_size(C);
  return launch_kernel(kernel, dim3(rows, 1, cs), dim3(kRowThreads), 0, stream, cs, args...);
}

}  // namespace bre
