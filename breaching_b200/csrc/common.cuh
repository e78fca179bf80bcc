// Shared helpers for the breaching_b200 sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <string>

namespace bre {

void set_error(const std::string& msg);

#define BRE_CUDA_CHECK(expr)                                                                        \
  do {                                                                                              \
    cudaError_t _err = (expr);                                                                      \
    if (_err != cudaSuccess) {                                                                      \
      ::bre::set_error(std::string(#expr) + " failed: " + cudaGetErrorString(_err) + " at " +       \
                       __FILE__ + ":" + std::to_string(__LINE__));                                  \
      return -2;                                                                                    \
    }                                                                                               \
  } while (0)

#define BRE_CHECK_LAUNCH()                                                                          \
  do {                                                                                              \
    cudaError_t _err = cudaGetLastError();                                                          \
    if (_err != cudaSuccess) {                                                                      \
      ::bre::set_error(std::string("kernel launch failed: ") + cudaGetErrorString(_err) + " at " +  \
                       __FILE__ + ":" + std::to_string(__LINE__));                                  \
      return -2;                                                                                    \
    }                                                                                               \
  } while (0)

constexpr int kNumSMs = 132;  // H100 SXM

// ---- programmatic dependent launch (PDL) -------------------------------------------------------------------
// Every kernel of the iteration is launched with cudaLaunchAttributeProgrammaticStreamSerialization: it may be
// scheduled while its predecessor is still draining, runs its private prologue (barrier init, index
// pre-computation) and then blocks in griddepcontrol.wait until the predecessor grid has completed and flushed its
// memory.  This hides the ~2-3 us launch latency between the ~200 dependent kernels of one iteration; stream capture
// records the edges as programmatic dependencies of the CUDA graph.  Without the launch attribute both instructions
// are no-ops.  BRE_PDL=0 disables it.
bool use_pdl();
// The next launch_kernel() on this thread is issued without the programmatic attribute: it starts only after its predecessor has
// completed and flushed, so every later kernel -- also the part that runs ahead of its own griddepcontrol.wait -- sees the
// predecessor's output (the engine puts this after make_v: weight-side loads of the tangent sweeps may then run ahead).
void serialize_next_launch();
bool consume_serialize_once();
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_prologue() { pdl_launch_dependents(); pdl_wait(); }

template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                 int cluster_z, Args... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attrs[2];
  int n = 0;
  if (cluster_z > 1) {
    attrs[n].id = cudaLaunchAttributeClusterDimension;
    attrs[n].val.clusterDim.x = 1; attrs[n].val.clusterDim.y = 1; attrs[n].val.clusterDim.z = (unsigned)cluster_z;
    ++n;
  }
  if (use_pdl() && !consume_serialize_once()) {
    attrs[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attrs[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  cfg.attrs = attrs;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
#define BRE_KLAUNCH(kernel, grid, block, smem, stream, ...)                                                          \
  do {                                                                                                                 \
    cudaError_t _lerr = ::bre::launch_kernel(kernel, dim3(grid), dim3(block), smem, stream, 1, __VA_ARGS__);           \
    if (_lerr != cudaSuccess) {                                                                                        \
      ::bre::set_error(std::string("kernel launch failed: ") + cudaGetErrorString(_lerr) + " at " + __FILE__ + ":" +  \
                       std::to_string(__LINE__));                                                                      \
      return -2;                                                                                                       \
    }                                                                                                                  \
  } while (0)

static inline int ceil_div(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

// Round-to-nearest onto the TF32 grid (10-bit mantissa, low 13 bits cleared).  the tensor cores read fp32 operands and
// simply ignores the low mantissa bits (truncation, biased towards zero); tensors that feed the tensor-core GEMMs are
// therefore rounded by the kernel that produces them, so that the products are those of cuDNN's TF32 path (cvt.rna).
__device__ __forceinline__ float tf32_rna(float v) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v));
  return __uint_as_float(u);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Block-wide sum of a double; result valid in thread 0.  `scratch` must hold >= 32 doubles.
__device__ __forceinline__ double block_sum(double v, double* scratch) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) scratch[warp] = v;
  __syncthreads();
  const int nwarps = (blockDim.x * blockDim.y + 31) >> 5;
  double r = 0.0;
  if (warp == 0) {
    r = lane < nwarps ? scratch[lane] : 0.0;
    r = warp_sum(r);
  }
  return r;
}

// ---------------------------------------------------------------------------------------------
// Device-resident scalar block shared by all stages of one iteration (no host round trips).
// ---------------------------------------------------------------------------------------------
struct Scalars {
  // matching reduction (objectives.py list reductions), accumulated in double
  double dot, nG, ng, sq, l1w;
  // objective pieces of the current evaluation
  double match, task_loss, tv, norm, di, feat;
  // coefficients of v = c1*g + c2*G + c3*w*sign(G-g)
  float c1, c2, c3, pad0;
  // trial state
  double fmin;           // minimal objective so far (optimization_based_attack.py:103,119-121)
  double last_objective;
  double grad_norm_sq;   // for grad clipping
  int it;                // iterations executed (0-based index of the *next* step)
  int recorded;          // len(stats["Trial_k_Val"])
  int stopped;           // non-finite objective seen (:131-133)
  int trial;             // global index of the running trial: every restart draws its own Langevin noise field
};

}  // namespace bre
