// Hopper TF32 implicit-GEMM back end (sm_90a): the dense contractions of the four sweeps on the tensor cores.  A CTA
// computes a 128 x BN tile with one consumer warpgroup (warps 0-3) holding the fp32 accumulator in registers, fed from a
// TC_STAGES-deep shared-memory ring by a producer warpgroup (warps 4-7) over mbarriers:
//   * FPROP (both operands K-major in memory): wgmma.mma_async m64nBNk8 .tf32 straight from the 128-byte-swizzled ring
//     stages through shared-memory matrix descriptors (two wgmma per 8-wide k step: rows 0-63 and 64-127);
//   * DGRAD / WGRAD: one operand (the weight of dgrad) or both (wgrad) are contiguous along M / N in memory, and wgmma
//     reads tf32 operands K-major only.  Rather than materialise transposed copies, the consumer warps load mma.sync
//     m16n8k8 .tf32 fragments from the swizzled stages with ld.shared (any layout is addressable that way).
// Both consumers leave the accumulator in the same register layout (warp w: rows 16w + [0, 16) and 64 + 16w + [0, 16)),
// so the epilogue is shared.  Launches whose m-tile holds <= 64 GEMM rows run 64-row tiles (rows 0-63 only, BM = 64).
// Operand staging, two producers:
//   * TMA (default wherever the geometry allows): one thread issues cp.async.bulk.tensor loads -- im2col-mode tensor
//     maps for the gathered activation operand (the hardware walks 128 output pixels x 32 channels of one filter tap,
//     zero-filling the padding halo), tiled maps for the weight operand -- which land directly in the 128-byte-swizzled
//     layouts and complete on the stage's mbarrier (expect_tx);
//   * cp.async (strided dgrad, whose "every stride-th tap" gather no tensor map expresses, and BRE_TC_TMA=0): the four
//     producer warps issue 16-byte LDGSTS with precomputed per-row tap masks, completion via cp.async.mbarrier.arrive.
// Split-K runs inside a thread-block cluster (<= 8 CTAs along z) with a deterministic DSMEM reduction.
//
// fp32 storage everywhere; TF32 (10-bit mantissa) multiplies with fp32 accumulation -- the numeric mode cuDNN uses
// for the reference's GPU path by default (SURVEY.md section 8c, torch.backends.cudnn.allow_tf32).
#include <stdlib.h>
#include <string.h>

#include <array>
#include <map>
#include <mutex>
#include <type_traits>

#include <cuda.h>

#include "igemm.cuh"

namespace bre {

namespace {

constexpr int TC_BM = 128;      // tile rows: two wgmma M = 64 halves
constexpr int TC_BK = 32;       // k-block per pipeline stage (4 MMA steps of K = 8)
constexpr int TC_STAGES = 4;       // default ring depth
constexpr int TC_MAX_STAGES = 8;   // deep ring (chosen per launch, TcDims::stage_shift): stage / phase of k-block i are i & (n - 1), (i >> log2 n) & 1
constexpr int TC_THREADS = 128;       // consumer warpgroup (MMA + epilogue) = producer warpgroup size
constexpr int TC_BLOCK = 2 * TC_THREADS;

struct TcDims {
  int M, Nc, K;
  int kblocks_per_src, total_kblocks, kblocks_per_split;
  int stage_shift;   // log2 of the ring depth of this launch (2 or 3)
};

// ---- PTX wrappers -------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t done = 0;
  for (uint32_t spin = 0; !done; ++spin) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
    if (spin > (1u << 24)) __trap();  // never hang the GPU: a lost arrival becomes a launch error
  }
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// ---- wgmma (FPROP) ---------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor of a K-major, 128-byte-swizzled operand: start address and stride byte offset (8-row
// groups, 1024 B) in 16-byte units, leading byte offset unused for swizzled K-major layouts, layout type 1 = SWIZZLE_128B
// in bits 62-63.  The k step of 8 tf32 (32 bytes) inside the 128-byte swizzle atom is a plain start-address offset: the
// swizzle is a function of the absolute address (ring stages are 1024-byte aligned).
__device__ __forceinline__ uint64_t wgmma_desc_k128(uint32_t saddr) {
  return (uint64_t)((saddr >> 4) & 0x3FFF) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from touching accumulator registers across an outstanding wgmma (it does not see the async write)
template <int NR>
__device__ __forceinline__ void fence_regs(float (&d)[NR]) {
#pragma unroll
  for (int i = 0; i < NR; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64 x BN] += A[64 x 8] . B[BN x 8]^T, both from shared memory (K-major), fp32 accumulate
template <int BN>
__device__ __forceinline__ void wgmma_tf32(float (&d)[BN / 2], uint64_t da, uint64_t db);
template <>
__device__ __forceinline__ void wgmma_tf32<64>(float (&d)[32], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(1));
}
template <>
__device__ __forceinline__ void wgmma_tf32<32>(float (&d)[16], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(1));
}

// ---- mma.sync (DGRAD / WGRAD) ------------------------------------------------------------------------------------
// m16n8k8 .tf32: a = A(g, t), A(g + 8, t), A(g, t + 4), A(g + 8, t + 4); b = B(n = g, t), B(g, t + 4);
// d = D(g, 2t), D(g, 2t + 1), D(g + 8, 2t), D(g + 8, 2t + 1)   (g = lane / 4, t = lane % 4)
__device__ __forceinline__ void mma_tf32(float* d, const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// Shared-memory layouts of a [ROWS x 32] fp32 operand tile (ROWS = extent along M or N).  Both are what TMA writes with
// CU_TENSOR_MAP_SWIZZLE_128B into a 1024-byte-aligned box (16-byte granule c of 128-byte smem row r lands at c ^ (r % 8)):
//   K-major (the operand is contiguous along k): one 128-byte smem row per operand row = the whole 32-wide k-block:
//       byte(row, k) = (row/8) * 1024 + (row%8) * 128 + (((k/4) ^ (row%8)) * 16) + (k%4) * 4
//   MN-major (contiguous along M / N; boxes of 32 rows x 32 k, 4 KB each): one 128-byte smem row per k:
//       byte(row, k) = (row/32) * 4096 + k * 128 + ((((row%32)/4) ^ (k%8)) * 16) + (row%4) * 4
// 128-byte swizzle gives coalesced 128-byte global reads and conflict-free 16-byte shared stores for the cp.async producer;
// the mma.sync fragment loads are conflict-free on the K-major layout and 2-way on the MN-major one.
// K-major: granule = 16 bytes (4 k), `g` = granule column 0..7 of the 32-wide k-block
__device__ __forceinline__ uint32_t off_k128(int row, int g) {
  return (uint32_t)((row >> 3) * 1024 + (row & 7) * 128 + ((g ^ (row & 7)) << 4));
}
__device__ __forceinline__ uint32_t off_mn128(int row, int k) {
  return (uint32_t)((row >> 5) * 4096 + k * 128 + ((((row >> 2) & 7) ^ (k & 7)) << 4) + (row & 3) * 4);
}
template <bool MN>
__device__ __forceinline__ uint32_t ld_op(const uint8_t* base, int row, int k) {
  return *reinterpret_cast<const uint32_t*>(base + (MN ? off_mn128(row, k) : off_k128(row, k >> 2) + (k & 3) * 4));
}

// 16-byte asynchronous global -> shared copy; src_bytes = 0 zero-fills the destination (padding, out-of-range taps)
__device__ __forceinline__ void cp_async16(uint32_t dst_smem, const float* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst_smem), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
// arrive on `bar` once all cp.async issued so far by this thread have landed (counts against the barrier's init count)
__device__ __forceinline__ void cp_async_arrive(uint64_t* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, %0;" ::"n"(TC_THREADS) : "memory"); }
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// 16-byte load from the shared memory of CTA `rank` of this cluster at the same offset as local address `saddr`
__device__ __forceinline__ float4 ld_dsmem4(uint32_t saddr, uint32_t rank) {
  uint32_t raddr;
  asm("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(raddr) : "r"(saddr), "r"(rank));
  float4 v;
  // volatile (not reordered across the cluster barriers, themselves volatile) but no memory clobber: a batch of these is issued
  // back to back instead of one round trip at a time
  asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(raddr));
  return v;
}

// ---- TMA -------------------------------------------------------------------------------------------------
struct TcMaps {
  CUtensorMap act[2];  // gathered operand (im2col mode; WGRAD: the activation, B operand)
  CUtensorMap wgt[2];  // plain operand (tiled mode; WGRAD: dout, A operand)
};

// Strided data gradient as per-parity-class stride-1 gathers (specification + CPU check: oracle/strided_dgrad.py,
// tests/test_strided_dgrad_spec.py).  The output pixels split into the stride x stride classes (ey, ex) = ((y + pad) % stride,
// (x + pad) % stride); class pixels are y = stride * iy + y0, and only the taps r = ey + stride * tr reach them:
//     din[y, x] = sum_{tr, ts} dout[iy + cy - tr, ix + cx - ts] . w[ey + stride tr, ex + stride ts]
// i.e. an im2col load over dout with traversal stride 1, lower corner L = c - (T - 1) and filter offset (T - 1) - t.  One launch
// covers all classes (blockIdx.x enumerates (class, m-tile) pairs); a class no tap reaches writes zeros.  Replaces the cp.async
// producer with its 4x zero-filled taps.
constexpr int TC_MAXCLS = 4;   // stride 2
struct ClsPlan {
  int ncls, stride;
  int tile0[TC_MAXCLS + 1];                                  // first m-tile of each class, tile0[ncls] = all tiles
  int Hc[TC_MAXCLS], Wc[TC_MAXCLS], y0[TC_MAXCLS], x0[TC_MAXCLS];   // class pixel grid and its first pixel
  int Ty[TC_MAXCLS], Tx[TC_MAXCLS], Ly[TC_MAXCLS], Lx[TC_MAXCLS], ey[TC_MAXCLS], ex[TC_MAXCLS];
};
struct TcMapsCls {
  CUtensorMap act[2 * TC_MAXCLS];  // [class][source]: im2col maps over dout with the class's corners
  CUtensorMap wgt[2];
};

__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// im2col load of `pixelsPerColumn` pixels x `channelsPerPixel` channels starting at base pixel (w, h, n), filter offset (ow, oh)
__device__ __forceinline__ void tma_im2col(uint32_t dst, const CUtensorMap* tm, uint64_t* bar, int c, int w, int h, int n, int ow, int oh) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c), "r"(w), "r"(h), "r"(n), "h"((uint16_t)ow), "h"((uint16_t)oh)
      : "memory");
}
__device__ __forceinline__ void tma_tile2d(uint32_t dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(dst), "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_tile3d(uint32_t dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
               ::"r"(dst), "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}

// Fused consumer of an FPROP result (GemmEpilogue): NV consecutive channels n..n+NV-1 of GEMM row `row` (element offset
// row = m * Nc).  Mirrors layers.cu bnact_fwd_kernel (kind 1) / bnact_tan_fwd_kernel (kind 2) expression by expression.
template <int NV>
__device__ __forceinline__ void fused_bnact(const GemmEpilogue& e, long long row, int n, float (&v)[NV]) {
  const long long o = row + n;
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    float u = v[j];
    if (e.kind == 1) {
      if (e.has_bn) u = fmaf(u, __ldg(e.scale + n + j), __ldg(e.shift + n + j));
      if (e.res != nullptr) u += e.res[o + j];
      u = e.relu ? fmaxf(u, 0.f) : u;
      v[j] = e.round_out ? tf32_rna(u) : u;
    } else {
      if (e.has_bn) {
        const float xhat = fmaf(e.pre[o + j], __ldg(e.inv + n + j), __ldg(e.nrm + n + j));
        u = fmaf(__ldg(e.scale + n + j), u, fmaf(__ldg(e.v_gamma + n + j), xhat, __ldg(e.v_beta + n + j)));
      }
      if (e.res != nullptr) u += e.res[o + j];
      if (e.relu && !(e.post[o + j] > 0.f)) u = 0.f;
      v[j] = e.round_out ? tf32_rna(u) : u;
    }
  }
}

// Phase timestamps of CTA (0,0,0) (SM clock), compiled in with -DBRE_TC_TRACE (read back with bre_debug_tc_trace).
#ifdef BRE_TC_TRACE
__device__ long long g_tc_trace[16];
#define TC_MARK(i, cond) do { if ((cond) && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) g_tc_trace[i] = clock64(); } while (0)
#else
#define TC_MARK(i, cond) do { } while (0)
#endif

// BM = 64 (launches whose m-tile holds <= 64 GEMM rows): the im2col box, the MMAs and the epilogue cover rows 0-63 only, and the
// stage is half as large (see launch_igemm_tc).
template <int MODE, int BN, bool TMA, bool CLS = false, int BM = TC_BM>
__global__ void __launch_bounds__(TC_BLOCK) igemm_tc_kernel(GemmArgs a, TcDims d, int proxy_fence,
                                                            const __grid_constant__ std::conditional_t<CLS, TcMapsCls, TcMaps> maps, ClsPlan plan) {
  static_assert(!CLS || (MODE == GEMM_DGRAD && TMA), "per-class gathers: strided dgrad with the TMA producer only");
  static_assert(BM == TC_BM || (BM == 64 && TMA && !CLS && MODE != GEMM_WGRAD), "64-row tiles: fprop / stride-1 dgrad on the TMA producer");
  constexpr int MH = BM / 64;   // wgmma M = 64 row halves
  constexpr uint32_t A_BYTES = BM * TC_BK * 4, B_BYTES = BN * TC_BK * 4;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sA = smem;                                  // [STAGES][A_BYTES]
  const int nst = 1 << d.stage_shift, stage_mask = nst - 1;
  uint8_t* sB = smem + nst * A_BYTES;                  // [stages][B_BYTES]
  __shared__ __align__(8) uint64_t bar_full[TC_MAX_STAGES];   // producers -> consumers (TMA transaction bytes / 128 cp.async arrivals)
  __shared__ __align__(8) uint64_t bar_empty[TC_MAX_STAGES];  // consumers -> producers (one arrival per consumer warp)

  TC_MARK(0, threadIdx.x == 0);
  pdl_launch_dependents();   // the successor may start its own prologue; it blocks in its griddepcontrol.wait
  const ConvGeom g = a.g;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int ptid = tid & (TC_THREADS - 1);   // index inside the producer warpgroup (warps 4-7)
  const bool consumer = warp < TC_THREADS / 32;
  const int n0 = blockIdx.y * BN, z = blockIdx.z;
  int m0 = blockIdx.x * BM;
  int kb_begin = z * d.kblocks_per_split;
  int kb_end = min(d.total_kblocks, kb_begin + d.kblocks_per_split);
  const int HoWo = g.Ho * g.Wo, HW = g.H * g.W;
  // per-class view (CLS): which class this CTA serves, its pixel grid / taps, and its own k-block range
  int cls = 0, cHc = 0, cWc = 0, cTy = 0, cTx = 0, cls_kps = 0, Mrows = d.M;
  if (CLS) {
#pragma unroll
    for (int c = 1; c < TC_MAXCLS; ++c)
      if (c < plan.ncls && (int)blockIdx.x >= plan.tile0[c]) cls = c;
    m0 = ((int)blockIdx.x - plan.tile0[cls]) * TC_BM;
    cHc = plan.Hc[cls]; cWc = plan.Wc[cls]; cTy = plan.Ty[cls]; cTx = plan.Tx[cls];
    Mrows = g.N * cHc * cWc;
    cls_kps = cTy * cTx * (g.Co / TC_BK);
    const int total = cls_kps * a.nsrc, per = (total + (int)gridDim.z - 1) / (int)gridDim.z;
    kb_begin = z * per;
    kb_end = min(total, kb_begin + per);
  }

  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < TC_MAX_STAGES; ++s) { mbar_init(&bar_full[s], TMA ? 1 : TC_THREADS); mbar_init(&bar_empty[s], TC_THREADS / 32); }
    fence_barrier_init();
  }
  __syncthreads();
  TC_MARK(1, threadIdx.x == 0);

  // operand majors in shared memory: A is MN-major for WGRAD (dout, contiguous along ko), B for DGRAD and WGRAD
  constexpr bool a_mn = MODE == GEMM_WGRAD;
  constexpr bool b_mn = MODE != GEMM_FPROP;

  // ---- per-thread fixed decode of the gathered (activation) operand ----------------------------------------
  // Loader thread t handles 16-byte granule column (t % 8) of A rows (t / 8) + 16 j, j = 0..7: the eight lanes of a
  // quarter warp read one full 128-byte line of a pixel row (coalesced) and write one swizzled 128-byte smem row
  // (conflict-free).  Everything that depends only on the row is computed once: the element offset of the row's
  // anchor pixel and a bit mask over the R*S filter taps saying which taps land inside the tensor, so that staging a
  // k-block costs one shift/and + one add + one cp.async per row (the loader warps are issue-latency bound otherwise).
  constexpr int A_VEC = TC_BM * TC_BK / 4 / TC_THREADS;  // 16-byte granules per thread per stage: 8
  constexpr int B_VEC = BN * TC_BK / 4 / TC_THREADS;     // 4 (BN = 64)
  const int gcol = ptid & 7, grow = (ptid >> 3) & 15;
  int a_off[A_VEC];                  // element offset of the anchor pixel (+ granule column)
  unsigned long long a_taps[A_VEC];  // bit rs: tap (r, s) of this row reads inside the tensor
  int a_yx[A_VEC];                   // slow path (strided dgrad): packed (y << 16) | x and image index in a_off
  if (!TMA && !consumer && (MODE == GEMM_FPROP || MODE == GEMM_DGRAD)) {
#pragma unroll
    for (int j = 0; j < A_VEC; ++j) {
      const int m = m0 + grow + 16 * j;
      a_off[j] = 0; a_taps[j] = 0ull; a_yx[j] = 0;
      if (m < d.M) {
        if (MODE == GEMM_FPROP) {
          const int img = m / HoWo, rem = m - img * HoWo;
          const int p = rem / g.Wo, q = rem - p * g.Wo;
          const int y0 = p * g.stride - g.pad, x0 = q * g.stride - g.pad;
          a_off[j] = (int)(img * a.x_sN) + (y0 * g.W + x0) * a.x_sP + gcol * 4;
          for (int r = 0; r < g.R; ++r)
            for (int s2 = 0; s2 < g.S; ++s2)
              if (y0 + r >= 0 && y0 + r < g.H && x0 + s2 >= 0 && x0 + s2 < g.W) a_taps[j] |= 1ull << (r * g.S + s2);
        } else {
          const int img = m / HW, rem = m - img * HW;
          const int y = rem / g.W, x = rem - y * g.W;
          // p = (y + pad - r) / stride must be exact.  With yb = y + pad = stride * py + ey the valid taps are r = ey + stride * t
          // and p = py - t: anchor the row at (py, qx) and keep (ey, ex) so that a tap costs two shifts/divides and an fma.
          const int yb = y + g.pad, xb = x + g.pad;
          const int py = yb / g.stride, qx = xb / g.stride;
          const int ey = yb - py * g.stride, ex = xb - qx * g.stride;
          a_off[j] = ((img * g.Ho + py) * g.Wo + qx) * g.Co + gcol * 4;
          a_yx[j] = (ey << 16) | ex;
          for (int r = ey, pp = py; r < g.R; r += g.stride, --pp)
            for (int s2 = ex, qq = qx; s2 < g.S; s2 += g.stride, --qq)
              if (pp >= 0 && pp < g.Ho && qq >= 0 && qq < g.Wo) a_taps[j] |= 1ull << (r * g.S + s2);
        }
      }
    }
  }
  // running decode of the k-block sequence this CTA walks: (source, filter tap, first channel) advance incrementally
  int it_src, it_rs, it_c0;
  {
    const int kch = (MODE == GEMM_DGRAD) ? g.Co : g.Ci;
    it_src = kb_begin / d.kblocks_per_src;
    const int kbase = (kb_begin - it_src * d.kblocks_per_src) * TC_BK;
    it_rs = (MODE == GEMM_WGRAD) ? 0 : kbase / kch;
    it_c0 = (MODE == GEMM_WGRAD) ? kbase : kbase - it_rs * kch;
  }

  const int nkb = kb_end > kb_begin ? kb_end - kb_begin : 0;  // a trailing split may be empty: it contributes zeros
  // TMA producer (one thread): the CTA's first GEMM row fixes the base pixel of every im2col load; per k-block only the
  // filter-tap offsets and the channel coordinate change.
  int base_n = 0, base_h = 0, base_w = 0;
  if (CLS) {
    const int per = cHc * cWc;
    base_n = m0 / per;
    const int rem = m0 - base_n * per;
    const int iy0 = rem / cWc, ix0 = rem - iy0 * cWc;
    base_h = iy0 + plan.Ly[cls]; base_w = ix0 + plan.Lx[cls];
  } else if (TMA && MODE != GEMM_WGRAD) {
    const int per = (MODE == GEMM_FPROP) ? HoWo : HW, wid = (MODE == GEMM_FPROP) ? g.Wo : g.W;
    base_n = m0 / per;
    const int rem = m0 - base_n * per;
    const int p0 = rem / wid, q0 = rem - p0 * wid;
    if (MODE == GEMM_FPROP) { base_h = p0 * g.stride - g.pad; base_w = q0 * g.stride - g.pad; }
    else { base_h = p0 + g.pad - (g.R - 1); base_w = q0 + g.pad - (g.S - 1); }   // stride-1 dgrad: flipped taps
  }
  // Running decode of the producer's k-block sequence.  The producer lane is a single thread on the critical path of the
  // whole CTA: no divisions inside the loop (an integer division costs it ~100 cycles), everything advances incrementally.
  struct KbState { int src, rs, r, s, c0, img, p, q; };
  auto kb_init = [&](int kb) {
    KbState st;
    const int kch = (MODE == GEMM_DGRAD) ? g.Co : g.Ci;
    if (CLS) {   // k = (source, class tap (tr, ts), channel); st.r / st.s hold the class-tap indices, st.rs the weight's filter cell
      st.src = cls_kps > 0 ? kb / cls_kps : 0;
      const int rem = kb - st.src * cls_kps, cpb = g.Co / TC_BK;
      const int tap = rem / cpb;
      st.c0 = (rem - tap * cpb) * TC_BK;
      st.r = cTx > 0 ? tap / cTx : 0; st.s = tap - st.r * cTx;
      st.rs = (plan.ey[cls] + plan.stride * st.r) * g.S + plan.ex[cls] + plan.stride * st.s;
      st.img = st.p = st.q = 0;
      return st;
    }
    st.src = kb / d.kblocks_per_src;
    const int kbase = (kb - st.src * d.kblocks_per_src) * TC_BK;
    if (MODE == GEMM_WGRAD) {
      st.rs = st.r = st.s = 0; st.c0 = kbase;
      st.img = kbase / HoWo;
      const int rem = kbase - st.img * HoWo;
      st.p = rem / g.Wo; st.q = rem - st.p * g.Wo;
    } else {
      st.rs = kbase / kch; st.c0 = kbase - st.rs * kch;
      st.r = st.rs / g.S; st.s = st.rs - st.r * g.S;
      st.img = st.p = st.q = 0;
    }
    return st;
  };
  auto kb_advance = [&](KbState& st) {
    const int kch = (MODE == GEMM_DGRAD) ? g.Co : g.Ci;
    st.c0 += TC_BK;
    if (CLS) {
      if (st.c0 >= kch) {
        st.c0 = 0;
        if (++st.s == cTx) { st.s = 0; if (++st.r == cTy) { st.r = 0; ++st.src; } }
        st.rs = (plan.ey[cls] + plan.stride * st.r) * g.S + plan.ex[cls] + plan.stride * st.s;
      }
      return;
    }
    if (MODE == GEMM_WGRAD) {
      if (st.c0 >= d.kblocks_per_src * TC_BK) { st.c0 = 0; ++st.src; st.img = st.p = st.q = 0; }
      else {
        st.q += TC_BK;
        while (st.q >= g.Wo) { st.q -= g.Wo; if (++st.p == g.Ho) { st.p = 0; ++st.img; } }
      }
    } else if (st.c0 >= kch) {
      st.c0 = 0; ++st.rs;
      if (++st.s == g.S) { st.s = 0; if (++st.r == g.R) { st.r = 0; st.rs = 0; ++st.src; } }
    }
  };
  // WGRAD: the filter tap / channel of the CTA's B columns are fixed
  int wg_c[BN / 32], wg_r[BN / 32], wg_s[BN / 32];
  if (TMA && MODE == GEMM_WGRAD) {
#pragma unroll
    for (int h = 0; h < BN / 32; ++h) {
      const int n = n0 + 32 * h;
      const int rs = n / g.Ci;
      wg_c[h] = n - rs * g.Ci; wg_r[h] = rs / g.S; wg_s[h] = rs - wg_r[h] * g.S;
    }
  }
  // One k-block = the weight-side loads and the activation-side loads on the same stage barrier.  They are separate calls because
  // the weight side of the first ring stages is issued *before* griddepcontrol.wait (below): weights do not depend on the
  // predecessor kernel, so their HBM / L2 round trip overlaps the predecessor's tail.
  auto issue_wgt_tma = [&](int stage, const KbState& st) {
    uint64_t* bar = &bar_full[stage];
    const uint32_t pb = smem_u32(sB) + stage * B_BYTES;
    if (MODE == GEMM_FPROP) {
      tma_tile2d(pb, &maps.wgt[st.src], bar, st.rs * g.Ci + st.c0, n0);
    } else if (MODE == GEMM_DGRAD) {
#pragma unroll
      for (int h = 0; h < BN / 32; ++h) tma_tile3d(pb + h * 4096, &maps.wgt[st.src], bar, n0 + 32 * h, st.rs, st.c0);
    } else {
      const uint32_t pa = smem_u32(sA) + stage * A_BYTES;
#pragma unroll
      for (int h = 0; h < TC_BM / 32; ++h) tma_tile2d(pa + h * 4096, &maps.wgt[st.src], bar, m0 + 32 * h, st.c0);   // k = pixel
    }
  };
  auto issue_act_tma = [&](int stage, const KbState& st) {
    uint64_t* bar = &bar_full[stage];
    const uint32_t pa = smem_u32(sA) + stage * A_BYTES, pb = smem_u32(sB) + stage * B_BYTES;
    if (MODE == GEMM_FPROP) {
      tma_im2col(pa, &maps.act[st.src], bar, st.c0, base_w, base_h, base_n, st.s, st.r);
    } else if (MODE == GEMM_DGRAD) {
      if (CLS) tma_im2col(pa, &maps.act[2 * cls + st.src], bar, st.c0, base_w, base_h, base_n, cTx - 1 - st.s, cTy - 1 - st.r);
      else tma_im2col(pa, &maps.act[st.src], bar, st.c0, base_w, base_h, base_n, g.S - 1 - st.s, g.R - 1 - st.r);
    } else {
#pragma unroll
      for (int h = 0; h < BN / 32; ++h)
        tma_im2col(pb + h * 4096, &maps.act[st.src], bar, wg_c[h], st.q * g.stride - g.pad, st.p * g.stride - g.pad, st.img, wg_s[h], wg_r[h]);
    }
  };

  if (TMA && tid == 0 && (proxy_fence & 2)) {
    for (int sidx = 0; sidx < a.nsrc; ++sidx) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&maps.act[(CLS ? 2 * cls : 0) + sidx])) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&maps.wgt[sidx])) : "memory");
    }
  }
  // `nprod` producer lanes (lane 0 of producer warps 4..4+nprod-1, default 2), k-blocks dealt round-robin: a
  // cp.async.bulk.tensor costs its issuing thread on the order of 100 cycles, so the six loads per k-block of the wgrad form
  // want two issuers
  const int nprod = (proxy_fence >> 2) & 7;
  const int pw = warp - TC_THREADS / 32;   // producer warp index
  const bool producer = TMA && !consumer && lane == 0 && pw < nprod && pw < nkb;
  KbState pst;
  memset(&pst, 0, sizeof(pst));
  uint32_t pre_wgt = 0;   // ring stages whose weight loads are already in flight when the wait below returns
  if (producer) {
    pst = kb_init(kb_begin + pw);
    if (MODE != GEMM_WGRAD && a.wgt_static != 0) {
      KbState st = pst;
      for (int i = pw; i < nkb && i < nst; i += nprod) {
        if ((a.wgt_static >> st.src) & 1) {
          mbar_expect_tx(&bar_full[i], A_BYTES + B_BYTES);
          issue_wgt_tma(i, st);
          pre_wgt |= 1u << i;
        }
        for (int u = 0; u < nprod; ++u) kb_advance(st);
      }
    }
  }

  // Everything above touched only kernel parameters, shared memory and weights the caller declared constant across the
  // predecessor (GemmArgs::wgt_static); from here on global memory written by the predecessor kernel is read.
  pdl_wait();
  TC_MARK(2, threadIdx.x == 0);

  // Stage one k-block: cp.async (LDGSTS, 16 B, zero-fill for padding / out-of-range taps) straight from global memory
  // into the swizzled operand layouts -- no register staging, so up to TC_STAGES k-blocks of loads stay in flight.
  auto issue_block = [&](int stage) {
    const int src = it_src;
    const int kch = (MODE == GEMM_DGRAD) ? g.Co : g.Ci;
    const int kbase = (MODE == GEMM_WGRAD) ? it_c0 : it_rs * kch + it_c0;
    const float* __restrict__ act = a.act[src];
    const float* __restrict__ wgt = a.wgt[src];
    const uint32_t pa = smem_u32(sA + stage * A_BYTES), pb = smem_u32(sB + stage * B_BYTES);
    if (MODE == GEMM_FPROP) {
      // A(m, k) = in[img, y0 + r, x0 + s, c], k = (r, s, c); the 32-wide k-block lies inside one (r, s) cell (Ci % 32 == 0)
      const int r = it_rs / g.S, s = it_rs - r * g.S;
      const int tapoff = (r * g.W + s) * a.x_sP + it_c0;
#pragma unroll
      for (int j = 0; j < A_VEC; ++j) {
        const bool ok = (a_taps[j] >> it_rs) & 1ull;
        cp_async16(pa + off_k128(grow + 16 * j, gcol), ok ? act + (a_off[j] + tapoff) : act, ok ? 16u : 0u);
      }
      // B(n, k) = W[n][k] (row-major [Co][K])
      const float* q = wgt + (long long)(n0 + grow) * d.K + kbase + gcol * 4;
#pragma unroll
      for (int j = 0; j < B_VEC; ++j) cp_async16(pb + off_k128(grow + 16 * j, gcol), q + (long long)(16 * j) * d.K, 16u);
    } else if (MODE == GEMM_DGRAD) {
      // A(m, k) = dout[img, (y + pad - r)/stride, (x + pad - s)/stride, ko], k = (r, s, ko)   (Co % 32 == 0)
      const int rs = it_rs, k0 = it_c0;
      const int r = rs / g.S, s = rs - r * g.S;
      if (g.stride == 1) {
        const int tapoff = k0 - (r * g.Wo + s) * g.Co;
#pragma unroll
        for (int j = 0; j < A_VEC; ++j) {
          const bool ok = (a_taps[j] >> rs) & 1ull;
          cp_async16(pa + off_k128(grow + 16 * j, gcol), ok ? act + (a_off[j] + tapoff) : act, ok ? 16u : 0u);
        }
      } else {
        const bool st2 = g.stride == 2;
#pragma unroll
        for (int j = 0; j < A_VEC; ++j) {
          const bool ok = (a_taps[j] >> rs) & 1ull;
          const int dr = r - (a_yx[j] >> 16), ds = s - (a_yx[j] & 0xffff);
          const int tr = st2 ? dr >> 1 : dr / g.stride, ts = st2 ? ds >> 1 : ds / g.stride;
          cp_async16(pa + off_k128(grow + 16 * j, gcol), ok ? act + (a_off[j] + k0 - (tr * g.Wo + ts) * g.Co) : act, ok ? 16u : 0u);
        }
      }
      // B(n = ci, k) = W[ko][r][s][ci]: contiguous along n -> MN-major.  lanes along n (16 granules = 64 ci), 8 k per pass
      const int n4 = ptid & 15, kk = ptid >> 4;
#pragma unroll
      for (int j = 0; j < B_VEC; ++j) {
        const int k = kk + 8 * j;
        const float* gb = wgt + ((long long)(k0 + k) * (g.R * g.S) + rs) * g.Ci + n0 + n4 * 4;
        cp_async16(pb + off_mn128(4 * n4, k), gb, 16u);
      }
    } else {
      // WGRAD: k = pixel.  A(m = ko, k) = dout[pixel][ko] (MN-major): lanes along m (32 granules = 128 ko), 4 k per pass
      {
        const int m4 = ptid & 31, kk = ptid >> 5;
#pragma unroll
        for (int j = 0; j < A_VEC; ++j) {
          const int k = kk + 4 * j;
          const int pix = kbase + k;
          const bool kok = pix < d.K;
          const bool mok = kok && (m0 + m4 * 4 < d.M);
          const float* ga = mok ? wgt + (long long)pix * g.Co + m0 + m4 * 4 : wgt;
          cp_async16(pa + off_mn128(4 * m4, k), ga, mok ? 16u : 0u);
        }
      }
      // B(n = (r, s, c), k) = in[img, p*stride - pad + r, q*stride - pad + s, c] (MN-major, Ci % 4 == 0)
      {
        const int n4 = ptid & 15, kk = ptid >> 4;
        const int n = n0 + n4 * 4;
        const int rs = n / g.Ci, c = n - rs * g.Ci;
        const int r = rs / g.S, s = rs - r * g.S;
#pragma unroll
        for (int j = 0; j < B_VEC; ++j) {
          const int k = kk + 8 * j;
          const int pix = kbase + k;
          bool ok = pix < d.K;
          const float* gb = act;
          if (ok) {
            const int img = pix / HoWo, rem = pix - img * HoWo;
            const int p = rem / g.Wo, q = rem - p * g.Wo;
            const int h = p * g.stride - g.pad + r, w = q * g.stride - g.pad + s;
            ok = h >= 0 && h < g.H && w >= 0 && w < g.W;
            if (ok) gb = act + img * a.x_sN + (long long)(h * g.W + w) * a.x_sP + c;
          }
          cp_async16(pb + off_mn128(4 * n4, k), gb, ok ? 16u : 0u);
        }
      }
    }
    // advance the running (source, tap, channel) decode to the next k-block
    it_c0 += TC_BK;
    if (MODE == GEMM_WGRAD) {
      if (it_c0 >= d.kblocks_per_src * TC_BK) { it_c0 = 0; ++it_src; }
    } else if (it_c0 >= kch) {
      it_c0 = 0;
      if (++it_rs == g.R * g.S) { it_rs = 0; ++it_src; }
    }
  };

  // ---- main loop, warp-specialised: the producer warpgroup streams k-blocks into the TC_STAGES-deep ring (TMA: one or two
  //      issuing lanes, completion by transaction bytes; cp.async: all 128 threads, cp.async.mbarrier.arrive), the consumer
  //      warpgroup waits for "full", runs the MMAs of the k-block and signals "empty" (one arrival per warp) once the stage
  //      has been read.  No CTA-wide barrier inside the loop.
  // acc[h][4 j + q] = tile element (64 h + 16 w + g + 8 (q >> 1), 8 j + 2 t + (q & 1)), w = warp, g = lane / 4, t = lane % 4
  // (the wgmma m64nN accumulator fragment of half h, and the union of the mma.sync m16n8 fragments of the same elements)
  float acc[MH][BN / 2];
#pragma unroll
  for (int h = 0; h < MH; ++h)
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[h][i] = 0.f;
  const int gq = lane >> 2, tq = lane & 3;
  if (consumer) {
    for (int i = 0; i < nkb; ++i) {
      const int stage = i & stage_mask;
      mbar_wait(&bar_full[stage], (uint32_t)((i >> d.stage_shift) & 1));
      TC_MARK(4, i == 0 && tid == 0);
      if constexpr (MODE == GEMM_FPROP) {
        // cp.async stores are generic-proxy writes and wgmma reads through the async proxy (TMA writes need no fence)
        if (!TMA || (proxy_fence & 1)) fence_proxy_async();
        const uint32_t sa = smem_u32(sA) + stage * A_BYTES, sb = smem_u32(sB) + stage * B_BYTES;
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < TC_BK / 8; ++j) {
          const uint64_t db = wgmma_desc_k128(sb + 32 * j);
#pragma unroll
          for (int h = 0; h < MH; ++h) wgmma_tf32<BN>(acc[h], wgmma_desc_k128(sa + h * 64 * 128 + 32 * j), db);
        }
        wgmma_commit();
        // this k-block's MMAs stay in flight while the next stage is waited for; the previous stage is free once its group is
        wgmma_wait<1>();
#pragma unroll
        for (int h = 0; h < MH; ++h) fence_regs(acc[h]);
        __syncwarp();
        if (i > 0 && lane == 0) mbar_arrive(&bar_empty[(i - 1) & stage_mask]);
      } else {
        const uint8_t* pa = sA + stage * A_BYTES;
        const uint8_t* pb = sB + stage * B_BYTES;
#pragma unroll
        for (int j = 0; j < TC_BK / 8; ++j) {
          const int k0 = 8 * j + tq;
          uint32_t af[MH][4];
#pragma unroll
          for (int h = 0; h < MH; ++h) {
            const int r = 64 * h + 16 * warp + gq;
            af[h][0] = ld_op<a_mn>(pa, r, k0);
            af[h][1] = ld_op<a_mn>(pa, r + 8, k0);
            af[h][2] = ld_op<a_mn>(pa, r, k0 + 4);
            af[h][3] = ld_op<a_mn>(pa, r + 8, k0 + 4);
          }
#pragma unroll
          for (int jn = 0; jn < BN / 8; ++jn) {
            const uint32_t b0 = ld_op<b_mn>(pb, 8 * jn + gq, k0), b1 = ld_op<b_mn>(pb, 8 * jn + gq, k0 + 4);
#pragma unroll
            for (int h = 0; h < MH; ++h) mma_tf32(&acc[h][4 * jn], af[h], b0, b1);
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&bar_empty[stage]);
      }
    }
    if constexpr (MODE == GEMM_FPROP) {
      wgmma_wait<0>();
#pragma unroll
      for (int h = 0; h < MH; ++h) fence_regs(acc[h]);
    }
    TC_MARK(5, tid == 0);
  } else {
    if (TMA) {
      if (producer) {
        KbState st = pst;
        for (int i = pw; i < nkb; i += nprod) {
          const int stage = i & stage_mask;
          if (i >= nst) mbar_wait(&bar_empty[stage], (uint32_t)(((i >> d.stage_shift) - 1) & 1));
          if (i >= nst || !((pre_wgt >> i) & 1u)) {
            mbar_expect_tx(&bar_full[stage], A_BYTES + B_BYTES);
            issue_wgt_tma(stage, st);
          }
          issue_act_tma(stage, st);
          TC_MARK(3, i == (nkb < nst ? nkb : nst) - 1);
          for (int u = 0; u < nprod; ++u) kb_advance(st);
        }
      }
      __syncwarp();
    } else {
      for (int i = 0; i < nkb; ++i) {
        const int stage = i & stage_mask;
        if (i >= nst) mbar_wait(&bar_empty[stage], (uint32_t)(((i >> d.stage_shift) - 1) & 1));
        issue_block(stage);
        cp_async_arrive(&bar_full[stage]);
      }
      cp_async_wait<0>();
    }
  }

  // ---- epilogue (consumer warpgroup): accumulator registers -> global memory, or -> this CTA's split-K partial ----------
  const int splits = gridDim.z;
  auto out_row = [&](int mm, long long& row, int& cs) {
    if (CLS) {   // class pixel (img, iy, ix) -> input pixel (y0 + stride * iy, x0 + stride * ix)
      const int per = cHc * cWc;
      const int img = mm / per, rem = mm - img * per;
      const int iy = rem / cWc, ix = rem - iy * cWc;
      row = img * a.x_sN + (long long)((plan.y0[cls] + plan.stride * iy) * g.W + plan.x0[cls] + plan.stride * ix) * a.x_sP;
      cs = a.x_sC;
    } else if (MODE == GEMM_DGRAD) {
      const int img = mm / HW;
      row = img * a.x_sN + (long long)(mm - img * HW) * a.x_sP;
      cs = a.x_sC;
    } else {
      row = (long long)mm * d.Nc;
      cs = 1;
    }
  };
  if (consumer && splits == 1) {
    // (a class no filter tap reaches has nkb = 0 and writes the zero accumulator)
#pragma unroll
    for (int h = 0; h < MH; ++h) {
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const int mm = m0 + 64 * h + 16 * warp + gq + 8 * hr;
        if (mm >= Mrows) continue;
        long long row;
        int cs;
        out_row(mm, row, cs);
#pragma unroll
        for (int jn = 0; jn < BN / 8; ++jn) {
          const int n = n0 + 8 * jn + 2 * tq;
          float v[2] = {acc[h][4 * jn + 2 * hr], acc[h][4 * jn + 2 * hr + 1]};
          if (MODE == GEMM_FPROP && a.bias != nullptr) {
            v[0] += __ldg(a.bias + n);
            v[1] += __ldg(a.bias + n + 1);
          }
          float* op = a.out + row + (long long)n * cs;
          if (MODE == GEMM_FPROP && a.epi.kind != 0) {
            if (a.out != nullptr) *reinterpret_cast<float2*>(op) = make_float2(v[0], v[1]);
            fused_bnact<2>(a.epi, row, n, v);
            *reinterpret_cast<float2*>(a.epi.out2 + row + n) = make_float2(v[0], v[1]);
          } else if (cs == 1) {
            float2 t2 = make_float2(v[0], v[1]);
            if (a.accumulate) {
              const float2 o = *reinterpret_cast<const float2*>(op);
              t2.x += o.x; t2.y += o.y;
            }
            *reinterpret_cast<float2*>(op) = t2;
          } else {
#pragma unroll
            for (int j = 0; j < 2; ++j) {
              float* q = op + (long long)j * cs;
              *q = a.accumulate ? *q + v[j] : v[j];
            }
          }
        }
      }
    }
  } else if (consumer) {
    // split-K inside a thread-block cluster (cluster = the `splits` CTAs of one output tile along z): every CTA parks
    // its partial accumulator tile in its own shared memory (the operand ring is idle once all consumer warps are done
    // reading it), one cluster barrier, then CTA `z` sums rows [z*128/S, (z+1)*128/S) of all S partials straight out of
    // the peers' shared memory (DSMEM, ld.shared::cluster) in fixed rank order -- deterministic, no global workspace, no
    // atomics, no "last CTA" tail.
    consumer_sync();
    float* part = reinterpret_cast<float*>(sA);  // [BM rows][BN] fp32, 16-byte chunks XOR-swizzled by (row & 15)
#pragma unroll
    for (int h = 0; h < MH; ++h) {
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const int r = 64 * h + 16 * warp + gq + 8 * hr;
#pragma unroll
        for (int jn = 0; jn < BN / 8; ++jn) {
          const int c = 8 * jn + 2 * tq;
          const int chunk = (c >> 2) ^ (r & (BN / 4 - 1) & 15);
          *reinterpret_cast<float2*>(part + r * BN + chunk * 4 + (c & 3)) = make_float2(acc[h][4 * jn + 2 * hr], acc[h][4 * jn + 2 * hr + 1]);
        }
      }
    }
  }
  if (splits > 1) {
    TC_MARK(7, tid == 0);
    cluster_sync_all();   // every thread of every CTA in the cluster (partials visible cluster-wide)
    TC_MARK(8, tid == 0);
    if (consumer) {
      // Every thread owns BN/(4 S) float4 slots of this CTA's row slice and needs the S peers' copies of each: BN/4 = 16
      // remote 16-byte loads per thread whatever S is.  All of them are issued before the first is consumed (a DSMEM round
      // trip is ~0.5 us; one slot at a time made this phase 2.2 us), then summed in fixed rank order.
      // A slice with fewer slots than threads (BM = 64, S = 8, BN = 32: 64 slots) leaves the surplus threads idle.
      auto reduce_rows = [&](auto s_tag) {
        constexpr int S = decltype(s_tag)::value;
        constexpr int C4 = BN / 4, NSLOT = (BM / S) * C4, SLOTS = NSLOT / TC_THREADS > 0 ? NSLOT / TC_THREADS : 1;
        const uint32_t part_s = smem_u32(sA);
        float4 t[SLOTS][S];
        int rr[SLOTS], cc[SLOTS];
#pragma unroll
        for (int sl = 0; sl < SLOTS; ++sl) {
          const int slot = tid + sl * TC_THREADS;
          rr[sl] = z * (BM / S) + slot / C4;
          cc[sl] = slot % C4;
          if (NSLOT < TC_THREADS && slot >= NSLOT) continue;
          const uint32_t local = part_s + (uint32_t)(rr[sl] * BN + ((cc[sl] ^ (rr[sl] & (BN / 4 - 1) & 15)) << 2)) * 4u;
#pragma unroll
          for (int q = 0; q < S; ++q) t[sl][q] = ld_dsmem4(local, (uint32_t)q);
        }
#pragma unroll
        for (int sl = 0; sl < SLOTS; ++sl) {
          const int r = rr[sl], c4 = cc[sl];
          if ((NSLOT < TC_THREADS && tid + sl * TC_THREADS >= NSLOT) || m0 + r >= Mrows) continue;
          float4 acc4 = t[sl][0];
#pragma unroll
          for (int q = 1; q < S; ++q) { acc4.x += t[sl][q].x; acc4.y += t[sl][q].y; acc4.z += t[sl][q].z; acc4.w += t[sl][q].w; }
          const int n = n0 + c4 * 4;
          if (MODE == GEMM_FPROP && a.bias != nullptr) {
            acc4.x += __ldg(a.bias + n); acc4.y += __ldg(a.bias + n + 1); acc4.z += __ldg(a.bias + n + 2); acc4.w += __ldg(a.bias + n + 3);
          }
          long long row;
          int cs;
          out_row(m0 + r, row, cs);
          float* op = a.out + row + (long long)n * cs;
          if (MODE == GEMM_FPROP && a.epi.kind != 0) {
            if (a.out != nullptr) *reinterpret_cast<float4*>(op) = acc4;
            float vv[4] = {acc4.x, acc4.y, acc4.z, acc4.w};
            fused_bnact<4>(a.epi, row, n, vv);
            *reinterpret_cast<float4*>(a.epi.out2 + row + n) = make_float4(vv[0], vv[1], vv[2], vv[3]);
          } else if (cs == 1) {
            if (a.accumulate) {
              const float4 o = *reinterpret_cast<const float4*>(op);
              acc4.x += o.x; acc4.y += o.y; acc4.z += o.z; acc4.w += o.w;
            }
            *reinterpret_cast<float4*>(op) = acc4;
          } else {
            const float vv[4] = {acc4.x, acc4.y, acc4.z, acc4.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              float* qq = op + (long long)j * cs;
              *qq = a.accumulate ? *qq + vv[j] : vv[j];
            }
          }
        }
      };
      switch (splits) {
        case 2: reduce_rows(std::integral_constant<int, 2>{}); break;
        case 4: reduce_rows(std::integral_constant<int, 4>{}); break;
        default: reduce_rows(std::integral_constant<int, 8>{}); break;
      }
    }
    TC_MARK(9, tid == 0);
    cluster_sync_all();   // nobody leaves (and frees its shared memory) while a peer may still be reading it
  }
  TC_MARK(10, tid == 0);
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// ---- tensor maps (host) ----------------------------------------------------------------------------------
// cuTensorMapEncode* are driver entry points; they are fetched through the runtime so that the library does not depend on
// the link order of libcuda.  Maps are cached by (pointer, geometry): the engine's buffers are static, so every map is
// encoded once per engine lifetime and reused by every launch / graph replay.
typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const int*,
                                   const int*, cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

struct TmaApi {
  EncodeIm2colFn im2col = nullptr;
  EncodeTiledFn tiled = nullptr;
  int driver = 0;
  bool ok = false;
};
const TmaApi& tma_api() {
  static const TmaApi api = [] {
    TmaApi t;
    cudaDriverEntryPointQueryResult q;
    void* f = nullptr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &f, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      t.im2col = reinterpret_cast<EncodeIm2colFn>(f);
    f = nullptr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      t.tiled = reinterpret_cast<EncodeTiledFn>(f);
    cudaDriverGetVersion(&t.driver);
    t.ok = t.im2col != nullptr && t.tiled != nullptr;
    return t;
  }();
  return api;
}

using MapKey = std::array<long long, 16>;
std::mutex g_map_mutex;
std::map<MapKey, CUtensorMap> g_map_cache;

// im2col map over an NHWC view [N][H][W][C] (element strides sN, sP = pixel stride, channels contiguous).  One load =
// `pixels` consecutive base pixels (walked along W, then H, then N inside the box [lower, dim - 1 + upper], step `stride`)
// x `chans` channels; elements outside the tensor read as zero.
bool im2col_map(CUtensorMap* out, const float* base, int N, int H, int W, int C, long long sN, int sP, int lower_w, int lower_h,
                int upper_w, int upper_h, int stride, int chans, int pixels, CUtensorMapSwizzle swz) {
  const MapKey key = {0, (long long)reinterpret_cast<uintptr_t>(base), N, H, W, C, sN, sP, lower_w, lower_h, upper_w, upper_h, stride, chans,
                      pixels, (long long)swz};
  std::lock_guard<std::mutex> lock(g_map_mutex);
  auto it = g_map_cache.find(key);
  if (it != g_map_cache.end()) { *out = it->second; return true; }
  const TmaApi& api = tma_api();
  if (!api.ok) return false;
  const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  const cuuint64_t strides[3] = {(cuuint64_t)sP * 4, (cuuint64_t)W * sP * 4, (cuuint64_t)sN * 4};
  const int lower[2] = {lower_w, lower_h}, upper[2] = {upper_w, upper_h};
  const cuuint32_t estr[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
  CUtensorMap tm;
  const CUresult res = api.im2col(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(base), dims, strides, lower, upper,
                                  (cuuint32_t)chans, (cuuint32_t)pixels, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                                  CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (res != CUDA_SUCCESS) return false;
  g_map_cache.emplace(key, tm);
  *out = tm;
  return true;
}

bool tiled_map(CUtensorMap* out, const float* base, int rank, const long long* dims_ll, const long long* strides_elems, const int* box_i,
               CUtensorMapSwizzle swz) {
  MapKey key = {1, (long long)reinterpret_cast<uintptr_t>(base), rank, (long long)swz};
  for (int i = 0; i < rank; ++i) { key[4 + i] = dims_ll[i]; key[8 + i] = box_i[i]; if (i + 1 < rank) key[12 + i] = strides_elems[i]; }
  std::lock_guard<std::mutex> lock(g_map_mutex);
  auto it = g_map_cache.find(key);
  if (it != g_map_cache.end()) { *out = it->second; return true; }
  const TmaApi& api = tma_api();
  if (!api.ok) return false;
  cuuint64_t dims[3], strides[2];
  cuuint32_t box[3], estr[3] = {1, 1, 1};
  for (int i = 0; i < rank; ++i) { dims[i] = (cuuint64_t)dims_ll[i]; box[i] = (cuuint32_t)box_i[i]; }
  for (int i = 0; i + 1 < rank; ++i) strides[i] = (cuuint64_t)strides_elems[i] * 4;
  CUtensorMap tm;
  const CUresult res = api.tiled(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, const_cast<float*>(base), dims, strides, box, estr,
                                 CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (res != CUDA_SUCCESS) return false;
  g_map_cache.emplace(key, tm);
  *out = tm;
  return true;
}

// Does the TMA producer cover this contraction?  (strided dgrad does not: see the header of this file.)
bool tma_eligible(const GemmArgs& a) {
  if (!gemm_switches().tc_tma || !tma_api().ok) return false;
  const ConvGeom& g = a.g;
  if (g.stride > 8 || g.pad > 127 || g.R - 1 - g.pad > 127 || g.S - 1 - g.pad > 127 || g.R > 128 || g.S > 128) return false;
  if (a.mode == GEMM_DGRAD) return g.stride == 1;
  if (a.mode == GEMM_WGRAD) return g.Ci % 32 == 0;
  return true;
}

// 128 x 32 / 64 x 32 tiles exist for the TMA producer only
bool narrow_tiles_ok(const GemmArgs& a) { return gemm_switches().tc_narrow && tma_eligible(a); }

// BM: pixels per im2col box (the tile's rows; part of the map's cache key)
bool build_maps(const GemmArgs& a, int BN, TcMaps* maps, int BM = TC_BM) {
  const ConvGeom& g = a.g;
  const CUtensorMapSwizzle K128 = CU_TENSOR_MAP_SWIZZLE_128B;
  for (int s = 0; s < a.nsrc; ++s) {
    if (a.mode == GEMM_FPROP) {
      if (!im2col_map(&maps->act[s], a.act[s], g.N, g.H, g.W, g.Ci, a.x_sN, a.x_sP, -g.pad, -g.pad, g.pad - (g.S - 1), g.pad - (g.R - 1),
                      g.stride, TC_BK, BM, K128))
        return false;
      const long long K = (long long)g.R * g.S * g.Ci;
      const long long dims[2] = {K, g.Co}, strides[1] = {K};
      const int box[2] = {TC_BK, BN};
      if (!tiled_map(&maps->wgt[s], a.wgt[s], 2, dims, strides, box, K128)) return false;
    } else if (a.mode == GEMM_DGRAD) {
      // rows = pixels of the input gradient; the gathered tensor is dout [N][Ho][Wo][Co]; tap (r, s) reads (y + pad - r, x + pad - s)
      const int lw = g.pad - (g.S - 1), lh = g.pad - (g.R - 1);
      if (!im2col_map(&maps->act[s], a.act[s], g.N, g.Ho, g.Wo, g.Co, (long long)g.Ho * g.Wo * g.Co, g.Co, lw, lh, lw + g.W - g.Wo,
                      lh + g.H - g.Ho, 1, TC_BK, BM, K128))
        return false;
      const long long dims[3] = {g.Ci, (long long)g.R * g.S, g.Co}, strides[2] = {g.Ci, (long long)g.R * g.S * g.Ci};
      const int box[3] = {32, 1, TC_BK};
      if (!tiled_map(&maps->wgt[s], a.wgt[s], 3, dims, strides, box, K128)) return false;
    } else {
      // A(m = ko, k = pixel) = dout[pixel][ko]; B(n = (r, s, c), k = pixel) = im2col of the activation, 32 pixels x 32 channels
      const long long npix = (long long)g.N * g.Ho * g.Wo;
      const long long dims[2] = {g.Co, npix}, strides[1] = {g.Co};
      const int box[2] = {32, TC_BK};
      if (!tiled_map(&maps->wgt[s], a.wgt[s], 2, dims, strides, box, K128)) return false;
      if (!im2col_map(&maps->act[s], a.act[s], g.N, g.H, g.W, g.Ci, a.x_sN, a.x_sP, -g.pad, -g.pad, g.pad - (g.S - 1), g.pad - (g.R - 1),
                      g.stride, 32, TC_BK, K128))
        return false;
    }
  }
  return true;
}

// ---- per-class plan of a strided dgrad (oracle/strided_dgrad.py class_plan, per axis) ---------------------------------------------
struct AxisPlan { bool any; int y0, Hc, T, L, U; };
inline AxisPlan axis_plan(int H, int Ho, int R, int stride, int pad, int e) {
  AxisPlan p{false, 0, 0, 0, 0, 0};
  p.y0 = ((e - pad) % stride + stride) % stride;
  if (p.y0 >= H) return p;                       // no input pixel of this parity
  p.any = true;
  p.Hc = (H - p.y0 + stride - 1) / stride;
  if (e >= R) return p;                          // pixels exist, no tap reaches them: T = 0
  p.T = (R - e + stride - 1) / stride;
  const int c = (p.y0 + pad - e) / stride;
  p.L = c - (p.T - 1);
  p.U = p.Hc - Ho + p.L;
  return p;
}

bool cls_eligible(const GemmArgs& a) {
  const GemmSwitches& sw = gemm_switches();
  const ConvGeom& g = a.g;
  if (!sw.tc_strided_tma || !sw.tc_tma || a.mode != GEMM_DGRAD || g.stride != 2 || !tma_api().ok) return false;
  if (g.R > 16 || g.S > 16) return false;
  for (int ey = 0; ey < 2; ++ey)
    for (int horiz = 0; horiz < 2; ++horiz) {
      const AxisPlan p = horiz ? axis_plan(g.W, g.Wo, g.S, 2, g.pad, ey) : axis_plan(g.H, g.Ho, g.R, 2, g.pad, ey);
      if (p.any && p.T > 0 && (p.L < -128 || p.L > 127 || p.U < -128 || p.U > 127)) return false;
    }
  return true;
}

// The classes of a strided dgrad: pixel grids, taps, tap corners and m-tile ranges (host arithmetic only)
bool class_plan(const ConvGeom& g, ClsPlan* plan) {
  memset(plan, 0, sizeof(*plan));
  plan->stride = g.stride;
  int tiles = 0, n = 0;
  for (int ey = 0; ey < g.stride; ++ey) {
    const AxisPlan py = axis_plan(g.H, g.Ho, g.R, g.stride, g.pad, ey);
    if (!py.any) continue;
    for (int ex = 0; ex < g.stride; ++ex) {
      const AxisPlan px = axis_plan(g.W, g.Wo, g.S, g.stride, g.pad, ex);
      if (!px.any) continue;
      if (n >= TC_MAXCLS) return false;
      const bool taps = py.T > 0 && px.T > 0;
      plan->Hc[n] = py.Hc; plan->Wc[n] = px.Hc; plan->y0[n] = py.y0; plan->x0[n] = px.y0;
      plan->Ty[n] = taps ? py.T : 0; plan->Tx[n] = taps ? px.T : 0;
      plan->Ly[n] = py.L; plan->Lx[n] = px.L; plan->ey[n] = ey; plan->ex[n] = ex;
      plan->tile0[n] = tiles;
      tiles += ceil_div((long long)g.N * py.Hc * px.Hc, TC_BM);
      ++n;
    }
  }
  plan->ncls = n;
  plan->tile0[n] = tiles;
  return n > 0;
}

bool build_cls_maps(const GemmArgs& a, const ClsPlan& plan, TcMapsCls* maps) {
  const ConvGeom& g = a.g;
  for (int c = 0; c < plan.ncls; ++c) {
    if (plan.Ty[c] == 0) {   // never dereferenced (the class has no k-blocks), but a valid descriptor keeps prefetch.tensormap well defined
      for (int s = 0; s < a.nsrc; ++s) maps->act[2 * c + s] = maps->act[s];
      continue;
    }
    const int Uy = plan.Hc[c] - g.Ho + plan.Ly[c], Ux = plan.Wc[c] - g.Wo + plan.Lx[c];
    for (int s = 0; s < a.nsrc; ++s)
      if (!im2col_map(&maps->act[2 * c + s], a.act[s], g.N, g.Ho, g.Wo, g.Co, (long long)g.Ho * g.Wo * g.Co, g.Co, plan.Lx[c], plan.Ly[c], Ux, Uy,
                      1, TC_BK, TC_BM, CU_TENSOR_MAP_SWIZZLE_128B))
        return false;
  }
  for (int s = 0; s < a.nsrc; ++s) {
    const long long dims[3] = {g.Ci, (long long)g.R * g.S, g.Co}, strides[2] = {g.Ci, (long long)g.R * g.S * g.Ci};
    const int box[3] = {32, 1, TC_BK};
    if (!tiled_map(&maps->wgt[s], a.wgt[s], 3, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B)) return false;
  }
  return true;
}

template <int MODE, int BN, bool TMA, bool CLS = false, int BM = TC_BM>
int launch_tc(const GemmArgs& a, const GemmPlan& p, const std::conditional_t<CLS, TcMapsCls, TcMaps>& maps, cudaStream_t stream,
              const ClsPlan* cls = nullptr) {
  TcDims d;
  gemm_dims(a, d.M, d.Nc, d.K);
  d.kblocks_per_src = ceil_div(d.K, TC_BK);
  d.total_kblocks = p.total_kblocks;
  d.kblocks_per_split = p.kblocks_per_split;
  d.stage_shift = p.stages == 8 ? 3 : (p.stages == 2 ? 1 : 2);
  ClsPlan plan;
  memset(&plan, 0, sizeof(plan));
  if (CLS) plan = *cls;
  const int tm = CLS ? plan.tile0[plan.ncls] : ceil_div(d.M, BM), tn = d.Nc / BN;
  if (tn > 65535) { set_error("igemm_tc: grid too large"); return -1; }
  const size_t smem = (size_t)p.stages * (BM + BN) * TC_BK * 4;
  const size_t smem_max = (size_t)TC_MAX_STAGES * (BM + BN) * TC_BK * 4;
  static bool attr_done = false;
  if (!attr_done) {
    BRE_CUDA_CHECK(cudaFuncSetAttribute(igemm_tc_kernel<MODE, BN, TMA, CLS, BM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max));
    attr_done = true;
  }
  // At most one producer lane per ring stage: a lane that shares a stage with another one could wait on the "empty" parity of a
  // phase two rounds old, which reads as complete, and overwrite a stage still in use (BRE_TC_PRODUCERS=4 with a 2-deep ring).
  const GemmSwitches& sw = gemm_switches();
  const int nprod = sw.tc_producers < p.stages ? sw.tc_producers : p.stages;
  const int flags = (sw.tc_proxy_fence ? 1 : 0) | (sw.tc_prefetch ? 2 : 0) | (nprod << 2);
  cudaError_t lerr = launch_kernel(igemm_tc_kernel<MODE, BN, TMA, CLS, BM>, dim3(tm, tn, p.splits), dim3(TC_BLOCK), smem, stream, p.splits, a,
                                   d, flags, maps, plan);
  if (lerr != cudaSuccess) { set_error(std::string("igemm_tc launch failed: ") + cudaGetErrorString(lerr)); return -2; }
  BRE_CHECK_LAUNCH();
  return 0;
}

template <int MODE, int BN>
int launch_tma(const GemmArgs& a, const GemmPlan& p, const TcMaps& maps, cudaStream_t stream) {
  if constexpr (MODE != GEMM_WGRAD)
    if (p.tile_rows == 64) return launch_tc<MODE, BN, true, false, 64>(a, p, maps, stream);
  return launch_tc<MODE, BN, true>(a, p, maps, stream);
}

template <int MODE>
int launch_mode(const GemmArgs& a, const GemmPlan& p, const TcMaps& maps, cudaStream_t stream) {
  if (p.producer == GEMM_PROD_CP_ASYNC) return launch_tc<MODE, 64, false>(a, p, maps, stream);
  return p.tile_width == 32 ? launch_tma<MODE, 32>(a, p, maps, stream) : launch_tma<MODE, 64>(a, p, maps, stream);
}

}  // namespace

bool igemm_tc_supported(const GemmArgs& a) {
  const ConvGeom& g = a.g;
  int M, Nc, K;
  gemm_dims(a, M, Nc, K);
  for (int s = 0; s < a.nsrc; ++s)
    if (!aligned16(a.act[s]) || !aligned16(a.wgt[s])) return false;
  if (!aligned16(a.out) || a.ws == nullptr) return false;
  const bool x_nhwc = a.x_sC == 1 && a.x_sP % 4 == 0 && a.x_sN % 4 == 0;
  // output tiles are 128 x 64; widths that are only a multiple of 32 (token models: d = 96, 3 d = 288) run 128 x 32 tiles
  if (Nc % 64 != 0 && !(Nc % 32 == 0 && narrow_tiles_ok(a))) return false;
  switch (a.mode) {
    case GEMM_FPROP: return x_nhwc && g.Ci % TC_BK == 0 && g.R * g.S <= 64;  // k-block inside one (r, s) cell
    case GEMM_DGRAD: return x_nhwc && g.Co % TC_BK == 0 && g.R * g.S <= 64;   // (Nc = Ci: tile-width rule above)
    case GEMM_WGRAD: return x_nhwc && g.Co % 4 == 0 && g.Ci % 4 == 0 && g.R * g.S <= 64;
    default: return false;
  }
}

// Every launch rule of the tensor-core back end.  The producer: TMA where the geometry allows it (and allow_tma), per-class tensor maps
// for the stride-2 dgrad, otherwise the cp.async producer of the same kernel (same consumer, still on the GPU: a different loader, not
// a fallback to another implementation).
GemmPlan tc_plan(const GemmArgs& a, bool allow_tma) {
  const GemmSwitches& sw = gemm_switches();
  int M, Nc, K;
  gemm_dims(a, M, Nc, K);
  GemmPlan p;
  p.family = GEMM_FAM_TC; p.mode = a.mode; p.nsrc = a.nsrc;
  int kb = ceil_div(K, TC_BK) * a.nsrc;
  long long tm = ceil_div(M, TC_BM);
  ClsPlan cls;
  if (allow_tma && cls_eligible(a) && class_plan(a.g, &cls)) {
    // strided dgrad: the m-tiles of all classes side by side; the k extent that sizes the split is the largest class's
    int kmax = 0;
    for (int c = 0; c < cls.ncls; ++c) kmax = kmax > cls.Ty[c] * cls.Tx[c] ? kmax : cls.Ty[c] * cls.Tx[c];
    kb = kmax * (a.g.Co / TC_BK) * a.nsrc;
    if (kb < 1) kb = 1;
    tm = cls.tile0[cls.ncls];
    p.tile_rows = TC_BM; p.tile_width = 64; p.producer = GEMM_PROD_CLASSES;
  } else {
    const bool tma = allow_tma && tma_eligible(a), narrow = allow_tma && narrow_tiles_ok(a);
    if (Nc % 64 != 0 && !narrow) return GemmPlan();
    // 128 x 32 tiles: widths that are only a multiple of 32, and data / weight gradients whose 128 x 64 tiles would fill at most
    // half the SMs even at the full 8-CTA split while every CTA walks a long k-range (batch 1: ResNet-18's layer-3 / layer-4 dgrad,
    // 8 tiles x 8 = 64 CTAs over 9-36 k-blocks each; the stem's column wgrad, 3 tiles x 49).  Their mma.sync consumer (fragments
    // loaded with ld.shared) bounds the k-loop; halving the tile width doubles the CTAs and halves each CTA's MMA and fragment-load
    // work per k-block, while every output element keeps the same k-blocks per split, the same MMA accumulation chain and the same
    // fixed-order cluster reduction: the result is bitwise the one of 128 x 64 tiles.  Both grids stay <= kNumSMs, so the split-K
    // rule picks the same 8-way split for either.  Measured per launch on the H100 (scripts/profile_gemms.py, DESIGN.md section 6):
    // dgrad 15-44 -> 10-32 us, the stem wgrad 44 -> 34 us; the wgmma fprop of the same shapes gained 0-2 us on some and lost 2 us on
    // layer 4's, so it keeps 128 x 64 tiles.
    const bool underfilled = a.mode != GEMM_FPROP && Nc % 64 == 0 && tm * (Nc / 64) * 16 <= kNumSMs && kb >= 64 && narrow;
    p.tile_width = Nc % 64 != 0 || underfilled ? 32 : 64;
    // 64-row tiles for an m-tile of <= 64 GEMM rows (batch 1: every 7 x 7 layer-4 launch, M = 49): a 128-row im2col box would stage
    // 64+ rows past the end of the tensor every k-block.  Rows 0-63 see the same wgmma / mma.sync instructions on the same operands,
    // the tile count, split and k-ranges do not change (ceil(M / 64) = ceil(M / 128) = 1), so the result is bitwise that of
    // 128-row tiles.  BRE_TC_STREAM=0 keeps 128-row tiles.
    p.tile_rows = sw.tc_stream && M <= 64 && a.mode != GEMM_WGRAD && tma ? 64 : TC_BM;
    p.producer = tma ? GEMM_PROD_TMA : GEMM_PROD_CP_ASYNC;
  }
  // split-K factor = cluster size along z: a power of two <= 8 (portable cluster limit) that brings the grid to about one wave
  const long long tiles = tm * (Nc / p.tile_width);
  const int target = sw.tc_target_ctas > 0 ? sw.tc_target_ctas : kNumSMs;
  constexpr int kMaxCluster = 8;  // portable cluster size
  int splits = 1;
  while (splits < kMaxCluster && tiles * splits < target && kb / (splits * 2) >= 2) splits *= 2;
  if (sw.tc_max_splits > 0 && splits > sw.tc_max_splits) splits = sw.tc_max_splits;
  int pow2 = 1;
  while (pow2 * 2 <= splits && pow2 < kMaxCluster) pow2 *= 2;
  splits = pow2;
  while (splits > 1 && splits > kb) splits /= 2;
  p.splits = splits;
  p.total_kblocks = kb;
  p.kblocks_per_split = ceil_div(kb, splits);
  // Ring depth: 4 stages (96 KB: two CTAs per SM within the 227 KB an SM offers, and the next kernel's CTAs can become resident
  // during this one's tail -- what programmatic dependent launch needs).  BRE_TC_STAGES=2|4|8 forces a depth for experiments
  // (8 stages = 192 KB, one CTA per SM).
  // Short reductions on many tiles (the token models' decoder fprop: 786 tiles x 3-6 k-blocks): a 2-deep ring halves the shared
  // memory so more CTAs share an SM and the per-CTA prologue / epilogue overlap (BRE_TC_SHORTK_STAGES=4 turns it off).
  const bool shortk = sw.tc_shortk_stages == 2 && p.kblocks_per_split <= 6 && tm == 1 && tiles * splits > 2LL * kNumSMs;
  // 64-row tiles stage half the bytes per k-block, so an 8-deep ring (fprop 128 KB, 128 x 32 dgrad 96 KB) still leaves room for one
  // 96 KB CTA of the successor.  It pays on launches that are one wave or less and whose CTAs walk long k-ranges: there the k-loop
  // is the latency of the ring round trip divided by the k-blocks in flight.
  const bool deep = p.tile_rows == 64 && tiles * splits <= kNumSMs && p.kblocks_per_split >= 16;
  const int forced = sw.tc_stages;
  p.stages = (forced == 8 || forced == 2 || forced == 4) ? forced : (shortk ? 2 : (deep ? 8 : TC_STAGES));
  return p;
}

int launch_igemm_tc(const GemmArgs& a, GemmPlan& p, cudaStream_t stream) {
  if (p.producer == GEMM_PROD_CLASSES) {
    ClsPlan cls;
    TcMapsCls maps;
    memset(&maps, 0, sizeof(maps));
    if (class_plan(a.g, &cls) && build_cls_maps(a, cls, &maps)) return launch_tc<GEMM_DGRAD, 64, true, true>(a, p, maps, stream, &cls);
  } else {
    TcMaps maps;
    memset(&maps, 0, sizeof(maps));
    if (p.producer == GEMM_PROD_CP_ASYNC || build_maps(a, p.tile_width, &maps, p.tile_rows)) {
      if (a.mode == GEMM_FPROP) return launch_mode<GEMM_FPROP>(a, p, maps, stream);
      if (a.mode == GEMM_DGRAD) return launch_mode<GEMM_DGRAD>(a, p, maps, stream);
      return launch_mode<GEMM_WGRAD>(a, p, maps, stream);
    }
  }
  // a tensor map of the plan did not encode: the plan of the cp.async producer, which exists unless the width is only a multiple of 32
  p = tc_plan(a, false);
  if (p.family < 0) { set_error("igemm_tc: tensor-map encoding failed for a narrow-tile shape"); return -4; }
  return launch_igemm_tc(a, p, stream);
}

}  // namespace bre

#ifdef BRE_TC_TRACE
extern "C" int bre_debug_tc_trace(long long* out16) {
  return cudaMemcpyFromSymbol(out16, bre::g_tc_trace, sizeof(long long) * 16) == cudaSuccess ? 0 : -1;
}
#endif
