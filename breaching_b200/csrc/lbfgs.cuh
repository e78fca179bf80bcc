// L-BFGS on the device: the inner loop of torch.optim.LBFGS (no line search) as kernels that keep every scalar on the device, so
// that one optimizer.step runs inside a conditional CUDA graph (engine.cu iteration_lbfgs).  The two-loop recursion is evaluated
// over Gram matrices SY[i][j] = s_i.y_j and YY[i][j] = y_i.y_j of the ring (kept per slot, updated when a pair is pushed): one pass
// over the ring for the new pair's Gram row / column and S^T g, Y^T g; one CTA for the m x m scalar recurrence in fp64; one pass
// that forms d and reduces g.d and max|d|.
#pragma once
#include "../../include/breaching_b200.h"
#include "common.cuh"

namespace bre {

// Device buffers of one optimiser over a flat vector of n floats (the candidate, then the label logits of a joint trial).
struct LbfgsView {
  long long n = 0;
  int R = 0;                       // ring slots = history + 1 (one spare)
  bre_lbfgs_consts k;
  float *S = nullptr, *Y = nullptr;             // [R, n]
  float *g = nullptr, *prev_g = nullptr, *d = nullptr;   // [n]: processed gradient of the last closure, previous gradient, direction
  double* gram = nullptr;          // [SY R*R | YY R*R | rho R | coefficients 2R]
  double* partials = nullptr;      // [gram_blocks, 5R + 4] per-block partial dot products, then [blocks, 2] of the vector passes
  int* counter = nullptr;          // last-block counter of the vector passes
  bre_lbfgs_scalars* st = nullptr;
  int gram_blocks = 1;
  __host__ __device__ double* SY() const { return gram; }
  __host__ __device__ double* YY() const { return gram + (long long)R * R; }
  __host__ __device__ double* rho() const { return gram + 2LL * R * R; }
  __host__ __device__ double* coef() const { return gram + 2LL * R * R + R; }
};
// grid of the ring pass and capacity the partials need for a vector of n (history h)
int lbfgs_gram_blocks(long long n);
long long lbfgs_partials_size(long long n, int history);

// The segments of the optimised vector: x[0] = candidate (n[0] values, boxed to [lo, hi] per channel when `boxed`), x[1] = label
// logits (n[1] values, 0 when absent); best[] = their best-so-far copies.
struct LbfgsSegs {
  float* x[2]; float* best[2]; long long n[2];
  const float* lo; const float* hi; int C, HW, boxed;
};

// after a closure: loss = total objective, max|g| and sum|g|.  first: the step's first closure (records it, saves its objective
// terms, sets `loop` = whether the inner loop runs); else: counts the evaluation and applies tolerance_grad.  `use_handle` = 0
// outside a graph.
int launch_lbfgs_closure_tail(const LbfgsView& v, bool first, Scalars* sc, float task_reg, unsigned long long loop, int use_handle,
                              cudaStream_t s);
// the direction of one inner iteration: candidate pair + push, recurrence, d and g.d.  `eval` is set to whether the re-evaluation
// runs; lr_table NULL leaves t unchanged (the stand-alone entry).
int launch_lbfgs_direction(const LbfgsView& v, const float* lr_table, int n_lr, const Scalars* sc, unsigned long long eval, int use_handle,
                           cudaStream_t s);
// x += t d over the segments unless the inner loop broke on g.d
int launch_lbfgs_step(const LbfgsView& v, const LbfgsSegs& seg, cudaStream_t s);
// the remaining stop tests of the inner iteration -> `loop`
int launch_lbfgs_tail(const LbfgsView& v, unsigned long long loop, cudaStream_t s);
// after the step: box projection, best-so-far on the first loss of the step, and that closure's terms back into sc for launch_commit
int launch_lbfgs_finish(const LbfgsView& v, const LbfgsSegs& seg, Scalars* sc, cudaStream_t s);

}  // namespace bre
