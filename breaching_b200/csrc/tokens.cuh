// Token-sequence ops (tokens.cu): launchers used by the engine's sweeps for compiler.compile_transformer programs.
#pragma once
#include "common.cuh"

namespace bre {

// LayerNorm / attention sweeps (0 F, 1 B, 2 TF, 3 TB); operands per sweep as documented in tokens.cu.
// round_out (here and below): store `out` on the TF32 grid, after any accumulation (it is an operand of tensor-core GEMMs, see
// tf32_rna in common.cuh)
int launch_token_layernorm(int sweep, const float* x, const float* in1, const float* in2, const float* in3, const float* gamma,
                           const float* beta, const float* v_gamma, const float* v_beta, float eps, int rows, int C, float* stats, float* out,
                           int accumulate, bool round_out, cudaStream_t s);
int launch_token_ln_param_grad(const float* x, const float* dy, const float* stats, int rows, int C, float* g_gamma, float* g_beta,
                               cudaStream_t s);
int launch_token_attention(int sweep, const float* qkv, const float* in1, const float* in2, const float* in3, int B, int T, int heads, int dh,
                           float* P, float* Pd, float* out, int accumulate, bool round_out, cudaStream_t s);
// out[row] = (x ? x[row] : 0) + pos[row mod T]      (learnable positional embedding, language_models.py:133-146)
int launch_token_posadd(const float* x, const float* pos, float* out, int rows, int C, int T, bool round_out, cudaStream_t s);
// g_pos[t] = sum over sequences of d[b*T + t]        (rows t >= T of the embedding table keep a zero gradient)
int launch_token_pos_grad(const float* d, float* g_pos, int rows, int C, int T, cudaStream_t s);
// CausalLoss (losses.py:7-26) with class-probability targets q [rows, V]: row (b, t) is scored against q of row (b, t + 1),
// the last position of every sequence has no target; mean over the M = rows - rows / T scored rows.
// loss_n[row] is pre-scaled by rows / M so that the engine's mean over rows is that mean.
// V = vocabulary size, Vs >= V = row stride of the logits-shaped tensors (vocabulary padded to the GEMM tile width); the label-shaped
// tensors (q, label gradient) are dense [rows, V]
// (round_out: dlogits / tdlogits; the padded columns V .. Vs are not written)
int launch_token_ce_fwd(const float* logits, const float* q, int rows, int V, int Vs, int T, float* p, float* loss_n, float* dlogits, bool round_out,
                        cudaStream_t s);
int launch_token_ce_tan_bwd(const float* p, const float* zdot, int rows, int V, int Vs, int T, float* tdlogits, bool round_out, cudaStream_t s);
// d objective / d q [rows, V]: row (b, t + 1) receives -(zdot - <p, zdot>) / M (+ task_reg * dL/dq) of the logits row (b, t)
int launch_token_label_grad(const float* logits, const float* p, const float* zdot, int rows, int V, int Vs, int T, float task_reg,
                            float* out, cudaStream_t s);

}  // namespace bre
