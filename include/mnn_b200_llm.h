/* mnn_b200_llm.h -- C ABI of libmnn_b200_llm.so: the stateless float ops of MNN-LLM's decoder layers besides the linear layers
 * (LayerNorm / RMSNorm with the fused residual form, and the fused RoPE), as an extension of include/mnn_b200.h.
 *
 * The library links libmnn_b200.so and shares its runtime and execution handles: create takes an mnnb200_runtime from
 * mnnb200_runtime_create, work is enqueued on that runtime's stream, the executions are mnnb200_exec handles destroyed with
 * mnnb200_exec_destroy, and a failed call's message is mnnb200_last_error().  Every entry point refuses an execution of another
 * type (INVALID_VALUE), and the entry points of mnn_b200.h refuse these executions. */
#ifndef MNN_B200_LLM_H
#define MNN_B200_LLM_H
#include "mnn_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- LayerNorm / RMSNorm and the fused RoPE of MNN-LLM's decoder layers (CPULayerNorm, CPURoPE) on device fp32 tensors.
 *      layernorm_f32: every row of an [rows][inner] view: mean = sum(x) / inner (0 when rms != 0),
 *                  inv = 1 / sqrt(sum((x - mean)^2) / inner + eps), y = (x - mean) * inv, then y * gamma + beta when gamma and beta
 *                  are both given (a gamma alone is ignored, CPULayerNorm.cpp:35; affine_size must be inner then).
 *                  inner <= 32768 (the row stays in registers).  resize takes rows: outer size, or length(0) * group for a grouped
 *                  norm.  execute: residual and sum both NULL, or both given for the residual form sum = x + residual,
 *                  y = norm(sum).  The reductions run in another order than the CPU's: results within rounding of it.
 *      rope_f32:   q [seq][heads * head_dim], k [seq][kv_heads * head_dim], cos / sin [seq][ropeDim] (first half "even", second
 *                  half "odd"), ropeDim = rope_cut in (0, head_dim] else head_dim, rounded down to even.  Per head,
 *                  out[j] = x[j] * cos[j] - x[j + ropeDim / 2] * sin[j] and out[j + ropeDim / 2] = x[j + ropeDim / 2] * cos[j + ropeDim / 2]
 *                  + x[j] * sin[j + ropeDim / 2] for j < ropeDim / 2, each product and sum rounded as the CPU rounds it (bit-identical);
 *                  dims from ropeDim on are copied.  A q / k norm (gamma of head_dim values, beta NULL = zeros) normalises each head
 *                  first, as layernorm_f32 with the affine transform; then the copied dims are the normalised values.
 *                  resize takes seq and the inputs' widths, which must be heads * head_dim and kv_heads * head_dim.
 *      NOT_SUPPORT, the previous plan kept: affine size != inner, heads / kv_heads / head_dim <= 0, a norm table without gamma or
 *      of another size than head_dim, a width that does not match, zero rows / tokens, an index past 32-bit limits.
 *      x, y and the tensors need 4-byte alignment; 16-byte aligned rows take the vector path. */
typedef struct mnnb200_rope_norm {
    const float* gamma;   /* [size] */
    const float* beta;    /* [size] or NULL */
    int size;             /* must be head_dim */
    float eps;
    int rms;              /* 1: RMSNorm (no mean) */
} mnnb200_rope_norm;
MNNB200_API mnnb200_status mnnb200_layernorm_f32_create(mnnb200_runtime* rt, int inner, float eps, int rms, const float* gamma,
                                                        const float* beta, int affine_size, mnnb200_exec** out);
MNNB200_API mnnb200_status mnnb200_layernorm_f32_resize(mnnb200_exec* e, int rows);
MNNB200_API mnnb200_status mnnb200_layernorm_f32_execute(mnnb200_exec* e, const float* x, const float* residual, float* sum, float* y);
MNNB200_API mnnb200_status mnnb200_rope_f32_create(mnnb200_runtime* rt, int heads, int kv_heads, int head_dim, int rope_cut,
                                                   const mnnb200_rope_norm* q_norm, const mnnb200_rope_norm* k_norm,
                                                   mnnb200_exec** out);
MNNB200_API mnnb200_status mnnb200_rope_f32_resize(mnnb200_exec* e, int seq, int q_width, int k_width);
MNNB200_API mnnb200_status mnnb200_rope_f32_execute(mnnb200_exec* e, const float* q, const float* k, const float* cos, const float* sin,
                                                    float* q_out, float* k_out);

#ifdef __cplusplus
}
#endif
#endif /* MNN_B200_LLM_H */
