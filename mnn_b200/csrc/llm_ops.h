// llm_ops.h -- host-callable launchers of libmnn_b200_llm.so's kernels (llm_ops.cu), enqueue-only on the given stream.
#pragma once
#include <cuda_runtime.h>

namespace mnnb200 {

// LayerNorm / RMSNorm over the rows of an [rows][inner] fp32 view (llm_ops.cu).  r / s: the residual form (s = x + r, y = norm(s)),
// both or neither; gamma / beta: the affine transform, both or neither.
struct LayerNormParams {
    const float* x;
    const float* r;
    float* s;
    float* y;
    const float* gamma;
    const float* beta;
    int rows, inner;
    float eps;
    int rms;
};
constexpr int kLayerNormMaxV = 16;   // float4 units of a row per thread: a row of up to 512 * 16 * 4 = 32768 elements
// CTA size for a row of `inner` elements (0: the row does not fit in registers); *v = float4 units per thread
int layernorm_f32_threads(int inner, int* v);
cudaError_t launch_layernorm_f32(const LayerNormParams& p, cudaStream_t s);

// fused RoPE (llm_ops.cu): q [seq][heads][head_dim], k [seq][kv_heads][head_dim], cos / sin [seq][rope_dim] (the first half the
// "even", the second the "odd" table); the dims from rope_dim on are copied.  A norm with gamma != nullptr is applied per head
// before the rotation.
struct RopeNorm {
    const float* gamma;   // [head_dim] or nullptr: no norm
    const float* beta;    // [head_dim]
    float eps;
    int rms;
};
struct RopeParams {
    const float *q, *k, *cos, *sin;
    float *qo, *ko;
    int seq, heads, kv_heads, head_dim, rope_dim;
    RopeNorm qn, kn;
};
cudaError_t launch_rope_f32(const RopeParams& p, cudaStream_t s);

}  // namespace mnnb200
