// llm_ops.cu -- the stateless float ops of an MNN-LLM decoder layer besides its linear layers: LayerNorm / RMSNorm (with the
// fused residual form) and the fused RoPE (with the optional per-head q / k norm), fp32, on the linear device layouts.
//
// layernorm_f32_kernel: CPULayerNorm (source/backend/cpu/CPULayerNorm.cpp:70-226) over an [rows][inner] view, one CTA per row.
// The row stays in registers between the reductions and the write, so HBM sees one read and one write per element (two and
// two in the residual form).  Each thread holds V float4 units of the row (16-byte accesses) when every pointer is 16-byte
// aligned and inner % 4 == 0, else 4V scalars at a stride of the CTA size (the same coalesced rows, 4-byte accesses).
//
// rope_f32_kernel: CPURoPE::onExecute (CPURoPE.cpp:159-265) + MNNRoPEComputeBasic (compute/CommonOptFunction.cpp:4731-4773),
// one warp per (token, head) over the q heads and then the k heads of every token, one launch.  The rotation is written with
// explicitly rounded operations in the CPU's order (the reference's SSE Vec4::fms / fma are a rounded multiply then a rounded
// add: no FMA, compute/ is built without -mfma), so RoPE without q / k norms is bit-identical to the CPU.
#include "common.cuh"
#include "llm_ops.h"

namespace mnnb200 {
namespace {

// sum of v over the CTA, returned to every thread; red holds 32 floats and is free again when this returns
__device__ __forceinline__ float block_sum(float v, float* red) {
    for (int s = 16; s > 0; s >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, s));
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    if (lane == 0) red[warp] = v;
    __syncthreads();
    v = lane < nw ? red[lane] : 0.f;
    for (int s = 16; s > 0; s >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, s));
    __syncthreads();   // every warp has read red before the next reduction writes it
    return v;
}

// y = (x - mean) * inv, then y * gamma + beta when both are present (the CPU's unfused order)
__device__ __forceinline__ float norm_one(float v, float mean, float inv, const float* g, const float* b, int i) {
    float y = __fmul_rn(__fsub_rn(v, mean), inv);
    if (g) y = __fadd_rn(__fmul_rn(y, g[i]), b[i]);
    return y;
}

// mean = sum / n (0 for RMSNorm) and inv = 1 / sqrt(sumsq / n + eps), sumsq over (x - mean)^2 (MNNNorm's two passes)
__device__ __forceinline__ float inv_std(float sumsq, int n, float eps) {
    return __fdiv_rn(1.f, __fsqrt_rn(__fadd_rn(__fdiv_rn(sumsq, (float)n), eps)));
}

template <int V, bool VEC>
__global__ void __launch_bounds__(V == kLayerNormMaxV ? 512 : 256) layernorm_f32_kernel(LayerNormParams p) {
    __shared__ float red[32];
    const size_t row = blockIdx.x;
    const int n = p.inner, T = blockDim.x, t = threadIdx.x;
    const size_t base = row * (size_t)n;
    const float* x = p.x + base;
    const float* r = p.r ? p.r + base : nullptr;
    float v[4 * V];
    float sum = 0.f;
    if (VEC) {
        const int n4 = n >> 2;
#pragma unroll
        for (int k = 0; k < V; ++k) {
            const int u = k * T + t;
            float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
            if (u < n4) {
                a = reinterpret_cast<const float4*>(x)[u];
                if (r) {
                    const float4 b = reinterpret_cast<const float4*>(r)[u];
                    a.x = __fadd_rn(a.x, b.x); a.y = __fadd_rn(a.y, b.y); a.z = __fadd_rn(a.z, b.z); a.w = __fadd_rn(a.w, b.w);
                    reinterpret_cast<float4*>(p.s + base)[u] = a;
                }
            }
            v[4 * k] = a.x; v[4 * k + 1] = a.y; v[4 * k + 2] = a.z; v[4 * k + 3] = a.w;
        }
    } else {
#pragma unroll
        for (int k = 0; k < 4 * V; ++k) {
            const int e = k * T + t;
            float a = 0.f;
            if (e < n) {
                a = x[e];
                if (r) {
                    a = __fadd_rn(a, r[e]);
                    p.s[base + e] = a;
                }
            }
            v[k] = a;
        }
    }
    // element index of register slot k (n or more: outside the row)
    auto index = [&](int k) -> int { return VEC ? ((k >> 2) * T + t) * 4 + (k & 3) : k * T + t; };
    float mean = 0.f;
    if (!p.rms) {
#pragma unroll
        for (int k = 0; k < 4 * V; ++k) sum = __fadd_rn(sum, v[k]);   // slots outside the row hold 0
        mean = __fdiv_rn(block_sum(sum, red), (float)n);
    }
    float sq = 0.f;
#pragma unroll
    for (int k = 0; k < 4 * V; ++k) {
        const float d = __fsub_rn(v[k], mean);
        if (index(k) < n) sq = __fadd_rn(sq, __fmul_rn(d, d));
    }
    const float inv = inv_std(block_sum(sq, red), n, p.eps);
    float* y = p.y + base;
    if (VEC) {
        const int n4 = n >> 2;
#pragma unroll
        for (int k = 0; k < V; ++k) {
            const int u = k * T + t;
            if (u < n4) {
                float4 o;
                o.x = norm_one(v[4 * k], mean, inv, p.gamma, p.beta, 4 * u);
                o.y = norm_one(v[4 * k + 1], mean, inv, p.gamma, p.beta, 4 * u + 1);
                o.z = norm_one(v[4 * k + 2], mean, inv, p.gamma, p.beta, 4 * u + 2);
                o.w = norm_one(v[4 * k + 3], mean, inv, p.gamma, p.beta, 4 * u + 3);
                reinterpret_cast<float4*>(y)[u] = o;
            }
        }
    } else {
#pragma unroll
        for (int k = 0; k < 4 * V; ++k) {
            const int e = k * T + t;
            if (e < n) y[e] = norm_one(v[k], mean, inv, p.gamma, p.beta, e);
        }
    }
}

template <int V>
cudaError_t launch_v(const LayerNormParams& p, bool vec, int threads, cudaStream_t s) {
    if (vec) layernorm_f32_kernel<V, true><<<p.rows, threads, 0, s>>>(p);
    else layernorm_f32_kernel<V, false><<<p.rows, threads, 0, s>>>(p);
    return cudaGetLastError();
}

// One warp per (token, head).  A normalised head reads its input twice (statistics, then the rotation), the second time from L1.
__global__ void __launch_bounds__(256) rope_f32_kernel(RopeParams p) {
    const int lane = threadIdx.x & 31;
    const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int hall = p.heads + p.kv_heads;
    if (w >= (long long)p.seq * hall) return;
    const int token = (int)(w / hall), h = (int)(w - (long long)token * hall);
    const bool isq = h < p.heads;
    const int nh = isq ? p.heads : p.kv_heads, hh = isq ? h : h - p.heads;
    const int hd = p.head_dim, half = p.rope_dim >> 1;
    const size_t off = ((size_t)token * nh + hh) * hd;
    const float* src = (isq ? p.q : p.k) + off;
    float* dst = (isq ? p.qo : p.ko) + off;
    // the side's norm table, selected field by field so that the parameter block stays in constant memory
    const float* g = isq ? p.qn.gamma : p.kn.gamma;
    const float* beta = isq ? p.qn.beta : p.kn.beta;
    const float eps = isq ? p.qn.eps : p.kn.eps;
    const int rms = isq ? p.qn.rms : p.kn.rms;
    float mean = 0.f, inv = 1.f;
    if (g) {   // MNNNorm over the head, gamma and beta (zeros when the table has none) always applied (CPURoPE.cpp:20-49)
        if (!rms) {
            float s = 0.f;
            for (int j = lane; j < hd; j += 32) s = __fadd_rn(s, src[j]);
            for (int o = 16; o > 0; o >>= 1) s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
            mean = __fdiv_rn(s, (float)hd);
        }
        float sq = 0.f;
        for (int j = lane; j < hd; j += 32) {
            const float d = __fsub_rn(src[j], mean);
            sq = __fadd_rn(sq, __fmul_rn(d, d));
        }
        for (int o = 16; o > 0; o >>= 1) sq = __fadd_rn(sq, __shfl_xor_sync(0xffffffffu, sq, o));
        inv = inv_std(sq, hd, eps);
    }
    const float* cs = p.cos + (size_t)token * p.rope_dim;
    const float* sn = p.sin + (size_t)token * p.rope_dim;
    for (int j = lane; j < half; j += 32) {
        float q0 = src[j], q1 = src[j + half];
        if (g) {
            q0 = norm_one(q0, mean, inv, g, beta, j);
            q1 = norm_one(q1, mean, inv, g, beta, j + half);
        }
        // dst0 = q0 * cosEven - q1 * sinEven, dst1 = q1 * cosOdd + q0 * sinOdd, each product and the sum rounded
        dst[j] = __fsub_rn(__fmul_rn(q0, cs[j]), __fmul_rn(q1, sn[j]));
        dst[j + half] = __fadd_rn(__fmul_rn(q1, cs[j + half]), __fmul_rn(q0, sn[j + half]));
    }
    for (int j = 2 * half + lane; j < hd; j += 32) dst[j] = g ? norm_one(src[j], mean, inv, g, beta, j) : src[j];
}

}  // namespace

int layernorm_f32_threads(int inner, int* v) {
    const int n4 = (inner + 3) / 4;
    int V = 1;
    while (V < kLayerNormMaxV && (n4 + V - 1) / V > 256) V *= 2;
    const int threads = ((n4 + V - 1) / V + 31) / 32 * 32;
    if (v) *v = V;
    return threads > 512 ? 0 : threads;   // the launch bound of the widest instantiation
}

cudaError_t launch_layernorm_f32(const LayerNormParams& p, cudaStream_t s) {
    int V = 1;
    const int threads = layernorm_f32_threads(p.inner, &V);
    if (!threads || p.rows <= 0) return cudaErrorInvalidValue;
    auto a16 = [](const void* q) { return q == nullptr || ((uintptr_t)q & 15) == 0; };
    const bool vec = p.inner % 4 == 0 && a16(p.x) && a16(p.r) && a16(p.s) && a16(p.y) && a16(p.gamma) && a16(p.beta);
    cudaError_t e;
    switch (V) {
        case 1: e = launch_v<1>(p, vec, threads, s); break;
        case 2: e = launch_v<2>(p, vec, threads, s); break;
        case 4: e = launch_v<4>(p, vec, threads, s); break;
        case 8: e = launch_v<8>(p, vec, threads, s); break;
        default: e = launch_v<16>(p, vec, threads, s); break;
    }
    ++g_launch_count;
    return e;
}

cudaError_t launch_rope_f32(const RopeParams& p, cudaStream_t s) {
    const long long warps = (long long)p.seq * (p.heads + p.kv_heads);
    rope_f32_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, s>>>(p);
    ++g_launch_count;
    return cudaGetLastError();
}

}  // namespace mnnb200
