// elementwise.cu -- HBM-bound neighbours of the int8 GEMM path: boundary casts (fused with the
// NCHW <-> NHWC16 layout change), depthwise int8 conv, per-token dynamic activation quantisation.
// All are bandwidth kernels: 16-byte vector accesses on the NHWC16 side, one 16-channel group per thread.
#include "activations.cuh"
#include "common.cuh"
#include "kernels.h"

namespace mnnb200 {

static inline int grid_for(size_t work, int block) {
    size_t g = (work + block - 1) / block;
    return (int)(g > 0x7fffffff ? 0x7fffffff : (g == 0 ? 1 : g));
}

// ---- FloatToInt8: fp32 NCHW -> int8 NHWC16 (CPUCast.cpp:17-37 + x86_x64/avx512/GemmInt8.cpp:234-283)
__global__ void float_to_int8_kernel(const float* __restrict__ x, int n, int c, int hw, int cp, float inv_scale,
                                     float zero, float minv, float maxv, int8_t* __restrict__ y) {
    const int groups = cp >> 4;
    size_t total = (size_t)n * hw * groups;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        int pix = (int)(i % hw);
        size_t t = i / hw;
        int g = (int)(t % groups);
        int b = (int)(t / groups);
        uint32_t out[4];
#pragma unroll
        for (int v = 0; v < 4; ++v) {
            uint32_t word = 0;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                int ch = g * 16 + v * 4 + k;
                int q = 0;
                if (ch < c) q = quant_avx512_exact(x[((size_t)b * c + ch) * hw + pix], inv_scale, zero, minv, maxv);
                word |= (uint32_t)(q & 0xff) << (8 * k);
            }
            out[v] = word;
        }
        *reinterpret_cast<uint4*>(y + ((size_t)b * hw + pix) * cp + g * 16) = make_uint4(out[0], out[1], out[2], out[3]);
    }
}

// ---- Int8ToFloat: int8 NHWC16 -> fp32 NCHW (x86_x64/avx512/GemmInt8.cpp:285-347):
//      (float(q + 128) - (zero + 128)) * scale   -- both offsets are exact in fp32
__global__ void int8_to_float_kernel(const int8_t* __restrict__ x, int n, int c, int hw, int cp, float scale,
                                     float zero, float* __restrict__ y) {
    const int groups = cp >> 4;
    size_t total = (size_t)n * hw * groups;
    const float z128 = __fadd_rn(zero, 128.f);
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        int pix = (int)(i % hw);
        size_t t = i / hw;
        int g = (int)(t % groups);
        int b = (int)(t / groups);
        int4 v = *reinterpret_cast<const int4*>(x + ((size_t)b * hw + pix) * cp + g * 16);
        const int8_t* q = reinterpret_cast<const int8_t*>(&v);
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            int ch = g * 16 + k;
            if (ch < c) {
                float u = __int2float_rn((int)q[k] + 128);
                y[((size_t)b * c + ch) * hw + pix] = __fmul_rn(__fsub_rn(u, z128), scale);
            }
        }
    }
}

__global__ void pack_nchw_int8_kernel(const int8_t* __restrict__ x, int n, int c, int hw, int cp, int8_t* __restrict__ y) {
    const int groups = cp >> 4;
    size_t total = (size_t)n * hw * groups;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        int pix = (int)(i % hw);
        size_t t = i / hw;
        int g = (int)(t % groups);
        int b = (int)(t / groups);
        int4 v;
        int8_t* q = reinterpret_cast<int8_t*>(&v);
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            int ch = g * 16 + k;
            q[k] = ch < c ? x[((size_t)b * c + ch) * hw + pix] : (int8_t)0;
        }
        *reinterpret_cast<int4*>(y + ((size_t)b * hw + pix) * cp + g * 16) = v;
    }
}

__global__ void unpack_nchw_int8_kernel(const int8_t* __restrict__ x, int n, int c, int hw, int cp, int8_t* __restrict__ y) {
    const int groups = cp >> 4;
    size_t total = (size_t)n * hw * groups;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        int pix = (int)(i % hw);
        size_t t = i / hw;
        int g = (int)(t % groups);
        int b = (int)(t / groups);
        int4 v = *reinterpret_cast<const int4*>(x + ((size_t)b * hw + pix) * cp + g * 16);
        const int8_t* q = reinterpret_cast<const int8_t*>(&v);
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            int ch = g * 16 + k;
            if (ch < c) y[((size_t)b * c + ch) * hw + pix] = q[k];
        }
    }
}

cudaError_t launch_float_to_int8(const float* x, int n, int c, int h, int w, float inv_scale, float zero, float minv,
                                 float maxv, int8_t* y, cudaStream_t s) {
    int cp = up16(c);
    size_t work = (size_t)n * h * w * (cp >> 4);
    float_to_int8_kernel<<<grid_for(work, 256), 256, 0, s>>>(x, n, c, h * w, cp, inv_scale, zero, minv, maxv, y);
    ++g_launch_count;
    return cudaGetLastError();
}
cudaError_t launch_int8_to_float(const int8_t* x, int n, int c, int h, int w, float scale, float zero, float* y,
                                 cudaStream_t s) {
    int cp = up16(c);
    size_t work = (size_t)n * h * w * (cp >> 4);
    int8_to_float_kernel<<<grid_for(work, 256), 256, 0, s>>>(x, n, c, h * w, cp, scale, zero, y);
    ++g_launch_count;
    return cudaGetLastError();
}
cudaError_t launch_pack_nchw_int8(const int8_t* x, int n, int c, int h, int w, int8_t* y, cudaStream_t s) {
    int cp = up16(c);
    size_t work = (size_t)n * h * w * (cp >> 4);
    pack_nchw_int8_kernel<<<grid_for(work, 256), 256, 0, s>>>(x, n, c, h * w, cp, y);
    ++g_launch_count;
    return cudaGetLastError();
}
cudaError_t launch_unpack_nchw_int8(const int8_t* x, int n, int c, int h, int w, int8_t* y, cudaStream_t s) {
    int cp = up16(c);
    size_t work = (size_t)n * h * w * (cp >> 4);
    unpack_nchw_int8_kernel<<<grid_for(work, 256), 256, 0, s>>>(x, n, c, h * w, cp, y);
    ++g_launch_count;
    return cudaGetLastError();
}

__device__ __forceinline__ int ld_nc_4(const void* p) {
    int r;
    asm volatile("ld.global.nc.s32 %0, [%1];" : "=r"(r) : "l"(p));
    return r;
}

// ---- depthwise int8 conv, generic (CPUDepthwiseConvInt8.cpp:40-100, GemmInt8_VNNI.cpp:2978-3110): one 16-channel group of
//      one output pixel per work index.  acc = bias_i32 + sum (x+128)*w [the +128*sum(w) part is pre-added to bias_i32 on the
//      host]; f = float(acc)*scale; q = trunc(f +- 0.5); clamp AFTER rounding.
__device__ __forceinline__ void dwconv_generic_work(const DwParams& p, size_t i) {
    const int groups = p.Cp >> 4;
    int g = (int)(i % groups);
    size_t t = i / groups;
    int ox = (int)(t % p.OW);
    t /= p.OW;
    int oy = (int)(t % p.OH);
    int b = (int)(t / p.OH);
    int acc[16];
    {
        const int4* bp = reinterpret_cast<const int4*>(p.bias_i32 + g * 16);
#pragma unroll
        for (int v = 0; v < 4; ++v) {
            int4 bv = bp[v];
            acc[v * 4 + 0] = bv.x; acc[v * 4 + 1] = bv.y; acc[v * 4 + 2] = bv.z; acc[v * 4 + 3] = bv.w;
        }
    }
    for (int ky = 0; ky < p.KH; ++ky) {
        int iy = oy * p.sh + ky * p.dh - p.ph;
        for (int kx = 0; kx < p.KW; ++kx) {
            int ix = ox * p.sw + kx * p.dw - p.pw;
            int4 wv = *reinterpret_cast<const int4*>(p.w + (size_t)(ky * p.KW + kx) * p.Cp + g * 16);
            const int8_t* wq = reinterpret_cast<const int8_t*>(&wv);
            if ((unsigned)iy < (unsigned)p.IH && (unsigned)ix < (unsigned)p.IW) {
                int4 xv = ld_nc_16(p.x + (((size_t)b * p.IH + iy) * p.IW + ix) * p.Cp + g * 16);
                const int8_t* xq = reinterpret_cast<const int8_t*>(&xv);
#pragma unroll
                for (int k = 0; k < 16; ++k) acc[k] += (int)xq[k] * (int)wq[k];
            } else {
#pragma unroll
                for (int k = 0; k < 16; ++k) acc[k] += p.zin * (int)wq[k];
            }
        }
    }
    int4 out;
    int8_t* oq = reinterpret_cast<int8_t*>(&out);
#pragma unroll
    for (int k = 0; k < 16; ++k) {
        int ch = g * 16 + k;
        float f = __fmul_rn(__int2float_rn(acc[k]), p.scale[ch]);
        f = __fadd_rn(f, f < 0.0f ? -0.5f : 0.5f);
        int q = __float2int_rz(f);
        q = min(q, p.maxv);
        q = max(q, p.minv);
        oq[k] = ch < p.C ? (int8_t)q : (int8_t)0;
    }
    *reinterpret_cast<int4*>(p.y + (((size_t)b * p.OH + oy) * p.OW + ox) * p.Cp + g * 16) = out;
}

// 3x3 fast path (every depthwise layer of MobileNet / most CNNs): a work index owns 4 channels (one 32-bit word per pixel) and
// TW = 4 adjacent output pixels of a row.  Every tap word is pre-split into four single-byte masks so that ONE
// dp4a(x_word, mask_c, acc_c) is the exact signed product of channel c, and the (TW-1)*S+3 input words of a row are loaded
// once for all taps and outputs.  Same accumulator and the same rounding sequence as the generic body.
// Work index space: [N][OH][xblocks = ceil(OW/4)][quads = Cp/4], quads fastest.
template <int S>
__device__ __forceinline__ void dwconv3x3_work(const DwParams& p, size_t i) {
    constexpr int TW = 4, NX = (TW - 1) * S + 3;
    const int quads = p.Cp >> 2, xblocks = (p.OW + TW - 1) / TW;
    const int cq = (int)(i % quads);
    size_t t = i / quads;
    const int xb = (int)(t % xblocks);
    t /= xblocks;
    const int oy = (int)(t % p.OH), b = (int)(t / p.OH);
    const int ox0 = xb * TW;
    int wm[9][4];
#pragma unroll
    for (int tp = 0; tp < 9; ++tp) {
        const int w = *reinterpret_cast<const int*>(p.w + (size_t)tp * p.Cp + cq * 4);
        wm[tp][0] = w & 0x000000ff; wm[tp][1] = w & 0x0000ff00; wm[tp][2] = w & 0x00ff0000; wm[tp][3] = w & 0xff000000;
    }
    const int4 bv = *reinterpret_cast<const int4*>(p.bias_i32 + cq * 4);
    int acc[TW][4];
#pragma unroll
    for (int j = 0; j < TW; ++j) { acc[j][0] = bv.x; acc[j][1] = bv.y; acc[j][2] = bv.z; acc[j][3] = bv.w; }
    const uint32_t zb = (uint32_t)(uint8_t)(int8_t)p.zin;
    const int zsplat = (int)(zb | (zb << 8) | (zb << 16) | (zb << 24));
    const int ix0 = ox0 * S - p.pw;
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
        const int iy = oy * S + ky - p.ph;
        const bool yin = (unsigned)iy < (unsigned)p.IH;
        const int8_t* row = p.x + (((size_t)b * p.IH + (yin ? iy : 0)) * p.IW) * p.Cp + cq * 4;
        int xw[NX];
#pragma unroll
        for (int c = 0; c < NX; ++c) {
            const int ix = ix0 + c;
            xw[c] = (yin && (unsigned)ix < (unsigned)p.IW) ? ld_nc_4(row + (size_t)ix * p.Cp) : zsplat;
        }
#pragma unroll
        for (int j = 0; j < TW; ++j)
#pragma unroll
            for (int kx = 0; kx < 3; ++kx)
#pragma unroll
                for (int c = 0; c < 4; ++c) acc[j][c] = __dp4a(xw[j * S + kx], wm[ky * 3 + kx][c], acc[j][c]);
    }
    const float4 sc = *reinterpret_cast<const float4*>(p.scale + cq * 4);
    const float scv[4] = {sc.x, sc.y, sc.z, sc.w};
#pragma unroll
    for (int j = 0; j < TW; ++j) {
        const int ox = ox0 + j;
        if (ox >= p.OW) break;
        uint32_t packed = 0;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            float f = __fmul_rn(__int2float_rn(acc[j][c]), scv[c]);
            f = __fadd_rn(f, f < 0.0f ? -0.5f : 0.5f);
            int q = __float2int_rz(f);
            q = min(q, p.maxv);
            q = max(q, p.minv);
            if (cq * 4 + c >= p.C) q = 0;
            packed |= (uint32_t)(q & 0xff) << (8 * c);
        }
        *reinterpret_cast<uint32_t*>(p.y + (((size_t)b * p.OH + oy) * p.OW + ox) * p.Cp + cq * 4) = packed;
    }
}
static inline bool dw_is_3x3_fast(const DwParams& p) {
    return p.KH == 3 && p.KW == 3 && p.dh == 1 && p.dw == 1 && p.sh == p.sw && (p.sh == 1 || p.sh == 2);
}

__global__ void __launch_bounds__(256) dwconv_int8_kernel(const DwParams p) {
    const int groups = p.Cp >> 4;
    size_t total = (size_t)p.N * p.OH * p.OW * groups;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x)
        dwconv_generic_work(p, i);
}
template <int S>
__global__ void __launch_bounds__(256) dwconv3x3_int8_kernel(const DwParams p) {
    const size_t total = (size_t)p.N * p.OH * ((p.OW + 3) / 4) * (p.Cp >> 2);
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= total) return;
    dwconv3x3_work<S>(p, i);
}

cudaError_t launch_dwconv_int8(const DwParams& p, cudaStream_t s) {
    if (dw_is_3x3_fast(p)) {
        const size_t work = (size_t)p.N * p.OH * ((p.OW + 3) / 4) * (p.Cp >> 2);
        const unsigned grid = (unsigned)((work + 255) / 256);
        if (p.sh == 1) dwconv3x3_int8_kernel<1><<<grid, 256, 0, s>>>(p);
        else dwconv3x3_int8_kernel<2><<<grid, 256, 0, s>>>(p);
        ++g_launch_count;
        return cudaGetLastError();
    }
    size_t work = (size_t)p.N * p.OH * p.OW * (p.Cp >> 4);
    dwconv_int8_kernel<<<grid_for(work, 256), 256, 0, s>>>(p);
    ++g_launch_count;
    return cudaGetLastError();
}

// ---- int8 eltwise add (compute/Int8FunctionsOpt.cpp:1926-1975): a = float(q0-z0)*s0; b = float(q1-z1)*s1;
//      v = (int)roundf((a+b) * inv_out) + z_out; clamp.  roundf = half away from zero.  One 16-byte chunk per work index.
struct AddParams {
    const int8_t* x0;
    const int8_t* x1;
    int8_t* y;
    float s0, s1, inv_out;
    int z0, z1, z_out, minv, maxv, c, cp;
    size_t chunks;
};
__device__ __forceinline__ void binary_add_work(const AddParams& p, size_t i) {
    const int groups = p.cp >> 4;
    int g = (int)(i % groups);
    int4 a = ld_nc_16(p.x0 + i * 16), b = ld_nc_16(p.x1 + i * 16);
    const int8_t* qa = reinterpret_cast<const int8_t*>(&a);
    const int8_t* qb = reinterpret_cast<const int8_t*>(&b);
    int4 o;
    int8_t* qo = reinterpret_cast<int8_t*>(&o);
#pragma unroll
    for (int k = 0; k < 16; ++k) {
        float fa = __fmul_rn(__int2float_rn((int)qa[k] - p.z0), p.s0);
        float fb = __fmul_rn(__int2float_rn((int)qb[k] - p.z1), p.s1);
        float t = __fmul_rn(__fadd_rn(fa, fb), p.inv_out);
        int v = (int)roundf(t);   // true half-away-from-zero on the exact value (t +- 0.5 can round up in fp32)
        v += p.z_out;
        v = min(v, p.maxv);
        v = max(v, p.minv);
        qo[k] = (g * 16 + k) < p.c ? (int8_t)v : (int8_t)0;
    }
    *reinterpret_cast<int4*>(p.y + i * 16) = o;
}
__global__ void binary_add_int8_kernel(const AddParams p) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < p.chunks; i += (size_t)gridDim.x * blockDim.x)
        binary_add_work(p, i);
}
cudaError_t launch_binary_add_int8(const int8_t* x0, float s0, int z0, const int8_t* x1, float s1, int z1, int8_t* y,
                                   float inv_out, int z_out, int minv, int maxv, size_t pixels, int c, int cp, cudaStream_t s) {
    AddParams p;
    p.x0 = x0; p.x1 = x1; p.y = y; p.s0 = s0; p.s1 = s1; p.inv_out = inv_out; p.z0 = z0; p.z1 = z1; p.z_out = z_out;
    p.minv = minv; p.maxv = maxv; p.c = c; p.cp = cp; p.chunks = pixels * (cp >> 4);
    binary_add_int8_kernel<<<grid_for(p.chunks, 256), 256, 0, s>>>(p);
    ++g_launch_count;
    return cudaGetLastError();
}

// ---- avg pooling between int8 tensors with different quant attrs = Int8ToFloat -> poolingAvg<float> -> FloatToInt8
//      (CPUPool.hpp:227-394): interior windows accumulate x*(1/count) tap by tap; border windows sum first.
__global__ void avgpool_int8_via_float_kernel(const PoolParams p) {
    const int groups = p.Cp >> 4;
    size_t total = (size_t)p.N * p.OH * p.OW * groups;
    const float z128 = __fadd_rn(p.z_in, 128.f);
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        int g = (int)(i % groups);
        size_t t = i / groups;
        int ox = (int)(t % p.OW);
        t /= p.OW;
        int oy = (int)(t % p.OH);
        int b = (int)(t / p.OH);
        int iy0 = oy * p.sh - p.ph, ix0 = ox * p.sw - p.pw;
        bool interior = iy0 >= 0 && ix0 >= 0 && iy0 + p.KH <= p.IH && ix0 + p.KW <= p.IW;
        float sum[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) sum[k] = 0.f;
        int khs = max(0, -iy0), khe = min(p.KH, p.IH - iy0), kws = max(0, -ix0), kwe = min(p.KW, p.IW - ix0);
        float div;
        if (interior) {
            div = __fdiv_rn(1.0f, (float)(p.KH * p.KW));
        } else {
            int count = p.count_type == 1 ? (min(iy0 + p.KH, p.IH + p.ph) - iy0) * (min(ix0 + p.KW, p.IW + p.pw) - ix0)
                                          : (khe - khs) * (kwe - kws);
            div = count > 0 ? __fdiv_rn(1.0f, (float)count) : 0.f;
        }
        for (int ky = khs; ky < khe; ++ky)
            for (int kx = kws; kx < kwe; ++kx) {
                int4 v = ld_nc_16(p.x + (((size_t)b * p.IH + iy0 + ky) * p.IW + ix0 + kx) * p.Cp + g * 16);
                const int8_t* q = reinterpret_cast<const int8_t*>(&v);
#pragma unroll
                for (int k = 0; k < 16; ++k) {
                    float xf = __fmul_rn(__fsub_rn(__int2float_rn((int)q[k] + 128), z128), p.s_in);
                    sum[k] = interior ? __fadd_rn(sum[k], __fmul_rn(xf, div)) : __fadd_rn(sum[k], xf);
                }
            }
        int4 o;
        int8_t* qo = reinterpret_cast<int8_t*>(&o);
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            float r = interior ? sum[k] : __fmul_rn(sum[k], div);
            int q = quant_avx512_exact(r, p.inv_out, p.z_out, p.minv, p.maxv);
            qo[k] = (g * 16 + k) < p.C ? (int8_t)q : (int8_t)0;
        }
        *reinterpret_cast<int4*>(p.y + (((size_t)b * p.OH + oy) * p.OW + ox) * p.Cp + g * 16) = o;
    }
}
// Same arithmetic, one channel per thread: a global 7x7 pool over [32][1280] has only 2560 16-channel work items, each a serial
// chain of 49 dependent loads (38 us); with 41k single-channel threads the chain length is the same but 16x more of them are in
// flight.  The per-output order of the fp32 accumulation (tap by tap) is unchanged.
__global__ void __launch_bounds__(256) avgpool_int8_via_float_1ch_kernel(const PoolParams p) {
    const size_t total = (size_t)p.N * p.OH * p.OW * p.Cp;
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= total) return;
    const float z128 = __fadd_rn(p.z_in, 128.f);
    const int ch = (int)(i % p.Cp);
    size_t t = i / p.Cp;
    const int ox = (int)(t % p.OW);
    t /= p.OW;
    const int oy = (int)(t % p.OH), b = (int)(t / p.OH);
    const int iy0 = oy * p.sh - p.ph, ix0 = ox * p.sw - p.pw;
    const bool interior = iy0 >= 0 && ix0 >= 0 && iy0 + p.KH <= p.IH && ix0 + p.KW <= p.IW;
    const int khs = max(0, -iy0), khe = min(p.KH, p.IH - iy0), kws = max(0, -ix0), kwe = min(p.KW, p.IW - ix0);
    float div;
    if (interior) {
        div = __fdiv_rn(1.0f, (float)(p.KH * p.KW));
    } else {
        int count = p.count_type == 1 ? (min(iy0 + p.KH, p.IH + p.ph) - iy0) * (min(ix0 + p.KW, p.IW + p.pw) - ix0)
                                      : (khe - khs) * (kwe - kws);
        div = count > 0 ? __fdiv_rn(1.0f, (float)count) : 0.f;
    }
    float sum = 0.f;
    for (int ky = khs; ky < khe; ++ky)
        for (int kx = kws; kx < kwe; ++kx) {
            const int q = p.x[(((size_t)b * p.IH + iy0 + ky) * p.IW + ix0 + kx) * p.Cp + ch];
            const float xf = __fmul_rn(__fsub_rn(__int2float_rn(q + 128), z128), p.s_in);
            sum = interior ? __fadd_rn(sum, __fmul_rn(xf, div)) : __fadd_rn(sum, xf);
        }
    const float r = interior ? sum : __fmul_rn(sum, div);
    const int q = quant_avx512_exact(r, p.inv_out, p.z_out, p.minv, p.maxv);
    p.y[(((size_t)b * p.OH + oy) * p.OW + ox) * p.Cp + ch] = ch < p.C ? (int8_t)q : (int8_t)0;
}

cudaError_t launch_avgpool_int8_via_float(const PoolParams& p, cudaStream_t s) {
    size_t work = (size_t)p.N * p.OH * p.OW * (p.Cp >> 4);
    if (work < 64 * 1024) {      // few outputs, long windows: go wide
        const size_t threads = work * 16;
        avgpool_int8_via_float_1ch_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, s>>>(p);
        ++g_launch_count;
        return cudaGetLastError();
    }
    avgpool_int8_via_float_kernel<<<grid_for(work, 128), 128, 0, s>>>(p);
    ++g_launch_count;
    return cudaGetLastError();
}

// ---- fp32 pooling on NCHW tensors (the float Pooling the pipeline leaves between Int8ToFloat / FloatToInt8 casts when the
//      quant attrs of input and output differ): CPUPool.hpp:227-394 poolingAvg<float> / poolingMax<float> order of operations.
__global__ void pool_f32_kernel(const PoolParams p, const float* __restrict__ x, float* __restrict__ y, int is_avg) {
    size_t total = (size_t)p.N * p.C * p.OH * p.OW;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        int ox = (int)(i % p.OW);
        size_t t = i / p.OW;
        int oy = (int)(t % p.OH);
        size_t bc = t / p.OH;
        const float* xp = x + bc * p.IH * p.IW;
        int iy0 = oy * p.sh - p.ph, ix0 = ox * p.sw - p.pw;
        bool interior = iy0 >= 0 && ix0 >= 0 && iy0 + p.KH <= p.IH && ix0 + p.KW <= p.IW;
        int khs = max(0, -iy0), khe = min(p.KH, p.IH - iy0), kws = max(0, -ix0), kwe = min(p.KW, p.IW - ix0);
        float r;
        if (is_avg) {
            float div;
            if (interior) {
                div = __fdiv_rn(1.0f, (float)(p.KH * p.KW));
            } else {
                int count = p.count_type == 1 ? (min(iy0 + p.KH, p.IH + p.ph) - iy0) * (min(ix0 + p.KW, p.IW + p.pw) - ix0)
                                              : (khe - khs) * (kwe - kws);
                div = count > 0 ? __fdiv_rn(1.0f, (float)count) : 0.f;
            }
            float sum = 0.f;
            for (int ky = khs; ky < khe; ++ky)
                for (int kx = kws; kx < kwe; ++kx) {
                    float xf = xp[(size_t)(iy0 + ky) * p.IW + ix0 + kx];
                    sum = interior ? __fadd_rn(sum, __fmul_rn(xf, div)) : __fadd_rn(sum, xf);
                }
            r = interior ? sum : __fmul_rn(sum, div);
        } else {
            // pooling_max_pad (CPUPool.hpp:19-51) reads the edge row / column for a tap in the padding, so a window wholly in
            // the padding (large pads, ceil mode) takes its edge's maximum; the reduction starts at VEC(-16777216) and takes
            // each tap as VEC::max(max, tap), maxps: the tap unless the running max is strictly greater (a NaN is replaced by
            // the next tap, of -0 and +0 the later one stays)
            // the taps in the CPU's order, an edge tap read again for each padded tap it stands for
            r = -16777216.f;
            for (int ky = 0; ky < p.KH; ++ky) {
                const int yy = min(max(iy0 + ky, 0), p.IH - 1);
                for (int kx = 0; kx < p.KW; ++kx) {
                    const float v = xp[(size_t)yy * p.IW + min(max(ix0 + kx, 0), p.IW - 1)];
                    r = r > v ? r : v;
                }
            }
        }
        y[i] = r;
    }
}
cudaError_t launch_pool_f32(const PoolParams& p, const float* x, float* y, int is_avg, cudaStream_t s) {
    size_t work = (size_t)p.N * p.C * p.OH * p.OW;
    pool_f32_kernel<<<grid_for(work, 256), 256, 0, s>>>(p, x, y, is_avg);
    ++g_launch_count;
    return cudaGetLastError();
}

// ---- batched 2-D transpose of 4-byte elements: dst[b][c][r] = src[b][r][c] (32 x 32 smem tiles, both sides coalesced).
//      The MNN tensor of an LLM linear layer is [N][C][tokens] (NC4HW4 format, stored NCHW-linear here); the W8A8 GEMM wants
//      token-major rows.
__global__ void transpose_b32_kernel(const uint32_t* __restrict__ src, uint32_t* __restrict__ dst, int rows, int cols) {
    __shared__ uint32_t tile[32][33];
    const uint32_t* s = src + (size_t)blockIdx.z * rows * cols;
    uint32_t* d = dst + (size_t)blockIdx.z * rows * cols;
    const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
    for (int i = threadIdx.y; i < 32; i += 8) {
        int r = r0 + i, c = c0 + threadIdx.x;
        if (r < rows && c < cols) tile[i][threadIdx.x] = s[(size_t)r * cols + c];
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += 8) {
        int c = c0 + i, r = r0 + threadIdx.x;
        if (r < rows && c < cols) d[(size_t)c * rows + r] = tile[threadIdx.x][i];
    }
}
cudaError_t launch_transpose_b32(const void* src, void* dst, int batch, int rows, int cols, cudaStream_t s) {
    dim3 grid((cols + 31) / 32, (rows + 31) / 32, batch), block(32, 8);
    transpose_b32_kernel<<<grid, block, 0, s>>>((const uint32_t*)src, (uint32_t*)dst, rows, cols);
    ++g_launch_count;
    return cudaGetLastError();
}

// ---- Raster: 3-level strided region copies between 4-byte-element tensors in their linear (NCHW / NHWC) layout
//      (Tensor::InsideDescribe::Region, source/core/TensorUtils.hpp:45-52; CPURaster.cpp executeFaster / blit).
__global__ void raster_b32_kernel(const RasterRegion r, const uint32_t* __restrict__ src, uint32_t* __restrict__ dst) {
    size_t total = (size_t)r.size[0] * r.size[1] * r.size[2];
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        int k = (int)(i % r.size[2]);
        size_t t = i / r.size[2];
        int j = (int)(t % r.size[1]);
        int a = (int)(t / r.size[1]);
        dst[(size_t)r.dst_offset + (size_t)a * r.dst_stride[0] + (size_t)j * r.dst_stride[1] + (size_t)k * r.dst_stride[2]] =
            src[(size_t)r.src_offset + (size_t)a * r.src_stride[0] + (size_t)j * r.src_stride[1] + (size_t)k * r.src_stride[2]];
    }
}
cudaError_t launch_raster_b32(const RasterRegion& r, const void* src, void* dst, cudaStream_t s) {
    size_t work = (size_t)r.size[0] * r.size[1] * r.size[2];
    if (work == 0) return cudaSuccess;
    raster_b32_kernel<<<grid_for(work, 256), 256, 0, s>>>(r, (const uint32_t*)src, (uint32_t*)dst);
    ++g_launch_count;
    return cudaGetLastError();
}

// ---- softmax over the channel axis of an int8 [rows][cp] tensor (CPUSoftmax.cpp:85-150, int8 mode):
//      dequantise, fp32 softmax, requantise.  One CTA per row.
__global__ void __launch_bounds__(256) softmax_int8_kernel(const int8_t* __restrict__ x, int c, int cp, float s_in, float z_in,
                                                           float inv_out, float z_out, float minv, float maxv,
                                                           int8_t* __restrict__ y) {
    __shared__ float red[8];
    __shared__ float bc;
    const int8_t* xr = x + (size_t)blockIdx.x * cp;
    int8_t* yr = y + (size_t)blockIdx.x * cp;
    const float z128 = __fadd_rn(z_in, 128.f);
    auto deq = [&](int k) { return __fmul_rn(__fsub_rn(__int2float_rn((int)xr[k] + 128), z128), s_in); };
    float mx = -3.4e38f;
    for (int k = threadIdx.x; k < c; k += blockDim.x) mx = fmaxf(mx, deq(k));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x == 0) { float m = red[0]; for (int i = 1; i < 8; ++i) m = fmaxf(m, red[i]); bc = m; }
    __syncthreads();
    mx = bc;
    float sum = 0.f;
    for (int k = threadIdx.x; k < c; k += blockDim.x) sum += expf(deq(k) - mx);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
    __syncthreads();
    if (threadIdx.x == 0) { float t = 0.f; for (int i = 0; i < 8; ++i) t += red[i]; bc = __fdiv_rn(1.0f, t); }
    __syncthreads();
    const float rs = bc;
    for (int k = threadIdx.x; k < cp; k += blockDim.x) {
        int q = 0;
        if (k < c) q = quant_avx512_exact(__fmul_rn(expf(deq(k) - mx), rs), inv_out, z_out, minv, maxv);
        yr[k] = (int8_t)q;
    }
}
cudaError_t launch_softmax_int8(const int8_t* x, int rows, int c, int cp, float s_in, float z_in, float inv_out, float z_out,
                                float minv, float maxv, int8_t* y, cudaStream_t s) {
    softmax_int8_kernel<<<rows, 256, 0, s>>>(x, c, cp, s_in, z_in, inv_out, z_out, minv, maxv, y);
    ++g_launch_count;
    return cudaGetLastError();
}

// ---- dynamic per-token activation quantisation, one CTA per token
//      (MNNAbsMax + MNNQuantScaleFP32 compute/CommonOptFunction.cpp:79-94, 310-330;
//       _AVX512_DynamicQuant x86_x64/avx512/PackedFunction.cpp:288-348: x*qscale, round-to-nearest-even)
//      also emits srcsum[token] = float(sum_k (xq_k + 128)) * dq (MNNSumByAxisLForMatmul_A,
//      compute/Int8FunctionsOpt.cpp:2584-2650) for the asymmetric-weight term.
//      bs > 0 (K-blocked weight scales): xsb[token][b] = float(sum_{k in block b} (xq_k + 128)) * dq per block of bs channels,
//      the block's share of srcsum, summed from the quantised row this CTA has just written (visible after __syncthreads)
__device__ __forceinline__ void quant_block_sums(const int8_t* qr, int ic, int bs, float dqv, float* xsb) {
    for (int b = threadIdx.x; b * bs < ic; b += blockDim.x) {
        const int4* q4 = reinterpret_cast<const int4*>(qr + (size_t)b * bs);
        int s = 0;
        for (int i = 0; i < (bs >> 4); ++i) {
            const int4 v = q4[i];
            s = __dp4a(v.x, 0x01010101, s); s = __dp4a(v.y, 0x01010101, s);
            s = __dp4a(v.z, 0x01010101, s); s = __dp4a(v.w, 0x01010101, s);
        }
        xsb[b] = __fmul_rn(__int2float_rn(s + 128 * bs), dqv);
    }
}

__global__ void __launch_bounds__(256) dynamic_quant_kernel(const float* __restrict__ x, int ic, int icp,
                                                            int8_t* __restrict__ xq, float* __restrict__ dq,
                                                            float* __restrict__ srcsum, int bs, float* __restrict__ xsb) {
    __shared__ float s_max[8];
    __shared__ int s_sum[8];
    const int tkn = blockIdx.x;
    const float* xr = x + (size_t)tkn * ic;
    float amax = 0.f;
    for (int k = threadIdx.x; k < ic; k += blockDim.x) amax = fmaxf(amax, fabsf(xr[k]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = amax;
    __syncthreads();
    amax = s_max[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) amax = fmaxf(amax, s_max[i]);
    float qs = 1.f, dqv = 1.f;
    if (!((double)amax < 1e-7)) {
        qs = __fdiv_rn(127.0f, amax);
        dqv = __fdiv_rn(amax, 127.0f);
    }
    int lsum = 0;
    int8_t* qr = xq + (size_t)tkn * icp;
    for (int k = threadIdx.x; k < icp; k += blockDim.x) {
        int q = 0;
        if (k < ic) {
            q = __float2int_rn(__fmul_rn(xr[k], qs));
            lsum += q + 128;
        }
        qr[k] = (int8_t)q;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) lsum += __shfl_xor_sync(0xffffffffu, lsum, o);
    if ((threadIdx.x & 31) == 0) s_sum[threadIdx.x >> 5] = lsum;
    __syncthreads();
    if (threadIdx.x == 0) {
        int tot = 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) tot += s_sum[i];
        dq[tkn] = dqv;
        srcsum[tkn] = __fmul_rn(__int2float_rn(tot), dqv);
    }
    if (bs) quant_block_sums(xq + (size_t)tkn * icp, ic, bs, dqv, xsb + (size_t)tkn * (ic / bs));
}

// Same arithmetic, one pass over HBM: the token's row stays in registers between the abs-max and the quantise step
// (float4 loads, packed 4-byte stores).  ic % 4 == 0, ic <= 1024 * NV.
template <int NV>
__global__ void __launch_bounds__(256) dynamic_quant_vec_kernel(const float* __restrict__ x, int ic, int icp,
                                                                int8_t* __restrict__ xq, float* __restrict__ dq,
                                                                float* __restrict__ srcsum, int bs, float* __restrict__ xsb) {
    __shared__ float s_max[8];
    __shared__ int s_sum[8];
    const int tkn = blockIdx.x;
    const float4* xr = reinterpret_cast<const float4*>(x + (size_t)tkn * ic);
    const int n4 = ic >> 2, np4 = icp >> 2;
    float4 v[NV];
    float amax = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const int idx = threadIdx.x + i * 256;
        v[i] = idx < n4 ? __ldg(xr + idx) : make_float4(0.f, 0.f, 0.f, 0.f);
        amax = fmaxf(amax, fmaxf(fmaxf(fabsf(v[i].x), fabsf(v[i].y)), fmaxf(fabsf(v[i].z), fabsf(v[i].w))));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = amax;
    __syncthreads();
    amax = s_max[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) amax = fmaxf(amax, s_max[i]);
    float qs = 1.f, dqv = 1.f;
    if (!((double)amax < 1e-7)) {
        qs = __fdiv_rn(127.0f, amax);
        dqv = __fdiv_rn(amax, 127.0f);
    }
    int lsum = 0;
    uint32_t* qr = reinterpret_cast<uint32_t*>(xq + (size_t)tkn * icp);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const int idx = threadIdx.x + i * 256;
        if (idx < np4) {
            uint32_t packed = 0;
            if (idx < n4) {
                const int q0 = __float2int_rn(__fmul_rn(v[i].x, qs)), q1 = __float2int_rn(__fmul_rn(v[i].y, qs));
                const int q2 = __float2int_rn(__fmul_rn(v[i].z, qs)), q3 = __float2int_rn(__fmul_rn(v[i].w, qs));
                lsum += q0 + q1 + q2 + q3 + 512;
                packed = (uint32_t)(q0 & 0xff) | ((uint32_t)(q1 & 0xff) << 8) | ((uint32_t)(q2 & 0xff) << 16) | ((uint32_t)(q3 & 0xff) << 24);
            }
            qr[idx] = packed;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) lsum += __shfl_xor_sync(0xffffffffu, lsum, o);
    if ((threadIdx.x & 31) == 0) s_sum[threadIdx.x >> 5] = lsum;
    __syncthreads();
    if (threadIdx.x == 0) {
        int tot = 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) tot += s_sum[i];
        dq[tkn] = dqv;
        srcsum[tkn] = __fmul_rn(__int2float_rn(tot), dqv);
    }
    if (bs) quant_block_sums(xq + (size_t)tkn * icp, ic, bs, dqv, xsb + (size_t)tkn * (ic / bs));
}

cudaError_t launch_dynamic_quant(const float* x, int tokens, int ic, int icp, int8_t* xq, float* dq, float* srcsum,
                                 cudaStream_t s, int bs, float* xsb) {
    const bool vec = (ic & 3) == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0;
    if (vec && icp <= 1024 * 2) dynamic_quant_vec_kernel<2><<<tokens, 256, 0, s>>>(x, ic, icp, xq, dq, srcsum, bs, xsb);
    else if (vec && icp <= 1024 * 4) dynamic_quant_vec_kernel<4><<<tokens, 256, 0, s>>>(x, ic, icp, xq, dq, srcsum, bs, xsb);
    else if (vec && icp <= 1024 * 8) dynamic_quant_vec_kernel<8><<<tokens, 256, 0, s>>>(x, ic, icp, xq, dq, srcsum, bs, xsb);
    else
    dynamic_quant_kernel<<<tokens, 256, 0, s>>>(x, ic, icp, xq, dq, srcsum, bs, xsb);
    ++g_launch_count;
    return cudaGetLastError();
}

}  // namespace mnnb200

// =================================================================================================================
// Round 2: the remaining ops of an int8 ResNet-50 .mnn (SURVEY F13): int8 Scale, int8 Pooling with equal quant attrs,
// float ReLU and float Reduction.
// =================================================================================================================
namespace mnnb200 {

// ---- int8 Scale (CPUScaleInt8.cpp:60-122 + MNNScaleAndAddBiasInt8, compute/Int8FunctionsOpt.cpp:2207-2252), pure integer:
//      val = (q - z_in) * alpha[c] + bias[c];  out = trunc((val +- 2^14) / 2^15) + z_out;  clamp.  alpha/bias are the 15-bit
//      fixed-point constants the host folds at resize time.
__global__ void scale_int8_kernel(const int8_t* __restrict__ x, int8_t* __restrict__ y, const int32_t* __restrict__ alpha,
                                  const int32_t* __restrict__ bias, int z_in, int z_out, int minv, int maxv, size_t chunks, int c,
                                  int cp) {
    const int groups = cp >> 4;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < chunks; i += (size_t)gridDim.x * blockDim.x) {
        const int g = (int)(i % groups);
        int4 a = ld_nc_16(x + i * 16);
        const int8_t* q = reinterpret_cast<const int8_t*>(&a);
        int4 o;
        int8_t* qo = reinterpret_cast<int8_t*>(&o);
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            const int ch = g * 16 + k;
            int v = 0;
            if (ch < c) {
                const int val = ((int)q[k] - z_in) * __ldg(alpha + ch) + __ldg(bias + ch);
                v = (val < 0 ? (val - (1 << 14)) : (val + (1 << 14))) / (1 << 15) + z_out;   // C division truncates toward zero
                v = min(v, maxv);
                v = max(v, minv);
            }
            qo[k] = (int8_t)v;
        }
        *reinterpret_cast<int4*>(y + i * 16) = o;
    }
}
cudaError_t launch_scale_int8(const int8_t* x, int8_t* y, const int32_t* alpha, const int32_t* bias, int z_in, int z_out, int minv,
                              int maxv, size_t pixels, int c, int cp, cudaStream_t s) {
    const size_t chunks = pixels * (cp >> 4);
    scale_int8_kernel<<<grid_for(chunks, 256), 256, 0, s>>>(x, y, alpha, bias, z_in, z_out, minv, maxv, chunks, c, cp);
    ++g_launch_count;
    return cudaGetLastError();
}

// ---- int8 pooling between tensors with EQUAL quant attrs (CPUPoolInt8.cpp:19-100 with the x86 kernels,
//      x86_x64/FunctionDispatcher.cpp:122-168): both work on the uint8 storage q + 128.
//      avg: ((sum of stored bytes) * floor(2^24 / count)) >> 24, count = the valid window;
//      max: the stored bytes are compared as SIGNED int8 (not a true maximum for mixed-sign windows) -- restated as it is.
__global__ void pool_int8_x86_kernel(const PoolParams p, int is_avg) {
    const int groups = p.Cp >> 4;
    const size_t total = (size_t)p.N * p.OH * p.OW * groups;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int g = (int)(i % groups);
        size_t t = i / groups;
        const int ox = (int)(t % p.OW);
        t /= p.OW;
        const int oy = (int)(t % p.OH);
        const int b = (int)(t / p.OH);
        const int iy0 = oy * p.sh - p.ph, ix0 = ox * p.sw - p.pw;
        const int ys = max(iy0, 0), ye = min(iy0 + p.KH, p.IH), xs = max(ix0, 0), xe = min(ix0 + p.KW, p.IW);
        unsigned int sum[16];
        int best[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) { sum[k] = 0u; best[k] = -128; }
        for (int yy = ys; yy < ye; ++yy)
            for (int xx = xs; xx < xe; ++xx) {
                int4 v = ld_nc_16(p.x + (((size_t)b * p.IH + yy) * p.IW + xx) * p.Cp + g * 16);
                const int8_t* q = reinterpret_cast<const int8_t*>(&v);
#pragma unroll
                for (int k = 0; k < 16; ++k) {
                    const unsigned int u = (unsigned int)((int)q[k] + 128);          // stored byte
                    sum[k] += u;
                    const int sgn = (int)(int8_t)(uint8_t)u;                          // ... read as signed
                    best[k] = sgn > best[k] ? sgn : best[k];
                }
            }
        const int count = (ye - ys) * (xe - xs);
        const unsigned int f = count > 0 ? (unsigned int)((1 << 24) / count) : 0u;
        int4 o;
        int8_t* qo = reinterpret_cast<int8_t*>(&o);
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            const unsigned int out_u = is_avg ? (((sum[k] * f) >> 24) & 0xffu) : (unsigned int)(uint8_t)best[k];
            qo[k] = (g * 16 + k) < p.C ? (int8_t)((int)out_u - 128) : (int8_t)0;
        }
        *reinterpret_cast<int4*>(p.y + i * 16) = o;
    }
}
cudaError_t launch_pool_int8_x86(const PoolParams& p, int is_avg, cudaStream_t s) {
    const size_t total = (size_t)p.N * p.OH * p.OW * (p.Cp >> 4);
    pool_int8_x86_kernel<<<grid_for(total, 128), 128, 0, s>>>(p, is_avg);
    ++g_launch_count;
    return cudaGetLastError();
}

// ---- float ReLU (CPURelu.cpp / MNNReluWithSlope): y = x < 0 ? x * slope : x
__global__ void relu_f32_kernel(const float* __restrict__ x, float* __restrict__ y, size_t n, float slope) {
    const size_t n4 = n >> 2;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
        float4 v = reinterpret_cast<const float4*>(x)[i];
        v.x = v.x < 0.f ? __fmul_rn(v.x, slope) : v.x;
        v.y = v.y < 0.f ? __fmul_rn(v.y, slope) : v.y;
        v.z = v.z < 0.f ? __fmul_rn(v.z, slope) : v.z;
        v.w = v.w < 0.f ? __fmul_rn(v.w, slope) : v.w;
        reinterpret_cast<float4*>(y)[i] = v;
    }
    if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
        const size_t i = (n4 << 2) + threadIdx.x;
        const float v = x[i];
        y[i] = v < 0.f ? __fmul_rn(v, slope) : v;
    }
}
cudaError_t launch_relu_f32(const float* x, float* y, size_t n, float slope, cudaStream_t s) {
    relu_f32_kernel<<<grid_for((n >> 2) + 1, 256), 256, 0, s>>>(x, y, n, slope);
    ++g_launch_count;
    return cudaGetLastError();
}

// ---- float Reduction over the middle axis of [outside][axis][inside] (CPUReduction.cpp: sum / mean / max / min / prod).
//      One thread per (outside, inside) when inside > 1 (coalesced along inside); one warp per row when inside == 1.
//      op: 0 SUM, 1 MEAN, 2 MAX, 3 MIN, 4 PROD.  SUM / MEAN / PROD: fp32 accumulation in another order than the CPU's SIMD order.
//      MAX / MIN restate CPUReduction.cpp:297-318 (`float Max = srcInside[0]; ... Max = std::max(Max, srcInside[a * inside])`,
//      MinReduce alike): the row's first element, then a value replaces it only when strictly greater (smaller), so a row of -inf
//      gives -inf, a NaN is kept only when it comes first, and of equal values (-0 and +0) the first one stays.
__device__ __forceinline__ float red_combine(float a, float b, int op) {
    return op <= 1 ? a + b : a * b;
}
__device__ __forceinline__ bool red_better(float v, float best, int op) {
    return op == 2 ? best < v : v < best;
}
__global__ void reduce_f32_kernel(const float* __restrict__ x, float* __restrict__ y, int outside, int axis, int inside, int op) {
    const float init = op <= 1 ? 0.f : 1.f;
    if (inside == 1) {
        const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
        if (warp >= outside) return;
        const float* xp = x + (size_t)warp * axis;
        if (op >= 2 && op <= 3) {
            // each lane keeps its first best non-NaN value and its index; the lanes' bests merge by value, then by index
            float best = 0.f;
            int idx = axis;
            for (int a = lane; a < axis; a += 32) {
                const float v = xp[a];
                if (v == v && (idx == axis || red_better(v, best, op))) { best = v; idx = a; }
            }
            for (int o = 16; o > 0; o >>= 1) {
                const float ov = __shfl_xor_sync(0xffffffffu, best, o);
                const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
                if (oi < axis && (idx == axis || red_better(ov, best, op) || (!red_better(best, ov, op) && oi < idx))) {
                    best = ov;
                    idx = oi;
                }
            }
            if (lane == 0) y[warp] = (xp[0] != xp[0] || idx == axis) ? xp[0] : best;
            return;
        }
        float acc = init;
        for (int a = lane; a < axis; a += 32) acc = red_combine(acc, xp[a], op);
        for (int o = 16; o > 0; o >>= 1) acc = red_combine(acc, __shfl_xor_sync(0xffffffffu, acc, o), op);
        if (lane == 0) y[warp] = op == 1 ? acc / (float)axis : acc;
        return;
    }
    const size_t total = (size_t)outside * inside;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t o = i / inside, in = i - o * inside;
        const float* xp = x + o * axis * inside + in;
        float acc;
        if (op >= 2 && op <= 3) {
            acc = xp[0];
            for (int a = 1; a < axis; ++a) {
                const float v = xp[(size_t)a * inside];
                if (red_better(v, acc, op)) acc = v;
            }
        } else {
            acc = init;
            for (int a = 0; a < axis; ++a) acc = red_combine(acc, xp[(size_t)a * inside], op);
        }
        y[i] = op == 1 ? acc / (float)axis : acc;
    }
}
cudaError_t launch_reduce_f32(const float* x, float* y, int outside, int axis, int inside, int op, cudaStream_t s) {
    if (inside == 1) {
        const int blocks = (outside * 32 + 255) / 256;
        reduce_f32_kernel<<<blocks, 256, 0, s>>>(x, y, outside, axis, inside, op);
    } else {
        reduce_f32_kernel<<<grid_for((size_t)outside * inside, 256), 256, 0, s>>>(x, y, outside, axis, inside, op);
    }
    ++g_launch_count;
    return cudaGetLastError();
}

// ---- fp32 depthwise conv (CPUConvolutionDepthwise): one thread per output element, NCHW (consecutive threads walk a row of the
//      output plane, so reads along the input row coalesce for stride 1); bias, then ReLU / ReLU6 (CPUConvolution.cpp:289-291)
__global__ void __launch_bounds__(256) dwconv_f32_kernel(const DwF32Params p) {
    const size_t total = (size_t)p.N * p.C * p.OH * p.OW;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int ow = (int)(i % p.OW);
        const size_t r = i / p.OW;
        const int oh = (int)(r % p.OH);
        const size_t nc = r / p.OH;
        const int c = (int)(nc % p.C);
        const float* xp = p.x + nc * p.IH * p.IW;
        const float* wp = p.w + (size_t)c * p.KH * p.KW;
        const int ih0 = oh * p.sh - p.ph, iw0 = ow * p.sw - p.pw;
        float acc = 0.f;
        for (int kh = 0; kh < p.KH; ++kh) {
            const int ih = ih0 + kh * p.dh;
            if ((unsigned)ih >= (unsigned)p.IH) continue;
            for (int kw = 0; kw < p.KW; ++kw) {
                const int iw = iw0 + kw * p.dw;
                if ((unsigned)iw < (unsigned)p.IW) acc = fmaf(xp[(size_t)ih * p.IW + iw], wp[kh * p.KW + kw], acc);
            }
        }
        float v = acc + p.bias[c];
        if (p.act >= 1) v = fmaxf(v, 0.f);
        if (p.act == 2) v = fminf(v, 6.f);
        p.y[i] = v;
    }
}
cudaError_t launch_dwconv_f32(const DwF32Params& p, cudaStream_t s) {
    dwconv_f32_kernel<<<grid_for((size_t)p.N * p.C * p.OH * p.OW, 256), 256, 0, s>>>(p);
    ++g_launch_count;
    return cudaGetLastError();
}

// ---- fp32 BinaryOp (CPUBinary + MNNSelectBinaryFunctionForFloat): y = a op b, then ReLU when relu != 0 (activationType 1).
//      a and b are either n elements or ONE element (read on the device: a runtime scalar may change between graph replays).
//      Every op is a single IEEE operation in round-to-nearest (no FMA contraction): bit-identical to the CPU's float path.
//      float4 when the full-size operands and the output are 16-byte aligned.  y may be a (Eltwise folds inputs into its output),
//      so the pointers are not __restrict__.
template <int OP>
__device__ __forceinline__ float binary_f32_op(float a, float b) {
    if (OP == kBinaryAdd) return __fadd_rn(a, b);
    if (OP == kBinarySub) return __fsub_rn(a, b);
    if (OP == kBinaryMul) return __fmul_rn(a, b);
    if (OP == kBinaryRealDiv) return __fdiv_rn(a, b);
    // x86 minps / maxps, which the CPU's VecBinaryMin / VecBinaryMax run (BinaryUtils.hpp:335-347, Vec::min / Vec::max):
    // the second operand unless the first is strictly smaller (greater), so MIN(-0, +0) = +0, MIN(NaN, 1) = 1, MIN(1, NaN) = NaN
    if (OP == kBinaryMinimum) return a < b ? a : b;
    if (OP == kBinaryMaximum) return a > b ? a : b;
    const float d = __fsub_rn(a, b);   // kBinarySquaredDifference
    return __fmul_rn(d, d);
}
template <int OP>
__device__ __forceinline__ float binary_f32_one(float a, float b, int relu) {
    // activationType 1 is CPURelu(0) over the output (CPUBinary.cpp:36-37, MNNReluWithSlopeChannel): x < 0 ? x * 0 : x, so a
    // negative result becomes -0, -inf becomes NaN and NaN stays NaN
    const float v = binary_f32_op<OP>(a, b);
    return relu && v < 0.f ? __fmul_rn(v, 0.f) : v;
}
template <int OP>
__global__ void binary_f32_kernel(const float* a, const float* b, float* y, size_t n, int a_one, int b_one, int relu, int vec) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    const size_t i0 = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    const float sa = a_one ? a[0] : 0.f, sb = b_one ? b[0] : 0.f;
    size_t done = 0;
    if (vec) {
        const size_t n4 = n >> 2;
        for (size_t i = i0; i < n4; i += stride) {
            const float4 u = a_one ? make_float4(sa, sa, sa, sa) : reinterpret_cast<const float4*>(a)[i];
            const float4 v = b_one ? make_float4(sb, sb, sb, sb) : reinterpret_cast<const float4*>(b)[i];
            reinterpret_cast<float4*>(y)[i] = make_float4(binary_f32_one<OP>(u.x, v.x, relu), binary_f32_one<OP>(u.y, v.y, relu),
                                                          binary_f32_one<OP>(u.z, v.z, relu), binary_f32_one<OP>(u.w, v.w, relu));
        }
        done = n4 << 2;
    }
    for (size_t i = done + i0; i < n; i += stride) y[i] = binary_f32_one<OP>(a_one ? sa : a[i], b_one ? sb : b[i], relu);
}
bool binary_f32_supported(int op) {
    return op == kBinaryAdd || op == kBinarySub || op == kBinaryMul || op == kBinaryRealDiv || op == kBinaryMinimum ||
           op == kBinaryMaximum || op == kBinarySquaredDifference;
}
cudaError_t launch_binary_f32(int op, const float* a, bool a_one, const float* b, bool b_one, float* y, size_t n, int relu,
                              cudaStream_t s) {
    const uintptr_t full = (a_one ? 0 : (uintptr_t)a) | (b_one ? 0 : (uintptr_t)b) | (uintptr_t)y;
    const int vec = (full & 15) == 0;
    const int grid = grid_for(vec ? (n >> 2) + 1 : n, 256);
    switch (op) {
        case kBinaryAdd: binary_f32_kernel<kBinaryAdd><<<grid, 256, 0, s>>>(a, b, y, n, a_one, b_one, relu, vec); break;
        case kBinarySub: binary_f32_kernel<kBinarySub><<<grid, 256, 0, s>>>(a, b, y, n, a_one, b_one, relu, vec); break;
        case kBinaryMul: binary_f32_kernel<kBinaryMul><<<grid, 256, 0, s>>>(a, b, y, n, a_one, b_one, relu, vec); break;
        case kBinaryRealDiv: binary_f32_kernel<kBinaryRealDiv><<<grid, 256, 0, s>>>(a, b, y, n, a_one, b_one, relu, vec); break;
        case kBinaryMinimum: binary_f32_kernel<kBinaryMinimum><<<grid, 256, 0, s>>>(a, b, y, n, a_one, b_one, relu, vec); break;
        case kBinaryMaximum: binary_f32_kernel<kBinaryMaximum><<<grid, 256, 0, s>>>(a, b, y, n, a_one, b_one, relu, vec); break;
        case kBinarySquaredDifference:
            binary_f32_kernel<kBinarySquaredDifference><<<grid, 256, 0, s>>>(a, b, y, n, a_one, b_one, relu, vec);
            break;
        default: return cudaErrorInvalidValue;
    }
    ++g_launch_count;
    return cudaGetLastError();
}
cudaError_t launch_binary_add_f32(const float* a, const float* b, float* y, size_t n, cudaStream_t s) {
    return launch_binary_f32(kBinaryAdd, a, false, b, false, y, n, 0, s);
}

// ---- fp32 UnaryOp (CPUUnary::selectForFloat, CPUUnary.cpp:353-440).  HARDSWISH, ABS, NEG, SQUARE, SQRT, RSQRT and RECIPROCAL
//      use the CPU's own formula in round-to-nearest steps; the transcendental ops (the CPU uses its own polynomials) are
//      accurate to a few ulp: SIGMOID / SILU / GELU through expf in a cancellation-free form (times_sigmoid, activations.cuh),
//      GELU_STANDARD through erfcf.
template <int OP>
__device__ __forceinline__ float unary_f32_op(float x) {
    // ABS is MNNReluWithSlope(x, -1) (CPUUnary.cpp:323-325): (x < 0 ? x * -1 : 0) + (x >= 0 ? x : 0), so |-0| = +0 and
    // |NaN| = +0; NEG is x * -1 + 0 (CPUUnary.cpp:47-49, MNNScaleAndAddBiasScalar), so -(+0) = +0
    if (OP == kUnaryAbs) return x < 0.f ? -x : (x >= 0.f ? __fadd_rn(0.f, x) : 0.f);
    if (OP == kUnaryNeg) return __fadd_rn(-x, 0.f);
    if (OP == kUnarySquare) return __fmul_rn(x, x);
    if (OP == kUnarySqrt) return __fsqrt_rn(x);
    if (OP == kUnaryRsqrt) return __fdiv_rn(1.f, __fsqrt_rn(x));
    if (OP == kUnaryReciprocal) return __fdiv_rn(1.f, x);
    if (OP == kUnaryExp) return expf(x);
    if (OP == kUnaryLog) return logf(x);
    if (OP == kUnaryTanh) return tanh_f32(x);
    if (OP == kUnarySigmoid) return sigmoid_f32(x);
    if (OP == kUnarySilu) return times_sigmoid(x, x);
    if (OP == kUnaryHardSwish)   // x86_x64/sse/MathFunctions.cpp:251-259: (x * min(max(x + 3, 0), 6)) / 6
        return __fdiv_rn(__fmul_rn(x, fminf(fmaxf(__fadd_rn(x, 3.f), 0.f), 6.f)), 6.f);
    if (OP == kUnaryGelu) {      // 0.5 x (1 + tanh(z)) = x sigmoid(2z), z = 0.79788458 (x + 0.044715 x^3)
        const float z = 0.79788458f * (x + 0.044715f * x * x * x);
        return times_sigmoid(x, 2.f * z);
    }
    return 0.5f * x * erfcf(-0.70710678f * x);   // kUnaryGeluStandard: 0.5 x (1 + erf(x / sqrt 2))
}
template <int OP>
__global__ void unary_f32_kernel(const float* __restrict__ x, float* __restrict__ y, size_t n, int vec) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    const size_t i0 = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    size_t done = 0;
    if (vec) {
        const size_t n4 = n >> 2;
        for (size_t i = i0; i < n4; i += stride) {
            const float4 u = reinterpret_cast<const float4*>(x)[i];
            reinterpret_cast<float4*>(y)[i] = make_float4(unary_f32_op<OP>(u.x), unary_f32_op<OP>(u.y), unary_f32_op<OP>(u.z),
                                                          unary_f32_op<OP>(u.w));
        }
        done = n4 << 2;
    }
    for (size_t i = done + i0; i < n; i += stride) y[i] = unary_f32_op<OP>(x[i]);
}
template <int OP>
static void launch_unary_op(const float* x, float* y, size_t n, int vec, int grid, cudaStream_t s) {
    unary_f32_kernel<OP><<<grid, 256, 0, s>>>(x, y, n, vec);
}
bool unary_f32_supported(int op) {
    switch (op) {
        case kUnaryAbs: case kUnaryNeg: case kUnarySquare: case kUnarySqrt: case kUnaryRsqrt: case kUnaryReciprocal:
        case kUnaryExp: case kUnaryLog: case kUnaryTanh: case kUnarySigmoid: case kUnarySilu: case kUnaryHardSwish:
        case kUnaryGelu: case kUnaryGeluStandard:
            return true;
        default:
            return false;
    }
}
cudaError_t launch_unary_f32(int op, const float* x, float* y, size_t n, cudaStream_t s) {
    const int vec = (((uintptr_t)x | (uintptr_t)y) & 15) == 0;
    const int grid = grid_for(vec ? (n >> 2) + 1 : n, 256);
    switch (op) {
        case kUnaryAbs: launch_unary_op<kUnaryAbs>(x, y, n, vec, grid, s); break;
        case kUnaryNeg: launch_unary_op<kUnaryNeg>(x, y, n, vec, grid, s); break;
        case kUnarySquare: launch_unary_op<kUnarySquare>(x, y, n, vec, grid, s); break;
        case kUnarySqrt: launch_unary_op<kUnarySqrt>(x, y, n, vec, grid, s); break;
        case kUnaryRsqrt: launch_unary_op<kUnaryRsqrt>(x, y, n, vec, grid, s); break;
        case kUnaryReciprocal: launch_unary_op<kUnaryReciprocal>(x, y, n, vec, grid, s); break;
        case kUnaryExp: launch_unary_op<kUnaryExp>(x, y, n, vec, grid, s); break;
        case kUnaryLog: launch_unary_op<kUnaryLog>(x, y, n, vec, grid, s); break;
        case kUnaryTanh: launch_unary_op<kUnaryTanh>(x, y, n, vec, grid, s); break;
        case kUnarySigmoid: launch_unary_op<kUnarySigmoid>(x, y, n, vec, grid, s); break;
        case kUnarySilu: launch_unary_op<kUnarySilu>(x, y, n, vec, grid, s); break;
        case kUnaryHardSwish: launch_unary_op<kUnaryHardSwish>(x, y, n, vec, grid, s); break;
        case kUnaryGelu: launch_unary_op<kUnaryGelu>(x, y, n, vec, grid, s); break;
        case kUnaryGeluStandard: launch_unary_op<kUnaryGeluStandard>(x, y, n, vec, grid, s); break;
        default: return cudaErrorInvalidValue;
    }
    ++g_launch_count;
    return cudaGetLastError();
}

// ---- ArgMax / ArgMin over the middle axis of [outside][axis][inside] -> int32 [outside][inside] (CPUArgMax.cpp:115-156, the
//      non-NC4HW4 branch): the running best starts at -FLT_MAX (ArgMin: +FLT_MAX) with index 0 and is replaced only by a strictly
//      better value, so the first extreme wins.  One warp per row when inside == 1 (lanes keep their own first best; the
//      reduction prefers the better value, then the lower index), else one thread per (outside, inside) column.
__device__ __forceinline__ bool argmax_better(float v, int i, float bv, int bi, int is_min) {
    return (is_min ? v < bv : v > bv) || (v == bv && i < bi);
}
__global__ void argmax_f32_kernel(const float* __restrict__ x, int32_t* __restrict__ y, int outside, int axis, int inside,
                                  int is_min) {
    const float init = is_min ? 3.402823466e38f : -3.402823466e38f;
    if (inside == 1) {
        const int row = (int)((blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
        if (row >= outside) return;
        const float* xp = x + (size_t)row * axis;
        float best = init;
        int idx = 0;
        for (int a = lane; a < axis; a += 32) {
            const float v = xp[a];
            if (is_min ? v < best : v > best) { best = v; idx = a; }
        }
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
            if (argmax_better(ov, oi, best, idx, is_min)) { best = ov; idx = oi; }
        }
        if (lane == 0) y[row] = idx;
        return;
    }
    const size_t total = (size_t)outside * inside;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t o = i / inside, in = i - o * inside;
        const float* xp = x + o * axis * inside + in;
        float best = init;
        int idx = 0;
        for (int a = 0; a < axis; ++a) {
            const float v = xp[(size_t)a * inside];
            if (is_min ? v < best : v > best) { best = v; idx = a; }
        }
        y[i] = idx;
    }
}
cudaError_t launch_argmax_f32(const float* x, int outside, int axis, int inside, int is_min, int32_t* y, cudaStream_t s) {
    if (inside == 1) argmax_f32_kernel<<<(unsigned)(((size_t)outside * 32 + 255) / 256), 256, 0, s>>>(x, y, outside, axis, inside, is_min);
    else argmax_f32_kernel<<<grid_for((size_t)outside * inside, 256), 256, 0, s>>>(x, y, outside, axis, inside, is_min);
    ++g_launch_count;
    return cudaGetLastError();
}

// ---- fp32 Scale (CPUScale, MNNScaleAndAddBias): y[n][c][i] = x[n][c][i] * scale[c] + bias[c]
__global__ void scale_f32_kernel(const float* __restrict__ x, const float* __restrict__ scale, const float* __restrict__ bias,
                                 float* __restrict__ y, int c, size_t plane, size_t total) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int ch = (int)((i / plane) % c);
        y[i] = fmaf(x[i], scale[ch], bias[ch]);
    }
}
cudaError_t launch_scale_f32(const float* x, const float* scale, const float* bias, float* y, int n, int c, size_t plane,
                             cudaStream_t s) {
    const size_t total = (size_t)n * c * plane;
    scale_f32_kernel<<<grid_for(total, 256), 256, 0, s>>>(x, scale, bias, y, c, plane, total);
    ++g_launch_count;
    return cudaGetLastError();
}

// ---- fp32 Softmax over the middle axis of [outside][axis][inside] (CPUSoftmax.cpp: max, sum of exp(x - max), divide).
//      One warp per (outside, inside) column.
__global__ void softmax_f32_kernel(const float* __restrict__ x, float* __restrict__ y, int outside, int axis, int inside) {
    const size_t col = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (col >= (size_t)outside * inside) return;
    const size_t o = col / inside, in = col - o * inside;
    const float* xp = x + o * axis * inside + in;
    float* yp = y + o * axis * inside + in;
    float mx = -3.402823466e38f;
    for (int a = lane; a < axis; a += 32) mx = fmaxf(mx, xp[(size_t)a * inside]);
    for (int s = 16; s > 0; s >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, s));
    float sum = 0.f;
    for (int a = lane; a < axis; a += 32) sum += expf(xp[(size_t)a * inside] - mx);
    for (int s = 16; s > 0; s >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, s);
    const float inv = 1.f / sum;
    for (int a = lane; a < axis; a += 32) yp[(size_t)a * inside] = expf(xp[(size_t)a * inside] - mx) * inv;
}
cudaError_t launch_softmax_f32(const float* x, float* y, int outside, int axis, int inside, cudaStream_t s) {
    softmax_f32_kernel<<<grid_for((size_t)outside * inside * 32, 256), 256, 0, s>>>(x, y, outside, axis, inside);
    ++g_launch_count;
    return cudaGetLastError();
}

}  // namespace mnnb200
