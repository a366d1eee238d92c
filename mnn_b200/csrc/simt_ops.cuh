// simt_ops.cuh -- the per-work-index bodies of the HBM-bound int8 neighbours of the conv path (depthwise conv, eltwise add) as
// device functions, shared by the stand-alone kernels (elementwise.cu) and by the whole-net program kernel
// (conv_group_wgmma.cu), where the consumer warps execute them between GEMM tiles.
//
// COH = false: activations through the read-only path (ld.global.nc): the producer kernel has finished.
// COH = true : activations written earlier in the SAME launch by other SMs: L2-coherent loads (ld.global.cg), never the
//              non-coherent / L1 paths.
#pragma once
#include "common.cuh"
#include "kernels.h"

namespace mnnb200 {

template <bool COH>
__device__ __forceinline__ int4 ld_act16(const void* p) {
    int4 r;
    if (COH) asm volatile("ld.global.cg.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
    else asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
template <bool COH>
__device__ __forceinline__ int ld_act4(const void* p) {
    int r;
    if (COH) asm volatile("ld.global.cg.s32 %0, [%1];" : "=r"(r) : "l"(p) : "memory");
    else asm volatile("ld.global.nc.s32 %0, [%1];" : "=r"(r) : "l"(p));
    return r;
}

// ---- depthwise int8 conv, generic (CPUDepthwiseConvInt8.cpp:40-100, GemmInt8_VNNI.cpp:2978-3110): one 16-channel group of
//      one output pixel per work index.  acc = bias_i32 + sum (x+128)*w [the +128*sum(w) part is pre-added to bias_i32 on the
//      host]; f = float(acc)*scale; q = trunc(f +- 0.5); clamp AFTER rounding.
template <bool COH>
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
                int4 xv = ld_act16<COH>(p.x + (((size_t)b * p.IH + iy) * p.IW + ix) * p.Cp + g * 16);
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
template <int S, bool COH>
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
            xw[c] = (yin && (unsigned)ix < (unsigned)p.IW) ? ld_act4<COH>(row + (size_t)ix * p.Cp) : zsplat;
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
__host__ __device__ inline bool dw_is_3x3_fast(const DwParams& p) {
    return p.KH == 3 && p.KW == 3 && p.dh == 1 && p.dw == 1 && p.sh == p.sw && (p.sh == 1 || p.sh == 2);
}
// work indices of a depthwise conv per OUTPUT ROW (a row of one image): the unit the program kernel tiles by
__host__ __device__ inline size_t dw_work_per_row(const DwParams& p) {
    return dw_is_3x3_fast(p) ? (size_t)((p.OW + 3) / 4) * (p.Cp >> 2) : (size_t)p.OW * (p.Cp >> 4);
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
template <bool COH>
__device__ __forceinline__ void binary_add_work(const AddParams& p, size_t i) {
    const int groups = p.cp >> 4;
    int g = (int)(i % groups);
    int4 a = ld_act16<COH>(p.x0 + i * 16), b = ld_act16<COH>(p.x1 + i * 16);
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

// per-op parameters of a SIMT op inside a whole-net program (GroupLayerParams.mode: 2 = depthwise conv, 3 = eltwise add)
struct ProgSimtOp {
    DwParams dw;
    AddParams add;
};

}  // namespace mnnb200
