// winograd_int8.cu -- transform kernels of the int8 Winograd convolution F(m x m, 3 x 3), m = 2 / 4 / 6.
//
// Arithmetic = the reference CPU backend's ConvInt8Winograd (source/backend/cpu/compute/ConvInt8Winograd.cpp:306-356,
// 396-651) on the x86 AVX2 build, bit for bit: int8 -> float, B^T d B in fp32 with the exact operation order of
// x86_x64/avx/WinogradFunctions.cpp:358-553, per-position requantisation to int8, [alpha^2 batched int8 GEMMs on
// wgmma -- gemm_i8_wgmma.cu, EPI 2], A^T M A in fp32 (:555-579, 661-712, 981-1051), FloatToInt8.
// Replaces the structure of the reference CUDA backend's float-only WinoInputTrans / WinoTrans2Output
// (source/backend/cuda/execution/WinogradTrans.cuh:7-595): there one thread walks one (tile, channel) with 16 strided
// scalar loads; here a thread owns CPT adjacent channels of one tile, so a warp reads/writes whole 32..128-byte
// channel runs of the NHWC16 activation and of the [position][tile][channel] operand.
//
// Every float step is an explicitly rounded intrinsic: ptxas must not contract mul+add (the CPU code is unfused).
#include <cuda.h>
#include "common.cuh"
#include "host_util.h"
#include "kernels.h"
#include "hopper_common.cuh"

namespace mnnb200 {

namespace {

#define FA(a, b) __fadd_rn((a), (b))
#define FS(a, b) __fsub_rn((a), (b))
#define FM(a, b) __fmul_rn((a), (b))
// Vec8::fma(a, b, c) = a + b * c, two roundings (x86_x64/avx/Vec8.hpp:187-190)
#define FMA2(a, b, c) __fadd_rn((a), __fmul_rn((b), (c)))

// source transform along one axis: in-place on b[0..ALPHA) with stride S
template <int ALPHA, int S>
__device__ __forceinline__ void wino_src(float* b) {
    if (ALPHA == 4) {   // _sourceUnrollTransformUnit4x4
        float m0 = FS(b[0], b[2 * S]), m1 = FA(b[S], b[2 * S]), m2 = FS(b[2 * S], b[S]), m3 = FS(b[3 * S], b[S]);
        b[0] = m0; b[S] = m1; b[2 * S] = m2; b[3 * S] = m3;
    } else if (ALPHA == 6) {   // _sourceUnrollTransformUnit6x6
        float mid0 = FMA2(b[4 * S], b[2 * S], -4.f), mid1 = FMA2(b[3 * S], b[S], -4.f), mid2 = FMA2(b[2 * S], b[0], -4.f);
        float mid3 = FMA2(b[5 * S], b[3 * S], -4.f), mid4 = FS(b[4 * S], b[2 * S]), mid5 = FM(FS(b[3 * S], b[S]), 2.f);
        b[0] = FS(mid0, mid2); b[S] = FA(mid0, mid1); b[2 * S] = FS(mid0, mid1);
        b[3 * S] = FA(mid4, mid5); b[4 * S] = FS(mid4, mid5); b[5 * S] = FS(mid3, mid1);
    } else {   // _sourceUnrollTransformUnit8x8
        const float b0 = b[0], b1 = b[S], b2 = b[2 * S], b3 = b[3 * S], b4 = b[4 * S], b5 = b[5 * S], b6 = b[6 * S], b7 = b[7 * S];
        float mid0 = FMA2(FMA2(b6, b2, 36.f), b4, -13.f);
        float mid1 = FMA2(FMA2(b4, b0, 36.f), b2, -13.f);
        b[0] = FS(mid1, mid0);
        float mid2 = FMA2(FMA2(b5, b1, 36.f), b3, -13.f);
        b[S] = FA(mid0, mid2); b[2 * S] = FS(mid0, mid2);
        mid1 = FMA2(FMA2(b7, b3, 36.f), b5, -13.f);
        b[7 * S] = FS(mid1, mid2);
        mid0 = FMA2(FMA2(b6, b2, 9.f), b4, -10.f);
        mid1 = FA(FMA2(b5, b1, 18.f), FMA2(b5, b3, -20.f));
        mid2 = FMA2(FM(b5, 3.f), b1, 12.f);
        b[3 * S] = FA(mid0, mid1); b[4 * S] = FS(mid0, mid1);
        mid0 = FMA2(FMA2(b6, b2, 4.f), b4, -5.f);
        mid1 = FMA2(mid2, b3, -15.f);
        b[5 * S] = FA(mid0, mid1); b[6 * S] = FS(mid0, mid1);
    }
}
// destination transform along one axis: ALPHA inputs with stride S -> ALPHA-2 outputs written to the first slots
template <int ALPHA, int S>
__device__ __forceinline__ void wino_dst(float* s) {
    if (ALPHA == 4) {   // _destUnrollTransformUnit4x2
        float m0 = FA(FA(s[0], s[S]), s[2 * S]), m1 = FA(FS(s[S], s[2 * S]), s[3 * S]);
        s[0] = m0; s[S] = m1;
    } else if (ALPHA == 6) {   // _destUnrollTransformUnit6x4
        float v0 = FA(s[3 * S], s[4 * S]), v1 = FS(s[3 * S], s[4 * S]), v2 = FA(s[S], s[2 * S]), v3 = FS(s[S], s[2 * S]);
        float m0 = FA(FA(s[0], v2), v0), m1 = FA(FA(v3, v1), v1), m2 = FA(v2, FM(v0, 4.f)), m3 = FA(FA(v3, FM(v1, 8.f)), s[5 * S]);
        s[0] = m0; s[S] = m1; s[2 * S] = m2; s[3 * S] = m3;
    } else {   // _destUnrollTransformUnit8x6
        float mid0 = FA(s[S], s[2 * S]), mid1 = FS(s[S], s[2 * S]), mid2 = FA(s[3 * S], s[4 * S]), mid3 = FS(s[3 * S], s[4 * S]);
        float mid4 = FA(s[5 * S], s[6 * S]), mid5 = FS(s[5 * S], s[6 * S]);
        float m0 = FA(FA(FA(s[0], mid0), mid2), mid4);
        float m1 = FA(FA(mid1, FM(mid3, 2.f)), FM(mid5, 3.f));
        float m2 = FA(FA(mid0, FM(mid2, 4.f)), FM(mid4, 9.f));
        float m3 = FA(FA(mid1, FM(mid3, 8.f)), FM(mid5, 27.f));
        float m4 = FA(FA(mid0, FM(mid2, 16.f)), FM(mid4, 81.f));
        float m5 = FA(FA(FA(mid1, FM(mid3, 32.f)), FM(mid5, 243.f)), s[7 * S]);
        s[0] = m0; s[S] = m1; s[2 * S] = m2; s[3 * S] = m3; s[4 * S] = m4; s[5 * S] = m5;
    }
}

// ---- input transform: x int8 NHWC16 -> V[a][tile][Cp] int8 -----------------------------------------------------
template <int ALPHA, int CPT>
__global__ void __launch_bounds__(256) wino_input_kernel(const WinoParams p) {
    constexpr int UNIT = ALPHA - 2;
    const int groups = p.Cp / CPT;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int cg = (int)(idx % groups);
    const long long t = idx / groups;
    if (t >= p.T) return;
    const int wx = (int)(t % p.wU), hy = (int)((t / p.wU) % p.hU), b = (int)(t / ((long long)p.wU * p.hU));
    const int sy0 = hy * UNIT - p.pad_h, sx0 = wx * UNIT - p.pad_w;
    const float zf = (float)p.z_in;

    float d[CPT][ALPHA * ALPHA];
#pragma unroll
    for (int yy = 0; yy < ALPHA; ++yy) {
        const int iy = sy0 + yy;
#pragma unroll
        for (int xx = 0; xx < ALPHA; ++xx) {
            const int ix = sx0 + xx;
            const bool in = iy >= 0 && iy < p.IH && ix >= 0 && ix < p.IW;
            int8_t q[CPT];
            if (in) {
                const int8_t* src = p.x + (((size_t)b * p.IH + iy) * p.IW + ix) * p.Cp + cg * CPT;
                if (CPT == 4) *reinterpret_cast<int*>(q) = *reinterpret_cast<const int*>(src);
                else q[0] = src[0];
            }
#pragma unroll
            for (int c = 0; c < CPT; ++c)   // MNNInt8ScaleToFloat: (q - zero) * scale; window outside the image = 0.0f
                d[c][yy * ALPHA + xx] = in ? FM(FS((float)q[c], zf), p.s_in) : 0.0f;
        }
    }
#pragma unroll
    for (int c = 0; c < CPT; ++c) {
#pragma unroll
        for (int yy = 0; yy < ALPHA; ++yy) wino_src<ALPHA, 1>(&d[c][yy * ALPHA]);       // srcTransXFunc: along x, per row
#pragma unroll
        for (int k = 0; k < ALPHA; ++k) wino_src<ALPHA, ALPHA>(&d[c][k]);                // srcTransYFunc: along y, per column
    }
    int8_t* dst = p.v + (size_t)t * p.Cp + cg * CPT;
    const size_t a_stride = (size_t)p.Mpad * p.Cp;
#pragma unroll
    for (int a = 0; a < ALPHA * ALPHA; ++a) {
        int8_t q[CPT];
#pragma unroll
        for (int c = 0; c < CPT; ++c)   // MNNFloat2Int8(scale = 1/inputScale[a], zero = inputZero[a], -127, 127)
            q[c] = (int8_t)quant_cpu_exact(d[c][a], p.in_inv[a], p.in_zero[a], -127.f, 127.f);
        if (CPT == 4) *reinterpret_cast<int*>(dst + a * a_stride) = *reinterpret_cast<int*>(q);
        else dst[a * a_stride] = q[0];
    }
}

// Word-wide variant for F(6,3) (alpha = 6): the thread still owns 4 adjacent channels, i.e. one 32-bit word per
// pixel on both sides, but the four channels are transformed ONE AFTER THE OTHER so that only alpha^2 floats are live
// (plus the packed input and output words) instead of 4 * alpha^2.  Same arithmetic per channel as wino_input_kernel.
template <int ALPHA>
__global__ void __launch_bounds__(128) wino_input_seq4_kernel(const WinoParams p) {
    constexpr int UNIT = ALPHA - 2, A2 = ALPHA * ALPHA;
    const int groups = p.Cp >> 2;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int cg = (int)(idx % groups);
    const long long t = idx / groups;
    if (t >= p.T) return;
    const int wx = (int)(t % p.wU), hy = (int)((t / p.wU) % p.hU), b = (int)(t / ((long long)p.wU * p.hU));
    const int sy0 = hy * UNIT - p.pad_h, sx0 = wx * UNIT - p.pad_w;
    const float zf = (float)p.z_in;
    int win[A2];            // packed int8x4 of the window
    unsigned inmask[(A2 + 31) / 32];
#pragma unroll
    for (int i = 0; i < (A2 + 31) / 32; ++i) inmask[i] = 0;
#pragma unroll
    for (int yy = 0; yy < ALPHA; ++yy) {
        const int iy = sy0 + yy;
#pragma unroll
        for (int xx = 0; xx < ALPHA; ++xx) {
            const int ix = sx0 + xx, a = yy * ALPHA + xx;
            const bool in = iy >= 0 && iy < p.IH && ix >= 0 && ix < p.IW;
            win[a] = in ? __ldg(reinterpret_cast<const int*>(p.x + (((size_t)b * p.IH + iy) * p.IW + ix) * p.Cp + cg * 4)) : 0;
            if (in) inmask[a >> 5] |= 1u << (a & 31);
        }
    }
    unsigned wout[A2];
#pragma unroll
    for (int a = 0; a < A2; ++a) wout[a] = 0;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        float d[A2];
#pragma unroll
        for (int a = 0; a < A2; ++a) {   // MNNInt8ScaleToFloat: (q - zero) * scale; window outside the image = 0.0f
            const int q = (int)(int8_t)((unsigned)win[a] >> (8 * c));
            d[a] = (inmask[a >> 5] >> (a & 31)) & 1u ? FM(FS((float)q, zf), p.s_in) : 0.0f;
        }
#pragma unroll
        for (int yy = 0; yy < ALPHA; ++yy) wino_src<ALPHA, 1>(&d[yy * ALPHA]);       // srcTransXFunc: along x, per row
#pragma unroll
        for (int k = 0; k < ALPHA; ++k) wino_src<ALPHA, ALPHA>(&d[k]);                // srcTransYFunc: along y, per column
#pragma unroll
        for (int a = 0; a < A2; ++a) {   // MNNFloat2Int8(scale = 1/inputScale[a], zero = inputZero[a], -127, 127)
            const int q = quant_cpu_exact(d[a], p.in_inv[a], p.in_zero[a], -127.f, 127.f);
            wout[a] |= (unsigned)(q & 0xff) << (8 * c);
        }
    }
    int8_t* dst = p.v + (size_t)t * p.Cp + cg * 4;
    const size_t a_stride = (size_t)p.Mpad * p.Cp;
#pragma unroll
    for (int a = 0; a < A2; ++a) *reinterpret_cast<unsigned*>(dst + a * a_stride) = wout[a];
}

// ---- output transform: M[a][tile][OCp] fp32 -> y int8 NHWC16 -----------------------------------------------------
template <int ALPHA, int CPT>
__global__ void __launch_bounds__(256) wino_output_kernel(const WinoParams p) {
    constexpr int UNIT = ALPHA - 2;
    const int groups = p.OCp / CPT;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int og = (int)(idx % groups);
    const long long t = idx / groups;
    if (t >= p.T) return;
    const int wx = (int)(t % p.wU), hy = (int)((t / p.wU) % p.hU), b = (int)(t / ((long long)p.wU * p.hU));

    float s[CPT][ALPHA * ALPHA];
    const float* src = p.m + (size_t)t * p.OCp + og * CPT;
    const size_t a_stride = (size_t)p.Mpad * p.OCp;
#pragma unroll
    for (int a = 0; a < ALPHA * ALPHA; ++a) {
        if (CPT == 4) {
            float4 v = *reinterpret_cast<const float4*>(src + a * a_stride);
            s[0][a] = v.x; s[1 % CPT][a] = v.y; s[2 % CPT][a] = v.z; s[3 % CPT][a] = v.w;
        } else if (CPT == 2) {
            float2 v = *reinterpret_cast<const float2*>(src + a * a_stride);
            s[0][a] = v.x; s[1 % CPT][a] = v.y;
        } else {
            s[0][a] = src[a * a_stride];
        }
    }
    float fused[CPT];
#pragma unroll
    for (int c = 0; c < CPT; ++c) {
        fused[c] = p.fused_bias[og * CPT + c];
#pragma unroll
        for (int k = 0; k < ALPHA; ++k) wino_dst<ALPHA, ALPHA>(&s[c][k]);          // dstTransYFunc: along y, per column
#pragma unroll
        for (int j = 0; j < UNIT; ++j) wino_dst<ALPHA, 1>(&s[c][j * ALPHA]);        // dstTransXFunc: along x, per output row
    }
#pragma unroll
    for (int j = 0; j < UNIT; ++j) {
        const int oy = hy * UNIT + j;
        if (oy >= p.OH) continue;
#pragma unroll
        for (int i = 0; i < UNIT; ++i) {
            const int ox = wx * UNIT + i;
            if (ox >= p.OW) continue;
            int8_t q[CPT];
#pragma unroll
            for (int c = 0; c < CPT; ++c) {   // mergeAddBiasScaleQuantize: MNNFloat2Int8(y * (1/s_out) + fusedBias[oc])
                int v = quant_cpu_exact(s[c][j * ALPHA + i], p.out_inv, fused[c], p.minv, p.maxv);
                q[c] = (og * CPT + c < p.OC) ? (int8_t)v : (int8_t)0;   // NHWC16 channel padding stays zero
            }
            int8_t* dst = p.y + (((size_t)b * p.OH + oy) * p.OW + ox) * p.OCp + og * CPT;
            if (CPT == 4) *reinterpret_cast<int*>(dst) = *reinterpret_cast<int*>(q);
            else if (CPT == 2) *reinterpret_cast<short*>(dst) = *reinterpret_cast<short*>(q);
            else dst[0] = q[0];
        }
    }
}


// =====================================================================================================================
// F(2x2, 3x3) with the 16 position GEMMs and the output transform in ONE kernel: all 16 accumulators of a (128-tile,
// 8-channel) block live in registers at once (16 positions x 4 per thread of each consumer warpgroup), so the fp32 M tensor
// (16 bytes per output byte, written and read back through HBM by the three-kernel form) never exists.
//   warp 8: TMA producer (V[a] tile 128 x K, U[a] chunk 8 x K per stage); warps 0-7: two consumer warpgroups, 64 Winograd
//   tiles each: wgmma m64n8k32 s8 per position into acc[a] -> acc*scale[a][oc] + offset[a][oc] -> A^T M A in the
//   reference's exact fp32 order -> FloatToInt8 -> stores per output pixel.  A thread holds every position of its
//   (tile, channel) pairs, so the output transform needs no data exchange.
// Arithmetic identical to gemm_i8_wgmma_kernel<2> + wino_output_kernel<4,4>, bit for bit.
// =====================================================================================================================
using namespace hop;
constexpr int kFStages = 6, kFBN = kWinoFusedBN, kFStageBytes = 128 * 128 + kFBN * 128;

__global__ void __launch_bounds__(kThreads, 1)
wino_f23_fused_kernel(const __grid_constant__ CUtensorMap tmap_v, const __grid_constant__ CUtensorMap tmap_u, const WinoFusedParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    uint8_t* smem = smem_raw + (base - raw);
    const int off_consts = kFStages * kFStageBytes;                 // [3][16][8] floats/ints
    const int off_bars = off_consts + 3 * 16 * kFBN * 4;
    const uint32_t bar0 = base + off_bars;
    auto full_bar = [&](int s) { return bar0 + 8u * s; };
    auto empty_bar = [&](int s) { return bar0 + 8u * (kFStages + s); };
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int num_kb = (p.K + 127) / 128;
    const int work_total = p.m_tiles * p.oc_chunks;

    if (warp == 8 && lane == 0) {
        prefetch_tmap(&tmap_v);
        prefetch_tmap(&tmap_u);
        for (int s = 0; s < kFStages; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 8); }
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            int stage = 0, phase = 0;
            for (int w = blockIdx.x; w < work_total; w += gridDim.x) {
                const int ch = w % p.oc_chunks, mt = w / p.oc_chunks;
                for (int a = 0; a < 16; ++a)
                    for (int kb = 0; kb < num_kb; ++kb) {
                        mbar_wait(empty_bar(stage), phase ^ 1);
                        mbar_expect_tx(full_bar(stage), (uint32_t)kFStageBytes);
                        const uint32_t dst = base + stage * kFStageBytes;
                        tma_load_2d(dst, &tmap_v, full_bar(stage), kb * 128, a * p.Mpad + mt * 128);
                        tma_load_2d(dst + 128 * 128, &tmap_u, full_bar(stage), kb * 128, a * p.OCb + ch * kFBN);
                        if (++stage == kFStages) { stage = 0; phase ^= 1; }
                    }
            }
        }
    } else {
        const int ct = threadIdx.x, wg = ct >> 7;
        const int r_base = wg * 64 + (warp & 3) * 16 + (lane >> 2);
        const int q4 = lane & 3;
        float* c_scale = reinterpret_cast<float*>(smem + off_consts);
        float* c_off = c_scale + 16 * kFBN;
        int* c_wsum = reinterpret_cast<int*>(c_off + 16 * kFBN);
        int stage = 0, phase = 0;
        int acc[16][4];
#pragma unroll
        for (int a = 0; a < 16; ++a)
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[a][i] = 0;
        for (int w = blockIdx.x; w < work_total; w += gridDim.x) {
            const int ch = w % p.oc_chunks, mt = w / p.oc_chunks;
            const int oc0 = ch * kFBN;
            named_sync(1, kConsumerThreads);                              // previous item's readers are done
            for (int i = ct; i < 16 * kFBN; i += kConsumerThreads) {
                const int a = i / kFBN, j = i - a * kFBN, oc = oc0 + j;
                const bool v = oc < p.OC;
                c_scale[i] = v ? p.scale[a * p.OCp + oc] : 0.f;
                c_off[i] = v ? p.offset[a * p.OCp + oc] : 0.f;
                c_wsum[i] = v ? p.wsum128[a * p.OCp + oc] : 0;
            }
            named_sync(1, kConsumerThreads);
            int prev = -1;
#pragma unroll
            for (int a = 0; a < 16; ++a) {
                for (int kb = 0; kb < num_kb; ++kb) {
                    mbar_wait(full_bar(stage), phase);
                    const uint32_t a_addr = base + stage * kFStageBytes + wg * 64 * 128, b_addr = base + stage * kFStageBytes + 128 * 128;
                    const int kleft = p.K - kb * 128;
                    const int nmma = kleft >= 128 ? 4 : (kleft + 31) / 32;
                    fence_acc(acc[a]);
                    wgmma_fence();
                    for (int k = 0; k < nmma; ++k)
                        wgmma<Kind::S8, kFBN>(acc[a], gdesc_sw128(a_addr + k * 32), gdesc_sw128(b_addr + k * 32), (kb | k) != 0);
                    wgmma_commit();
                    wgmma_wait<1>();
                    fence_acc(acc[a]);
                    if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(empty_bar(prev)); }
                    prev = stage;
                    if (++stage == kFStages) { stage = 0; phase ^= 1; }
                }
            }
            wgmma_wait<0>();
#pragma unroll
            for (int a = 0; a < 16; ++a) fence_acc(acc[a]);
            __syncwarp();
            if (lane == 0) mbar_arrive(empty_bar(prev));
            // register i of acc[a] = tile r_base + 8 * (i >> 1), channel 2 * q4 + (i & 1)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const long long t = (long long)mt * 128 + r_base + 8 * h;
                const bool tile_ok = t < p.T;
                const int wx = (int)(t % p.wU), hy = (int)((t / p.wU) % p.hU), b = (int)(t / ((long long)p.wU * p.hU));
                uint32_t outw[4] = {0, 0, 0, 0};                          // [pixel j*2+i] two packed bytes
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int cc = 2 * q4 + e, oc = oc0 + cc;
                    float s[16];                                          // [position]
#pragma unroll
                    for (int a = 0; a < 16; ++a) {
                        const int j = a * kFBN + cc;
                        // position GEMM output (avx/GemmInt8.cpp:672-772 float branch): float(acc) * scale[a][oc] + offset[a][oc]
                        s[a] = __fadd_rn(__fmul_rn(__int2float_rn(acc[a][2 * h + e] + c_wsum[j]), c_scale[j]), c_off[j]);
                    }
#pragma unroll
                    for (int k = 0; k < 4; ++k) wino_dst<4, 4>(&s[k]);           // dstTransYFunc: along y, per column
#pragma unroll
                    for (int j = 0; j < 2; ++j) wino_dst<4, 1>(&s[j * 4]);       // dstTransXFunc: along x, per output row
#pragma unroll
                    for (int px = 0; px < 4; ++px) {
                        int qv = 0;
                        if (oc < p.OC) qv = quant_cpu_exact(s[(px >> 1) * 4 + (px & 1)], p.out_inv, p.fused_bias[oc], p.minv, p.maxv);
                        outw[px] |= (uint32_t)(qv & 0xff) << (8 * e);
                    }
                }
                if (tile_ok) {
#pragma unroll
                    for (int px = 0; px < 4; ++px) {
                        const int oy = hy * 2 + (px >> 1), ox = wx * 2 + (px & 1);
                        if (oy < p.OH && ox < p.OW)
                            *reinterpret_cast<uint16_t*>(p.y + (((size_t)b * p.OH + oy) * p.OW + ox) * p.OCp + oc0 + 2 * q4) = (uint16_t)outw[px];
                    }
                }
            }
        }
    }
}

}  // namespace

cudaError_t launch_wino_input(const WinoParams& p, cudaStream_t s) {
    ++g_launch_count;
    const int alpha = p.unit + 2;
    // measured (r01): alpha = 6: 0.259 -> 0.239 ms on the ResNet set with the word-wide kernel; alpha = 8: no gain there (255
    // registers, 8 warps per SM), so F(6,3) keeps the one-channel-per-thread kernel
    if (alpha == 6) {
        const long long threads = (long long)p.T * (p.Cp / 4);
        wino_input_seq4_kernel<6><<<(unsigned)((threads + 127) / 128), 128, 0, s>>>(p);
        return cudaGetLastError();
    }
    const int cpt = alpha == 4 ? 4 : 1;
    const long long threads = (long long)p.T * (p.Cp / cpt);
    const unsigned grid = (unsigned)((threads + 255) / 256);
    if (alpha == 4) wino_input_kernel<4, 4><<<grid, 256, 0, s>>>(p);
    else if (alpha == 8) wino_input_kernel<8, 1><<<grid, 256, 0, s>>>(p);
    else return cudaErrorInvalidValue;
    return cudaGetLastError();
}
cudaError_t launch_wino_f23_fused(const WinoFusedParams& p, const void* tmap_v, const void* tmap_u, cudaStream_t s, int sm_count) {
    const int smem = kFStages * kFStageBytes + 3 * 16 * kFBN * 4 + 256 + 1024;
    {
        cudaError_t e = ensure_max_dynamic_smem((const void*)wino_f23_fused_kernel, smem);
        if (e != cudaSuccess) return e;
    }
    const int work = p.m_tiles * p.oc_chunks;
    const int grid = work < sm_count ? work : sm_count;
    ++g_launch_count;
    wino_f23_fused_kernel<<<grid, kThreads, smem, s>>>(*reinterpret_cast<const CUtensorMap*>(tmap_v), *reinterpret_cast<const CUtensorMap*>(tmap_u), p);
    return cudaGetLastError();
}

cudaError_t launch_wino_output(const WinoParams& p, cudaStream_t s) {
    ++g_launch_count;
    const int alpha = p.unit + 2;
    const int cpt = alpha == 4 ? 4 : (alpha == 6 ? 2 : 1);
    const long long threads = (long long)p.T * (p.OCp / cpt);
    const unsigned grid = (unsigned)((threads + 255) / 256);
    if (alpha == 4) wino_output_kernel<4, 4><<<grid, 256, 0, s>>>(p);
    else if (alpha == 6) wino_output_kernel<6, 2><<<grid, 256, 0, s>>>(p);
    else if (alpha == 8) wino_output_kernel<8, 1><<<grid, 256, 0, s>>>(p);
    else return cudaErrorInvalidValue;
    return cudaGetLastError();
}

}  // namespace mnnb200
