// conv_group_epilogue.cuh -- the int8 epilogue of the conv-group kernels (conv_group_wgmma.cu, conv_group_shallow_wgmma.cu):
// CPU-exact requant of a wgmma accumulator fragment (requant_cpu_exact, common.cuh), clamp on the rounded integers and
// predicated 8-byte stores to the NHWC16 output rows.  Both kernels run one tile's columns through group_column_run, so the
// two produce the same bytes for the same accumulators.
#pragma once
#include <cstdint>

namespace mnnb200 {
namespace {

// requant_cpu_exact (common.cuh) WITHOUT its clamp, which the epilogue applies to the rounded integers (see the column run's
// clamp4 for why that is exact).  The +-0.5 is copysign(0.5, f) = (f & sign) | 0.5 in one LOP3 with 0.5 in a register:
// written as an and and an or of two immediates, ptxas emits two LOP3s.
__device__ __forceinline__ int round_half_away(float f) {
    uint32_t h;
    asm("lop3.b32 %0, %1, 0x80000000, 0x3f000000, 0xEA;" : "=r"(h) : "r"(__float_as_uint(f)));   // 0xEA: (a & b) | c
    return __float2int_rz(__fadd_rn(f, __uint_as_float(h)));
}
__device__ __forceinline__ int requant_round(int acc_u, float wscale, float scale_x, float bias_float) {
    float f = __fmul_rn(__int2float_rn(acc_u), wscale);
    f = __fmul_rn(f, scale_x);
    return round_half_away(__fadd_rn(f, bias_float));
}
// the same sequence for accumulators with |acc_u| < 2^22: float(acc_u) = as_float(0x4B400000 + acc_u) - 1.5 * 2^23 is exact (the
// integer lands in the mantissa of a float in [2^23, 2^24)): one IADD + one FADD instead of an I2F on the conversion unit
// (the conv-group kernels' accumulators start at 0x4B400000 + 128 sum w, so acc_m here is already 0x4B400000 + acc_u)
__device__ __forceinline__ int requant_round_small(int acc_m, float wscale, float scale_x, float bias_float) {
    float f = __fmul_rn(__fsub_rn(__int_as_float(acc_m), 12582912.0f), wscale);
    f = __fmul_rn(f, scale_x);
    return round_half_away(__fadd_rn(f, bias_float));
}
// two int32 -> one s16 pair, each saturated to [-32768, 32767] (one I2IP): lo in bits 0-15, hi in bits 16-31
__device__ __forceinline__ uint32_t pack_sat_s16x2(int lo, int hi) {
    uint32_t d;
    asm("cvt.pack.sat.s16.s32 %0, %1, %2;" : "=r"(d) : "r"(hi), "r"(lo));
    return d;
}

// A global store the compiler does not treat as a memory write (no "memory" clobber): nothing in the kernels reads the output
// back, and the compiler may then keep shared-memory values in registers and issue later loads across it.  Predicated on
// j < lim inside the instruction, so a run of such stores over a column loop stays one straight run of code.
__device__ __forceinline__ void st_global_v2_if(int8_t* p, uint32_t lo, uint32_t hi, int j, int lim) {
    asm volatile("{\n .reg .pred q;\n setp.lt.s32 q, %3, %4;\n @q st.global.v2.b32 [%0], {%1, %2};\n}\n" ::"l"(p), "r"(lo), "r"(hi),
                 "r"(j), "r"(lim));
}
__device__ __forceinline__ void st_global_b32_if(int8_t* p, uint32_t v, int j, int lim) {
    asm volatile("{\n .reg .pred q;\n setp.lt.s32 q, %2, %3;\n @q st.global.b32 [%0], %1;\n}\n" ::"l"(p), "r"(v), "r"(j), "r"(lim));
}

// One tile's column run on one thread: every column group of both accumulator rows of the BN-wide tile, in one straight run.
// Register i of acc = row h = (i >> 1) & 1, GEMM column 8 * (i >> 2) + 2 * q4 + (i & 1); the chunk's columns are permuted
// (group_column_channel, kernels.h): in each 32-column group G the thread holds channels 32 G + 8 q4 ... + 7 of its rows (a
// 16-wide last group: 32 G + 4 q4 ... + 3), stored with one 8-byte (4-byte) store per row and group.  Columns past the chunk's
// valid ones read zero constants, only their stores are predicated off (lim[h]: the channels row h stores, 0 for a row outside
// the layer).  With no control flow inside, ptxas overlaps the requant chains.
//   kRegConsts: the thread's wscale / biasFloat pairs are ws[j] / bs[j] (registers); else they are read from wscale / bias
//   kSmall: |acc_u| < 2^22, the int -> float conversion runs on the FP32 pipe (requant_round_small)
//   kCorr: corrp[h] is row h's border-correction row (mode 1 with z_in != 0), added to the accumulators first
// mlo / mhi clear the bytes of pad channels when the clamp excludes 0; min2 / max2 are the clamp bounds as s16 pairs.
template <int BN, bool kRegConsts, bool kSmall, bool kCorr>
__device__ __forceinline__ void group_column_run(const int* acc, const float2* ws, const float2* bs, const float* wscale,
                                                 const float* bias, int q4, float scale_x, uint32_t min2, uint32_t max2,
                                                 const uint32_t* mlo, const uint32_t* mhi, int8_t* const* yrow, const int* lim,
                                                 const int32_t* const* corrp) {
    // 4 rounded outputs -> their 4 clamped bytes, q[0] in byte 0: the clamp runs on the rounded integers.  The reference's
    // rounding is monotone non-decreasing and maps every integer bound to itself, so max(min(round(f), maxv), minv) =
    // round(max(min(f, maxv), minv)) bit for bit; the saturating pack to s16 changes nothing for bounds in that range.
    auto clamp4 = [&](const int* q) -> uint32_t {
        const uint32_t p0 = __vmaxs2(__vmins2(pack_sat_s16x2(q[0], q[1]), max2), min2);
        const uint32_t p1 = __vmaxs2(__vmins2(pack_sat_s16x2(q[2], q[3]), max2), min2);
        return __byte_perm(p0, p1, 0x6420);
    };
#pragma unroll
    for (int G = 0; G < (BN + 31) / 32; ++G) {
        constexpr int kFull = 4;
        const int S = BN - 32 * G >= 32 ? kFull : 2;      // column pairs of the thread per row in this group
        const int ch = 32 * G + 2 * S * q4;              // its first channel
        float2 wg[kFull], bg[kFull];         // the group's constants serve both rows
#pragma unroll
        for (int s = 0; s < S; ++s) {
            if constexpr (kRegConsts) {
                wg[s] = ws[4 * G + s];
                bg[s] = bs[4 * G + s];
            } else {
                wg[s] = *reinterpret_cast<const float2*>(wscale + 8 * (4 * G + s) + 2 * q4);
                bg[s] = *reinterpret_cast<const float2*>(bias + 8 * (4 * G + s) + 2 * q4);
            }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            int q[2 * kFull];
#pragma unroll
            for (int s = 0; s < S; ++s) {
                const int j = 4 * G + s;
                int a0 = acc[j * 4 + 2 * h], a1 = acc[j * 4 + 2 * h + 1];
                if constexpr (kCorr) {
                    const int2 k = __ldg(reinterpret_cast<const int2*>(corrp[h] + 8 * j + 2 * q4));
                    a0 += k.x;
                    a1 += k.y;
                }
                if constexpr (kSmall) {   // |acc_u| < 2^22: int -> float on the FP32 pipe (exact)
                    q[2 * s] = requant_round_small(a0, wg[s].x, scale_x, bg[s].x);
                    q[2 * s + 1] = requant_round_small(a1, wg[s].y, scale_x, bg[s].y);
                } else {
                    q[2 * s] = requant_round(a0, wg[s].x, scale_x, bg[s].x);
                    q[2 * s + 1] = requant_round(a1, wg[s].y, scale_x, bg[s].y);
                }
            }
            const uint32_t lo = clamp4(q) & mlo[G];
            if (S == kFull) {
                const uint32_t hi = clamp4(q + 4) & mhi[G];
                st_global_v2_if(yrow[h] + ch, lo, hi, ch, lim[h]);
            } else {
                st_global_b32_if(yrow[h] + ch, lo, ch, lim[h]);
            }
        }
    }
}

// The byte masks of the thread's 32-column groups for a run on n chunk n0 of a layer with OC channels and clamp [minv, maxv]:
// the chunk's pad channels (>= OC) are stored and must stay zero.  Their table constants are zero, so they requantise to
// clamp(0): only a clamp without 0 needs their bytes cleared, and only in the chunk that holds them (all ones elsewhere).
template <int BN>
__device__ __forceinline__ void group_pad_masks(int OC, int n0, int ncols, int minv, int maxv, int q4, uint32_t* mlo, uint32_t* mhi) {
    const bool pad = OC - n0 < ncols && (minv > 0 || maxv < 0);
#pragma unroll
    for (int G = 0; G < (BN + 31) / 32; ++G) {
        const int nv = pad ? OC - n0 - (32 * G + 2 * (BN - 32 * G >= 32 ? 4 : 2) * q4) : 8;   // the group's valid channels
        mlo[G] = nv >= 4 ? 0xffffffffu : (nv <= 0 ? 0u : (1u << (8 * nv)) - 1u);
        mhi[G] = nv >= 8 ? 0xffffffffu : (nv <= 4 ? 0u : (1u << (8 * (nv - 4))) - 1u);
    }
}

}  // namespace
}  // namespace mnnb200
