/* The 4-bit form of the MNN-LLM linear layer (SURVEY a7), restated in scalar C next to mnn_oracle.c's 8-bit forms, whose input
 * quantisation it repeats operation for operation.  TEST INFRASTRUCTURE ONLY; built by oracle/w4_oracle.py with
 * -ffp-contract=off like mnn_oracle.c.  File:line citations are paths in the reference tree. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#define ORACLE_API __attribute__((visibility("default")))
#define X86_OFFSET 128   /* the x86 backend stores int8 activations as uint8 (q + 128) */

/* ------------------------------------------------------------------------------------------
 * a7 with 4-BIT weights (MNN-LLM's default export: --quant_bit 4, --quant_block 64), per channel (blocks == 1) or K-blocked.
 * wpacked is what ConvolutionCommon::load(op, bn, false, forceInt8 = true) returns for a 4-bit IDST buffer (canUseInt4,
 * ConvolutionCommon.cpp:279-307 / :357-371): oc * ic / 2 bytes of u = q + 8, the EVEN index in the high nibble; alpha / wzero
 * [oc][blocks], wzero already min - clampMin * scale (:757-766) or NULL.  The x86 executor (ConvInt8TiledExecutor.cpp):
 *   mWeightBits = 4 forces the asymmetric form (:454-458): weight bias wb_b = wzero_b + (-8) * alpha_b, or (-8) * alpha_b
 *   (_computeReorderQuantInfo, :208-263);  weightKernelSum, ONE per output (the input is not block-quantised), summed over the
 *   blocks in one of two roundings chosen by realInt4OrInt8 (:237-243, :264-268), which is true when the fast int4 reorder ran
 *   (directReadInt4weight / notConvertInt4ToInt8, :537-538, :567, :807-816): oc a multiple of the GEMM's H unit and ic of its L
 *   unit -- 64 and 4 on the AVX512 build:
 *     fast:  accum += ks_b * alpha_b + bs * wb_b
 *     else:  accum += (ks_b - bs * 8) * alpha_b + bs * wzero_b      (the last term absent when symmetric)
 *   with ks_b = sum_b u (exact in fp32: _AVX_MNNReorderWeightInt4 / reorderWeight's sums, avx/ReorderFunctions.cpp:520-637).
 * The GEMM kernel (_AVX512_MNNGemmInt8AddBiasScale_16x4_w4_Unit_VNNI, avx512/GemmInt8_VNNI.cpp:1626-1990; on a host without
 * VNNI _AVX512_NO_VNNI_4_4_64_w4, avx512/GemmInt8.cpp:363-378), block after block:
 *   acc_b = sum_b (xq + 128) * u  (int32, dpbusds);  f = float(acc_b) * alpha_b;  f = f * dq;
 *   block 0 only: f = f + (dq * -128) * weightKernelSum  (:1806-1852 "if input not block quant, only accum once");
 *   f = xsum_b * wb_b + f  (srcKernelSum, :1871-);  blocks > 0: f = accum + f;  last block: + bias, clamp.
 * The input quantisation is that of mnn_oracle_linear_w8_dynamic_blocks: per token, symmetric for >= 2 tokens, the single-quant
 * decode form with bias' = bias + weightKernelSum * (-qbias * scale) for ONE token (:2034-2047).  Pinned on the live reference
 * (tests/test_w4_linear_cpu.py, tests/golden/w4_linear_golden.npz, recorded by oracle/refdump_w4.cpp): <= 1.8e-6 relative over the 14 recorded cases; most outputs
 * differ in the last bits (the VNNI kernel associates the fp32 terms differently), as for the 8-bit blocked form.
 * ------------------------------------------------------------------------------------------ */
ORACLE_API void mnn_oracle_linear_w4_dynamic_blocks(const float* x, int tokens, int ic, const uint8_t* wpacked, int oc,
                                                    const float* alpha, const float* wzero, const float* bias, int blocks,
                                                    int relu, int relu6, float* y) {
    const int bs = ic / blocks;
    const int fast = (oc % 64 == 0) && (ic % 4 == 0);
    int32_t* xq = (int32_t*)malloc(sizeof(int32_t) * (size_t)ic);
    int32_t* u = (int32_t*)malloc(sizeof(int32_t) * (size_t)oc * ic);
    float* wb = (float*)malloc(sizeof(float) * (size_t)oc * blocks);
    float* wks = (float*)malloc(sizeof(float) * (size_t)oc);
    for (size_t i = 0; i < (size_t)oc * ic; ++i) u[i] = (i & 1) ? (wpacked[i >> 1] & 15) : (wpacked[i >> 1] >> 4);
    for (int o = 0; o < oc; ++o) {
        float accum = 0.f;
        for (int b = 0; b < blocks; ++b) {
            const size_t ob = (size_t)o * blocks + b;
            int32_t ks = 0;
            for (int k = b * bs; k < (b + 1) * bs; ++k) ks += u[(size_t)o * ic + k];
            const float a = alpha[ob];
            wb[ob] = wzero ? wzero[ob] + (float)(-8) * a : (float)(-8) * a;
            float term;
            if (fast) {
                term = (float)ks * a + (float)bs * wb[ob];
            } else {
                term = ((float)ks - (float)(bs * 8)) * a;
                if (wzero) term = term + (float)bs * wzero[ob];
            }
            accum = accum + term;
        }
        wks[o] = accum;
    }
    for (int t = 0; t < tokens; ++t) {
        const float* xr = x + (size_t)t * ic;
        float scale, izf = 0.f;
        if (tokens == 1) {
            float mn = xr[0], mx = xr[0];
            for (int k = 1; k < ic; ++k) { mn = xr[k] < mn ? xr[k] : mn; mx = xr[k] > mx ? xr[k] : mx; }
            if (ic % 16 != 0) { mn = mn < 0.f ? mn : 0.f; mx = mx > 0.f ? mx : 0.f; }
            float range = mx - mn, qscale, qbias;
            if (range <= 1e-7) { scale = 1.f; qscale = 1.f; qbias = -mx; }
            else {
                qscale = 255.f / range;
                scale = range / 255.f;
                float t0 = -mn * 255.f;
                qbias = roundf(t0 / range) - 128.0f;
            }
            for (int k = 0; k < ic; ++k) {
                float v = fmaf(xr[k], qscale, qbias);
                v = v > -128.f ? v : -128.f;
                v = v < 127.f ? v : 127.f;
                v = v + (v < 0.f ? -0.5f : 0.5f);
                xq[k] = (int32_t)v;
            }
            izf = -qbias * scale;
        } else {
            float absmax = 0.f;
            for (int k = 0; k < ic; ++k) {
                float a = fabsf(xr[k]);
                absmax = a > absmax ? a : absmax;
            }
            float qscale = 1.f;
            scale = 1.f;
            if (!(absmax < 1e-7)) {
                qscale = 127.0f / absmax;
                scale = absmax / 127.0f;
            }
            for (int k = 0; k < ic; ++k) xq[k] = (int32_t)nearbyintf(xr[k] * qscale);
        }
        for (int o = 0; o < oc; ++o) {
            float f = 0.f;
            for (int b = 0; b < blocks; ++b) {
                int32_t acc = 0, xsum = 0;
                const int32_t* ur = u + (size_t)o * ic;
                for (int k = b * bs; k < (b + 1) * bs; ++k) {
                    acc += (xq[k] + X86_OFFSET) * ur[k];
                    xsum += xq[k] + X86_OFFSET;
                }
                float part = (float)acc * alpha[(size_t)o * blocks + b];
                part = part * scale;
                if (b == 0) {
                    float corr = (scale * -128.f) * wks[o];
                    part = part + corr;
                }
                float zt = ((float)xsum * scale) * wb[(size_t)o * blocks + b];
                part = zt + part;
                f = b == 0 ? part : f + part;
            }
            if (tokens == 1) {
                float nb = wks[o] * izf;
                nb = (bias ? bias[o] : 0.0f) + nb;
                f = f + nb;
            } else if (bias) {
                f = f + bias[o];
            }
            if (relu || relu6) {
                float hi = relu6 ? 6.0f : 3.4028234663852886e38f;
                f = f < hi ? f : hi;
                f = f > 0.0f ? f : 0.0f;
            }
            y[(size_t)t * oc + o] = f;
        }
    }
    free(xq);
    free(u);
    free(wb);
    free(wks);
}
