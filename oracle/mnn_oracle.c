/*
 * mnn_oracle.c -- CPU restatement of the reference's int8 hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference leg may load this file's shared object.  It is the
 * checker, never the product: mnn_b200 fails loudly when its CUDA library is missing
 * and never calls into oracle/.
 *
 * What it restates: the arithmetic of alibaba/MNN's MNN_FORWARD_CPU backend on x86-64
 * (MNN_USE_SSE, AVX512-VNNI kernels) for
 *   - static-PTQ int8 Conv2D via im2col + int8 GEMM         (SURVEY 8a: a2, a3)
 *   - FloatToInt8 / Int8ToFloat boundary casts              (a10)
 *   - dynamic-quant W8A8 1x1 conv = MNN-LLM "quantized MatMul" (a7)
 *   - the int8 neighbours of the path (depthwise, eltwise add, pooling)  (8f rank 1)
 * Plain scalar loops over LOGICAL tensors (NCHW, int8 values without the x86 +128 storage
 * offset); every function cites the reference file:line it follows (paths relative to the
 * reference root).  Compile with -ffp-contract=off: the reference kernels are unfused
 * mul/add sequences and bit-exactness depends on that.
 *
 * Pinning: tests/test_oracle_vs_reference.py checks every function here bit-for-bit
 * against the UNMODIFIED reference built by oracle/build_ref.py (oracle/_ref/libMNN.so,
 * driven by oracle/refdump.cpp) on the reference's own ConvInt8Test generators, and
 * against committed golden fixtures (tests/golden/, made by tests/golden/make_golden.py).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORACLE_API __attribute__((visibility("default")))

/* x86 stores int8 activations as uint8 = value + 128 (source/backend/cpu/CPUConvolution.cpp:176-180,
 * compute/ConvInt8TiledExecutor.cpp:2269-2271).  The offset changes the float epilogue because the
 * 128*sum(w) correction is applied in float, so it is part of the arithmetic we must reproduce. */
#define X86_OFFSET 128

/* GemmInt8_VNNI.cpp:27-39 POSTTREAT: min, max, +-0.5, roundscale(3)=truncate. */
static inline int32_t post_round(float f, float minv, float maxv) {
    f = f < maxv ? f : maxv; /* _mm512_min_ps(f, max) */
    f = f > minv ? f : minv; /* _mm512_max_ps(f, min) */
    f = f + (f < 0.0f ? -0.5f : 0.5f);
    return (int32_t)truncf(f);
}

/* ------------------------------------------------------------------------------------------
 * a2: resize-time fold of tensor quant info into epilogue constants.
 * Modern models (op = Convolution, float bias + quanParameter.alpha, tensors carry quantAttr):
 *   CPUConvolution::MutableResourceInt8::updateInputOutputScale, CPUConvolution.cpp:144-201
 *   weightKernelSum[oc] = float(sum_k w_q) * alpha[oc]  (symmetric, blockNum=1),
 *   compute/ConvInt8TiledExecutor.cpp:243-267 (_computeReorderQuantInfo)
 *   biasFloat[oc] = (bias[oc] - wsum[oc]*(z_in+128)*s_in)/s_out + z_out   (:194-197)
 *   scaleX        = s_in / s_out   (compute/ConvInt8TiledExecutor.cpp:1967-1976)
 * ------------------------------------------------------------------------------------------ */
ORACLE_API void mnn_oracle_fold_modern(const int8_t* w, int oc, int kernel_len, const float* alpha,
                                       const float* bias, float s_in, int32_t z_in, float s_out,
                                       int32_t z_out, float* bias_float, float* scale_x) {
    for (int o = 0; o < oc; ++o) {
        int32_t isum = 0;
        for (int k = 0; k < kernel_len; ++k) isum += w[(size_t)o * kernel_len + k];
        float wsum = (float)isum * alpha[o] + (float)kernel_len * (0.0f * alpha[o]);
        float zoff = (float)z_in + 128.f;
        float t = wsum * zoff;
        t = t * s_in;
        float b = bias ? bias[o] : 0.0f;
        bias_float[o] = (b - t) / s_out + (float)z_out;
    }
    *scale_x = s_in / s_out;
}

/* Legacy models (op = ConvInt8, symmetricQuan{bias:int32, scale:float}): scale already contains
 * s_in*w_scale/s_out.  compute/ConvInt8TiledExecutor.cpp:796-805:
 *   bias_i32[oc] -= 128 * kernelsum[oc]     (float arithmetic, then truncated back to int32)
 * CPUConvolution.cpp:126-132 (mInputScale==0 when there is no quanParameter):
 *   biasFloat[oc] = float(bias_i32[oc]) * scale[oc]
 * and the GEMM is given inputScale = 1.0 (fakeInputScales, ConvInt8TiledExecutor.cpp:2187). */
ORACLE_API void mnn_oracle_fold_legacy(const int8_t* w, int oc, int kernel_len, const float* scale,
                                       const int32_t* bias_i32, float* bias_float, float* scale_x) {
    for (int o = 0; o < oc; ++o) {
        int32_t isum = 0;
        for (int k = 0; k < kernel_len; ++k) isum += w[(size_t)o * kernel_len + k];
        float ksum = (float)isum;
        int32_t b = bias_i32 ? bias_i32[o] : 0;
        float tmp = (float)b - 128.f * ksum; /* int32 -= float: evaluated in float */
        b = (int32_t)tmp;
        bias_float[o] = (float)b * scale[o];
    }
    *scale_x = 1.0f;
}

/* ------------------------------------------------------------------------------------------
 * a3: DenseConvInt8TiledExecutor::onExecute (static branch) + _AVX512_MNNGemmInt8AddBiasScale_16x4_Unit_VNNI
 *   compute/ConvInt8TiledExecutor.cpp:1914-2576 (params :2218-2245, im2col fill :2269-2271)
 *   x86_x64/avx512/GemmInt8_VNNI.cpp:122-415;  scalar twin compute/Int8FunctionsOpt.cpp:1555-1641
 *
 *   acc = sum_k (x_k + 128) * w_k   (int32; padded taps hold z_in + 128)
 *   f = float(acc) * wscale[oc];  f = f * scaleX;  f = f + 0 (symmetric weights);  f = f + biasFloat[oc]
 *   q = trunc(clamp(f, min, max) +- 0.5)
 * x: [n][ic][ih][iw] int8, w: [oc][ic][kh][kw] int8, y: [n][oc][oh][ow] int8.  group == 1.
 * ------------------------------------------------------------------------------------------ */
ORACLE_API void mnn_oracle_conv_int8(const int8_t* x, int n, int ic, int ih, int iw, const int8_t* w, int oc,
                                     int kh, int kw, int sh, int sw, int ph, int pw, int dh, int dw,
                                     const float* wscale, float scale_x, const float* bias_float,
                                     int32_t z_in, int32_t min_v, int32_t max_v, int8_t* y, int oh, int ow) {
    const float fmin = (float)min_v, fmax = (float)max_v;
    for (int b = 0; b < n; ++b)
        for (int o = 0; o < oc; ++o)
            for (int oy = 0; oy < oh; ++oy)
                for (int ox = 0; ox < ow; ++ox) {
                    int32_t acc = 0;
                    for (int c = 0; c < ic; ++c)
                        for (int ky = 0; ky < kh; ++ky) {
                            int iy = oy * sh + ky * dh - ph;
                            for (int kx = 0; kx < kw; ++kx) {
                                int ix = ox * sw + kx * dw - pw;
                                int32_t xv = z_in;
                                if (iy >= 0 && iy < ih && ix >= 0 && ix < iw)
                                    xv = x[(((size_t)b * ic + c) * ih + iy) * iw + ix];
                                acc += (xv + X86_OFFSET) * (int32_t)w[(((size_t)o * ic + c) * kh + ky) * kw + kx];
                            }
                        }
                    float f = (float)acc * wscale[o];
                    f = f * scale_x;
                    f = 0.0f * 0.0f + f; /* kernelSum * weightBias, symmetric => +0 */
                    f = f + bias_float[o];
                    y[(((size_t)b * oc + o) * oh + oy) * ow + ox] = (int8_t)post_round(f, fmin, fmax);
                }
}

/* ------------------------------------------------------------------------------------------
 * a10: boundary casts.
 *   CPUCastCreator::cast, source/backend/cpu/CPUCast.cpp:17-60 (scale -> 1/scale, 0 stays 0)
 *   _AVX512_MNNFloat2Int8 / _AVX512_MNNInt8ScaleToFloat, x86_x64/avx512/GemmInt8.cpp:234-347
 *   q = trunc(clamp(x*inv_scale + zero, min, max) +- 0.5);   x = (q - zero) * scale
 * ------------------------------------------------------------------------------------------ */
ORACLE_API void mnn_oracle_float_to_int8(const float* x, size_t count, float inv_scale, float zero,
                                         int32_t min_v, int32_t max_v, int8_t* y) {
    for (size_t i = 0; i < count; ++i) {
        /* _AVX512_MNNFloat2Int8 as SHIPPED: the avx512 directory is compiled with -mfma and GCC (-ffp-contract=fast by default)
         * fuses _mm256_mul_ps + _mm256_add_ps into vfmadd132ps (disassembly of oracle/_ref/libMNN.so); one rounding. */
        float f = fmaf(x[i], inv_scale, zero);
        y[i] = (int8_t)post_round(f, (float)min_v, (float)max_v);
    }
}

ORACLE_API float mnn_oracle_cast_inv_scale(float scale) { return scale == 0.f ? 0.f : 1.f / scale; }

ORACLE_API void mnn_oracle_int8_to_float(const int8_t* x, size_t count, float scale, float zero, float* y) {
    for (size_t i = 0; i < count; ++i) {
        /* (float(u8) - (zero + 128)) * scale with u8 = q + 128: float(q+128) and zero+128 are exact. */
        float u = (float)((int32_t)x[i] + X86_OFFSET);
        float z = zero + 128.f;
        y[i] = (u - z) * scale;
    }
}

/* ------------------------------------------------------------------------------------------
 * a7: the MNN-LLM linear layer = Convolution 1x1 with int8 weights, CPU Memory_Low path:
 *   DenseConvInt8TiledExecutor dynamic branch, compute/ConvInt8TiledExecutor.cpp:1990-2096
 *   MNNAbsMax / MNNQuantScaleFP32 (compute/CommonOptFunction.cpp:79-94, 310-330)
 *   _AVX512_DynamicQuant (x86_x64/avx512/PackedFunction.cpp:288-348): round-to-nearest-EVEN
 *   float-output GEMM tail, x86_x64/avx512/GemmInt8_VNNI.cpp:262-470
 *   weightKernelSum: compute/ConvInt8TiledExecutor.cpp:226-267
 *
 *   per token: absmax -> qscale = 127/absmax, dq = absmax/127 (both 1 if absmax < 1e-7)
 *   xq = rne(x*qscale);   acc = sum_k (xq_k + 128) * wq_k
 *   f = float(acc)*alpha[oc];  f *= dq;  f += (dq * -128) * wsum[oc];
 *   f += (float(sum_k (xq_k+128)) * dq) * wzero[oc];   f += bias[oc];  optional relu/relu6 clamp
 * x: [tokens][ic] float, wq: [oc][ic] int8, y: [tokens][oc] float.  wzero may be NULL (symmetric).
 * ------------------------------------------------------------------------------------------ */
ORACLE_API void mnn_oracle_linear_w8_dynamic(const float* x, int tokens, int ic, const int8_t* wq, int oc,
                                             const float* alpha, const float* wzero, const float* bias,
                                             int relu, int relu6, float* y) {
    int32_t* xq = (int32_t*)malloc(sizeof(int32_t) * (size_t)ic);
    float* wsum = (float*)malloc(sizeof(float) * (size_t)oc);
    for (int o = 0; o < oc; ++o) {
        int32_t isum = 0;
        for (int k = 0; k < ic; ++k) isum += wq[(size_t)o * ic + k];
        float zb = wzero ? wzero[o] : 0.0f * alpha[o];
        wsum[o] = (float)isum * alpha[o] + (float)ic * zb;
    }
    if (tokens == 1) {
        /* ONE token (the decode step): inputPlane == 1 leaves mUseBatchQuan false (ConvInt8TiledExecutor.cpp:1033-1035), so the
         * input is quantised ASYMMETRICALLY with one {scale, zero} for the whole row and the zero point is folded into the bias
         * (mToFuseInputbias2Bias, :1432, :2016-2050):
         *   min / max over the row INCLUDING the zero padding of the last 16-channel pack (x86_x64/avx512/PackedFunction.cpp:133-165,
         *   _AVX512_MNNAsyQuantInfo info[7] == 1: kernelsize * stride0 floats of the NC16HW16 buffer);
         *   range <= 1e-7: scale = qscale = 1, qbias = -max;  else qscale = 255 / range, scale = range / 255,
         *   qbias = roundf(-min * 255 / range) - 128;
         *   q = FloatToInt8(x; qscale, qbias, [-128, 127]) -- the fma-contracted AVX512 cast, see mnn_oracle_float_to_int8;
         *   bias'[oc] = bias[oc] + weightKernelSum[oc] * (-qbias * scale)   (MNNDynamicUpdateConvBiasScale, CommonOptFunction.cpp:96-103);
         *   then the same GEMM epilogue with the constant input scale.  Pinned on the live reference (tests/test_oracle.py,
         *   tests/golden/dw_linear_golden.npz decode cases): <= 1e-6 relative (the remainder-channel path of the x86 kernel
         *   contracts one mul + add pair, which moves single ulps). */
        float mn = x[0], mx = x[0];
        for (int k = 1; k < ic; ++k) { mn = x[k] < mn ? x[k] : mn; mx = x[k] > mx ? x[k] : mx; }
        if (ic % 16 != 0) { mn = mn < 0.f ? mn : 0.f; mx = mx > 0.f ? mx : 0.f; }
        float range = mx - mn, scale, qscale, qbias;
        if (range <= 1e-7) { scale = 1.f; qscale = 1.f; qbias = -mx; }
        else {
            qscale = 255.f / range;
            scale = range / 255.f;
            float t0 = -mn * 255.f;
            qbias = roundf(t0 / range) - 128.0f;
        }
        int32_t xsum = 0;
        for (int k = 0; k < ic; ++k) {
            float v = fmaf(x[k], qscale, qbias);
            v = v > -128.f ? v : -128.f;
            v = v < 127.f ? v : 127.f;
            v = v + (v < 0.f ? -0.5f : 0.5f);
            xq[k] = (int32_t)v;
            xsum += xq[k] + X86_OFFSET;
        }
        float srcsum = (float)xsum * scale;
        float izf = -qbias * scale;
        for (int o = 0; o < oc; ++o) {
            int32_t acc = 0;
            const int8_t* wr = wq + (size_t)o * ic;
            for (int k = 0; k < ic; ++k) acc += (xq[k] + X86_OFFSET) * (int32_t)wr[k];
            float nb = wsum[o] * izf;
            nb = (bias ? bias[o] : 0.0f) + nb;
            float f = (float)acc * alpha[o];
            f = f * scale;
            float corr = (scale * -128.f) * wsum[o];
            f = f + corr;
            float zt = srcsum * (wzero ? wzero[o] : 0.0f);
            f = zt + f;
            f = f + nb;
            if (relu || relu6) {
                float hi = relu6 ? 6.0f : 3.4028234663852886e38f;
                f = f < hi ? f : hi;
                f = f > 0.0f ? f : 0.0f;
            }
            y[o] = f;
        }
        free(xq);
        free(wsum);
        return;
    }
    for (int t = 0; t < tokens; ++t) {
        const float* xr = x + (size_t)t * ic;
        float absmax = 0.f;
        for (int k = 0; k < ic; ++k) {
            float a = fabsf(xr[k]);
            absmax = a > absmax ? a : absmax;
        }
        float qscale = 1.f, dq = 1.f;
        if (!(absmax < 1e-7)) {
            qscale = 127.0f / absmax;
            dq = absmax / 127.0f;
        }
        int32_t xsum = 0;
        for (int k = 0; k < ic; ++k) {
            xq[k] = (int32_t)nearbyintf(xr[k] * qscale); /* default rounding mode = nearest-even */
            xsum += xq[k] + X86_OFFSET;
        }
        float srcsum = (float)xsum * dq;
        for (int o = 0; o < oc; ++o) {
            int32_t acc = 0;
            const int8_t* wr = wq + (size_t)o * ic;
            for (int k = 0; k < ic; ++k) acc += (xq[k] + X86_OFFSET) * (int32_t)wr[k];
            float f = (float)acc * alpha[o];
            f = f * dq;
            float corr = (dq * -128.f) * wsum[o];
            f = f + corr;
            float zt = srcsum * (wzero ? wzero[o] : 0.0f);
            f = zt + f;
            if (bias) f = f + bias[o];
            if (relu || relu6) {
                float hi = relu6 ? 6.0f : 3.4028234663852886e38f;
                f = f < hi ? f : hi;
                f = f > 0.0f ? f : 0.0f;
            }
            y[(size_t)t * oc + o] = f;
        }
    }
    free(xq);
    free(wsum);
}

/* ------------------------------------------------------------------------------------------
 * a7 with K-BLOCKED weight scales (MNN-LLM's default export: quant_block 64 / 128): alpha[oc][blocks], wzero[oc][blocks],
 * K split into `blocks` equal runs.  ConvInt8TiledExecutor.cpp: mBlockNum (:1058), the per-block int32 accumulators of the
 * GEMM kernel are converted and summed in fp32 block after block (:2290-2440, accumbuff); the input is still quantised per TOKEN
 * (mInputBlockNum == 1 unless dynamicQuantOption == 2).  Two or more tokens: symmetric per-token quant; ONE token: the
 * single-quant decode arithmetic of mnn_oracle_linear_w8_dynamic with weightKernelSum summed over the blocks.
 * NOT on the CUDA path yet (the plugin declines block-wise layers); this restatement is the oracle the kernel will be built
 * against.  Pinned on the live reference (tests/test_oracle.py, tests/golden/block_linear_golden.npz): <= 4e-6 relative -- the
 * x86 kernel sums the blocks in a different association, so single ulps differ; the tolerance of an fp32 output is 1e-3.
 * ------------------------------------------------------------------------------------------ */
ORACLE_API void mnn_oracle_linear_w8_dynamic_blocks(const float* x, int tokens, int ic, const int8_t* wq, int oc,
                                                    const float* alpha, const float* wzero, const float* bias, int blocks,
                                                    int relu, int relu6, float* y) {
    const int bs = ic / blocks;
    int32_t* xq = (int32_t*)malloc(sizeof(int32_t) * (size_t)ic);
    float* wsum = (float*)malloc(sizeof(float) * (size_t)oc * blocks);
    for (int o = 0; o < oc; ++o)
        for (int b = 0; b < blocks; ++b) {
            int32_t isum = 0;
            for (int k = b * bs; k < (b + 1) * bs; ++k) isum += wq[(size_t)o * ic + k];
            float zb = wzero ? wzero[(size_t)o * blocks + b] : 0.0f;
            wsum[(size_t)o * blocks + b] = (float)isum * alpha[(size_t)o * blocks + b] + (float)bs * zb;
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
            float f = 0.f, wtot = 0.f;
            for (int b = 0; b < blocks; ++b) {
                int32_t acc = 0, xsum = 0;
                const int8_t* wr = wq + (size_t)o * ic;
                for (int k = b * bs; k < (b + 1) * bs; ++k) {
                    acc += (xq[k] + X86_OFFSET) * (int32_t)wr[k];
                    xsum += xq[k] + X86_OFFSET;
                }
                const float ws = wsum[(size_t)o * blocks + b];
                float part = (float)acc * alpha[(size_t)o * blocks + b];
                part = part * scale;
                float corr = (scale * -128.f) * ws;
                part = part + corr;
                float zt = ((float)xsum * scale) * (wzero ? wzero[(size_t)o * blocks + b] : 0.0f);
                part = zt + part;
                f = f + part;
                wtot = wtot + ws;
            }
            if (tokens == 1) {
                float nb = wtot * izf;
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
    free(wsum);
}

/* ------------------------------------------------------------------------------------------
 * 8f rank 1: depthwise int8 conv.
 *   CPUDepthwiseConvInt8 (source/backend/cpu/CPUDepthwiseConvInt8.cpp) with
 *   MutableResourceInt8::updateInputOutputScale depthwise branch, CPUConvolution.cpp:181-192:
 *     ws = |wscale| < 1e-6 ? 1e-6 : wscale;  scale = ws * (s_in/s_out)
 *     bias_i32 = int(bias/(s_in*ws)) - sum(w)*(z_in+128) + int(z_out/scale)
 *   kernel MNNLineDepthWiseInt8AddBiasScaleUnit, compute/Int8FunctionsOpt.cpp:1767-1814
 *   (x86: _AVX512/_AVX_ twin): acc = bias_i32 + sum (x+128)*w ; f = float(acc)*scale ;
 *     q = trunc(f +- 0.5) then clamp to [min,max]
 * x: [n][c][ih][iw], w: [c][kh][kw].
 * ------------------------------------------------------------------------------------------ */
ORACLE_API void mnn_oracle_fold_depthwise(const int8_t* w, int c, int kernel_len, const float* wscale,
                                          const float* bias, float s_in, int32_t z_in, float s_out,
                                          int32_t z_out, float* scale, int32_t* bias_i32) {
    float scale_div = s_in / s_out;
    for (int o = 0; o < c; ++o) {
        int32_t isum = 0;
        for (int k = 0; k < kernel_len; ++k) isum += w[(size_t)o * kernel_len + k];
        float ws = wscale[o];
        if (fabs(ws) < 1e-6) ws = 1e-6;
        scale[o] = ws * scale_div;
        int32_t zfused = (int32_t)((float)z_out / scale[o]);
        float b = bias ? bias[o] : 0.0f;
        /* int - float*float + int : evaluated in float, truncated on assignment */
        float v = (float)(int32_t)(b / (s_in * ws)) - (float)isum * ((float)z_in + 128.f) + (float)zfused;
        bias_i32[o] = (int32_t)v;
    }
}

ORACLE_API void mnn_oracle_depthwise_int8(const int8_t* x, int n, int c, int ih, int iw, const int8_t* w, int kh,
                                          int kw, int sh, int sw, int ph, int pw, int dh, int dw,
                                          const float* scale, const int32_t* bias_i32, int32_t z_in,
                                          int32_t min_v, int32_t max_v, int8_t* y, int oh, int ow) {
    for (int b = 0; b < n; ++b)
        for (int ch = 0; ch < c; ++ch)
            for (int oy = 0; oy < oh; ++oy)
                for (int ox = 0; ox < ow; ++ox) {
                    int32_t acc = bias_i32[ch];
                    for (int ky = 0; ky < kh; ++ky) {
                        int iy = oy * sh + ky * dh - ph;
                        for (int kx = 0; kx < kw; ++kx) {
                            int ix = ox * sw + kx * dw - pw;
                            int32_t xv = z_in;
                            if (iy >= 0 && iy < ih && ix >= 0 && ix < iw)
                                xv = x[(((size_t)b * c + ch) * ih + iy) * iw + ix];
                            acc += (xv + X86_OFFSET) * (int32_t)w[((size_t)ch * kh + ky) * kw + kx];
                        }
                    }
                    float f = (float)acc * scale[ch];
                    f = f + (f < 0.0f ? -0.5f : 0.5f);
                    int32_t q = (int32_t)truncf(f);
                    q = q > max_v ? max_v : q;
                    q = q < min_v ? min_v : q;
                    y[(((size_t)b * c + ch) * oh + oy) * ow + ox] = (int8_t)q;
                }
}

/* ------------------------------------------------------------------------------------------
 * 8f rank 1: int8 elementwise add.  CPUBinaryInt8 + MNNBinaryAddInt8
 *   source/backend/cpu/CPUBinaryInt8.cpp:21-64, compute/Int8FunctionsOpt.cpp:1926-1975
 *   a = float(q0 - z0) * s0;  b = float(q1 - z1) * s1;  sum = a + b
 *   v = (int)roundf(sum * (1 / s_out)) + z_out;  clamp to [min, max]     (1/s_out is 0 when s_out == 0)
 * ------------------------------------------------------------------------------------------ */
ORACLE_API void mnn_oracle_binary_add_int8(const int8_t* x0, float s0, int32_t z0, const int8_t* x1, float s1,
                                           int32_t z1, size_t count, float s_out, int32_t z_out, int32_t min_v,
                                           int32_t max_v, int8_t* y) {
    float inv = s_out != 0 ? 1 / s_out : 0;
    for (size_t i = 0; i < count; ++i) {
        float a = (float)((int32_t)x0[i] - z0) * s0;
        float b = (float)((int32_t)x1[i] - z1) * s1;
        float sum = a + b;
        int32_t v = (int32_t)roundf(sum * inv) + z_out;
        v = v > max_v ? max_v : v;
        v = v < min_v ? min_v : v;
        y[i] = (int8_t)v;
    }
}

/* ------------------------------------------------------------------------------------------
 * 8f rank 1: average pooling between int8 tensors whose quant attrs DIFFER: the pipeline brackets the float
 * pooling with casts (source/core/Pipeline.cpp:367-395; CPUBackend.cpp:925-936 refuses int8 pooling then):
 *   Int8ToFloat (a10)  ->  poolingAvg<float> (source/backend/cpu/CPUPool.hpp:271-394)  ->  FloatToInt8 (a10)
 * interior windows: sum = sum + x * (1/count), taps in (kh, kw) order, unfused;
 * windows touching padding: (sum of valid x) * (1/count'), count' per AvgPoolCountType (DEFAULT: CAFFE pad
 * type counts padding, others exclude it).  x: [n][c][ih][iw] int8.
 * ------------------------------------------------------------------------------------------ */
ORACLE_API void mnn_oracle_avgpool_int8_via_float(const int8_t* x, int n, int c, int ih, int iw, int kh, int kw,
                                                  int sh, int sw, int ph, int pw, int pad_type, int count_type,
                                                  float s_in, float z_in, float s_out, float z_out, int32_t min_v,
                                                  int32_t max_v, int8_t* y, int oh, int ow) {
    float inv_out = mnn_oracle_cast_inv_scale(s_out);
    if (count_type == 0) count_type = pad_type == 0 ? 1 : 2; /* DEFAULT -> INCLUDE_PADDING for CAFFE, else EXCLUDE */
    for (int b = 0; b < n; ++b)
        for (int ch = 0; ch < c; ++ch)
            for (int oy = 0; oy < oh; ++oy)
                for (int ox = 0; ox < ow; ++ox) {
                    int iy0 = oy * sh - ph, ix0 = ox * sw - pw;
                    int interior = iy0 >= 0 && ix0 >= 0 && iy0 + kh <= ih && ix0 + kw <= iw;
                    float sum = 0.0f, res;
                    const int8_t* xp = x + ((size_t)b * c + ch) * ih * iw;
                    if (interior) {
                        float div = 1.0f / (float)(kh * kw);
                        for (int ky = 0; ky < kh; ++ky)
                            for (int kx = 0; kx < kw; ++kx) {
                                float xf;
                                mnn_oracle_int8_to_float(&xp[(iy0 + ky) * iw + ix0 + kx], 1, s_in, z_in, &xf);
                                float t = xf * div;
                                sum = sum + t;
                            }
                        res = sum;
                    } else {
                        int khs = 0 < -iy0 ? -iy0 : 0, khe = kh < ih - iy0 ? kh : ih - iy0;
                        int kws = 0 < -ix0 ? -ix0 : 0, kwe = kw < iw - ix0 ? kw : iw - ix0;
                        int count;
                        if (count_type == 1) {
                            int ye = iy0 + kh < ih + ph ? iy0 + kh : ih + ph, xe = ix0 + kw < iw + pw ? ix0 + kw : iw + pw;
                            count = (ye - iy0) * (xe - ix0);
                        } else {
                            count = (khe - khs) * (kwe - kws);
                        }
                        for (int ky = khs; ky < khe; ++ky)
                            for (int kx = kws; kx < kwe; ++kx) {
                                float xf;
                                mnn_oracle_int8_to_float(&xp[(iy0 + ky) * iw + ix0 + kx], 1, s_in, z_in, &xf);
                                sum = sum + xf;
                            }
                        res = count > 0 ? sum * (1.0f / (float)count) : 0.0f;
                    }
                    mnn_oracle_float_to_int8(&res, 1, inv_out, z_out, min_v, max_v,
                                             &y[(((size_t)b * c + ch) * oh + oy) * ow + ox]);
                }
}

/* ------------------------------------------------------------------------------------------
 * 8f rank 2: Softmax on an int8 tensor (CPUSoftmax, mLowOrInt8 == 1, source/backend/cpu/CPUSoftmax.cpp:85-150):
 * Int8ToFloat -> fp32 softmax (max, sub, exp, sum, reciprocal, mul) -> FloatToInt8.  The reference evaluates exp
 * with its own polynomial (MNNExp); this restatement uses expf, so the int8 result is specified to +-1 LSB
 * (fp32 internal path: north_star's 1e-3 relative on the dequantised value).  x: [rows][c].
 * ------------------------------------------------------------------------------------------ */
ORACLE_API void mnn_oracle_softmax_int8(const int8_t* x, int rows, int c, float s_in, float z_in, float s_out,
                                        float z_out, int32_t min_v, int32_t max_v, int8_t* y) {
    float inv_out = mnn_oracle_cast_inv_scale(s_out);
    float* t = (float*)malloc(sizeof(float) * (size_t)c);
    for (int r = 0; r < rows; ++r) {
        mnn_oracle_int8_to_float(x + (size_t)r * c, (size_t)c, s_in, z_in, t);
        float mx = t[0];
        for (int i = 1; i < c; ++i) mx = t[i] > mx ? t[i] : mx;
        float sum = 0.f;
        for (int i = 0; i < c; ++i) { t[i] = expf(t[i] - mx); sum += t[i]; }
        float rs = 1.0f / sum;
        for (int i = 0; i < c; ++i) t[i] = t[i] * rs;
        mnn_oracle_float_to_int8(t, (size_t)c, inv_out, z_out, min_v, max_v, y + (size_t)r * c);
    }
    free(t);
}

/* ==========================================================================================
 * a5: int8 Winograd convolution -- ConvInt8Winograd (compute/ConvInt8Winograd.cpp, whole file).
 *
 * The reference arithmetic restated here is the x86 **AVX2** build (pack 8, MNN_USE_SSE, no FMA
 * in x86_x64/avx): the AVX512 build of this op is known-wrong upstream (SURVEY F8), so the
 * pinning target is oracle/_ref/libMNN_avx2.so.  Transform coefficient sequences follow
 *   x86_x64/avx/WinogradFunctions.cpp:358-553 (source 4x4 / 6x6 / 8x8),
 *   :555-579 (dest 4->2), :661-712 (dest 6->4), :981-1051 (dest 8->6);
 * Vec8::fma(a,b,c) = a + b*c with separate rounding (x86_x64/avx/Vec8.hpp:187-190).
 * One unit covering the whole kernel (kyStart = kxStart = 0), kernel 3x3, unit 2 / 4 / 6.
 * ========================================================================================== */

/* Math::WinogradGenerater(unit, kernel, interp=1, dividedInG=true): G only.
 * source/math/WingoradGenerater.cpp:96-135 (computeA, computeFDiag), :139-222.  g: [alpha][r]. */
static void wino_make_g(int unit, int r, float* g) {
    int alpha = unit + r - 1;
    float a[16];
    a[0] = 0.0f;
    int sign = 1;
    for (int i = 0; i < alpha - 1; ++i) {
        int value = 1 + i / 2;
        a[i + 1] = (float)(sign * value) * 1.0f;
        sign *= -1;
    }
    float fdiag[16];
    for (int x = 0; x < alpha - 1; ++x) {
        float product = 1.0f;
        for (int i = 0; i < alpha - 1; ++i) {
            if (x == i) continue;
            product *= (a[x] - a[i]);
        }
        fdiag[x] = product;
    }
    fdiag[alpha - 1] = 1.0f;
    if (fdiag[0] < 0) fdiag[0] = -fdiag[0];
    /* computeA(a, m=alpha, n=r) transposed: G[x][y] */
    for (int x = 0; x < alpha; ++x)
        for (int y = 0; y < r; ++y) {
            float v;
            if (x < alpha - 1) v = (x == 0 && y == 0) ? 1.0f : powf(a[x], (float)y);
            else v = (y == r - 1) ? 1.0f : 0.0f;
            g[x * r + y] = v / fdiag[x]; /* Matrix::divPerLine, source/math/Matrix.cpp:346-364 */
        }
}

/* makeWinoResource (ConvInt8Winograd.cpp:25-126): float-transform the dequantised weights, requantise per
 * (position, oc), build the per-(position, oc) float scale and offset.
 * wq_out [alpha2][oc][ic] int8, scale_out/offset_out [alpha2][oc]. */
ORACLE_API void mnn_oracle_wino_weights(const int8_t* w, int oc, int ic, int r, int unit, const float* wscale,
                                        const float* in_scales, const int32_t* in_zeros, const float* w_scales,
                                        int8_t* wq_out, float* scale_out, float* offset_out) {
    int alpha = unit + r - 1, alpha2 = alpha * alpha;
    float g[16 * 8];
    wino_make_g(unit, r, g);
    float* wt = (float*)malloc(sizeof(float) * (size_t)alpha2 * oc * ic);
    for (int o = 0; o < oc; ++o)
        for (int c = 0; c < ic; ++c) {
            float k[64], m[16 * 8], kt[256];
            for (int i = 0; i < r * r; ++i) k[i] = (float)w[((size_t)o * ic + c) * r * r + i] * wscale[o];
            /* M = G * K ; K_Transform = M * G^T   (Matrix::multi, source/math/Matrix.cpp:41-78) */
            for (int y = 0; y < alpha; ++y)
                for (int x = 0; x < r; ++x) {
                    float sum = 0.0f;
                    for (int i = 0; i < r; ++i) sum += g[y * r + i] * k[i * r + x];
                    m[y * r + x] = sum;
                }
            for (int y = 0; y < alpha; ++y)
                for (int x = 0; x < alpha; ++x) {
                    float sum = 0.0f;
                    for (int i = 0; i < r; ++i) sum += m[y * r + i] * g[x * r + i];
                    kt[y * alpha + x] = sum;
                }
            for (int i = 0; i < alpha2; ++i) wt[((size_t)i * oc + o) * ic + c] = kt[i];
        }
    for (int a = 0; a < alpha2; ++a)
        for (int o = 0; o < oc; ++o) {
            float offset = 0.f;
            float scale = w_scales[a * oc + o];
            for (int c = 0; c < ic; ++c) {
                float src = wt[((size_t)a * oc + o) * ic + c];
                float eps = (float)(((src / scale) > 0 ? 1 : -1) * 1e-6);
                float rv = roundf(src / scale + eps);
                rv = rv > -127.f ? rv : -127.f;
                rv = rv < 127.f ? rv : 127.f;
                int8_t q = (int8_t)rv;
                wq_out[((size_t)a * oc + o) * ic + c] = q;
                offset += (float)((int)q * (-in_zeros[a]));
                offset += (float)((int)q * (-128)); /* MNN_USE_SSE */
            }
            offset_out[a * oc + o] = offset * scale * in_scales[a];
            scale_out[a * oc + o] = scale * in_scales[a];
        }
    free(wt);
}

static void wino_src(int alpha, const float* b, float* m) {
    if (alpha == 4) {
        m[0] = b[0] - b[2]; m[1] = b[1] + b[2]; m[2] = b[2] - b[1]; m[3] = b[3] - b[1];
    } else if (alpha == 6) {
        float mid0 = b[4] + b[2] * -4.f, mid1 = b[3] + b[1] * -4.f, mid2 = b[2] + b[0] * -4.f, mid3 = b[5] + b[3] * -4.f;
        float mid4 = b[4] - b[2], mid5 = (b[3] - b[1]) * 2.f;
        m[0] = mid0 - mid2; m[1] = mid0 + mid1; m[2] = mid0 - mid1; m[3] = mid4 + mid5; m[4] = mid4 - mid5; m[5] = mid3 - mid1;
    } else {
        float mid0, mid1, mid2;
        mid0 = (b[6] + b[2] * 36.f) + b[4] * -13.f;
        mid1 = (b[4] + b[0] * 36.f) + b[2] * -13.f;
        m[0] = mid1 - mid0;
        mid2 = (b[5] + b[1] * 36.f) + b[3] * -13.f;
        m[1] = mid0 + mid2; m[2] = mid0 - mid2;
        mid1 = (b[7] + b[3] * 36.f) + b[5] * -13.f;
        m[7] = mid1 - mid2;
        mid0 = (b[6] + b[2] * 9.f) + b[4] * -10.f;
        mid1 = (b[5] + b[1] * 18.f) + (b[5] + b[3] * -20.f);
        mid2 = (b[5] * 3.f) + b[1] * 12.f;
        m[3] = mid0 + mid1; m[4] = mid0 - mid1;
        mid0 = (b[6] + b[2] * 4.f) + b[4] * -5.f;
        mid1 = mid2 + b[3] * -15.f;
        m[5] = mid0 + mid1; m[6] = mid0 - mid1;
    }
}
static void wino_dst(int alpha, const float* s, float* m) {
    if (alpha == 4) {
        m[0] = (s[0] + s[1]) + s[2]; m[1] = (s[1] - s[2]) + s[3];
    } else if (alpha == 6) {
        float v0 = s[3] + s[4], v1 = s[3] - s[4], v2 = s[1] + s[2], v3 = s[1] - s[2];
        m[0] = (s[0] + v2) + v0; m[1] = (v3 + v1) + v1; m[2] = v2 + v0 * 4.f; m[3] = (v3 + v1 * 8.f) + s[5];
    } else {
        float mid0 = s[1] + s[2], mid1 = s[1] - s[2], mid2 = s[3] + s[4], mid3 = s[3] - s[4], mid4 = s[5] + s[6], mid5 = s[5] - s[6];
        m[0] = ((s[0] + mid0) + mid2) + mid4;
        m[1] = (mid1 + mid3 * 2.f) + mid5 * 3.f;
        m[2] = (mid0 + mid2 * 4.f) + mid4 * 9.f;
        m[3] = (mid1 + mid3 * 8.f) + mid5 * 27.f;
        m[4] = (mid0 + mid2 * 16.f) + mid4 * 81.f;
        m[5] = ((mid1 + mid3 * 32.f) + mid5 * 243.f) + s[7];
    }
}

/* ConvInt8Winograd::onExecute + WinoExecution::onExecute + mergeAddBiasScaleQuantize
 * (ConvInt8Winograd.cpp:306-356, 396-651, 243-259).  x [n][ic][ih][iw] int8, y [n][oc][oh][ow] int8,
 * stride 1, dilation 1, kernel r x r, begin pads pad_h (rows) and pad_w (columns), each also added at the end (CAFFE).
 * clamp: min = relu ? z_out : clamp_min. */
ORACLE_API void mnn_oracle_wino_conv_int8(const int8_t* x, int n, int ic, int ih, int iw, const int8_t* w, int oc, int r,
                                          int pad_h, int pad_w, int unit, const float* wscale, const float* bias,
                                          const float* in_scales, const int32_t* in_zeros, const float* w_scales,
                                          float s_in, int32_t z_in, float s_out, int32_t z_out, int32_t clamp_min,
                                          int32_t clamp_max, int relu, int8_t* y) {
    int alpha = unit + r - 1, alpha2 = alpha * alpha;
    int oh = ih + 2 * pad_h - r + 1, ow = iw + 2 * pad_w - r + 1;
    int hU = (oh + unit - 1) / unit, wU = (ow + unit - 1) / unit;
    int8_t* wq = (int8_t*)malloc((size_t)alpha2 * oc * ic);
    float* sc = (float*)malloc(sizeof(float) * alpha2 * oc);
    float* of = (float*)malloc(sizeof(float) * alpha2 * oc);
    mnn_oracle_wino_weights(w, oc, ic, r, unit, wscale, in_scales, in_zeros, w_scales, wq, sc, of);
    uint8_t* v = (uint8_t*)malloc((size_t)alpha2 * ic); /* x86 storage: q + 128 */
    float* mo = (float*)malloc(sizeof(float) * alpha2 * oc);
    float out_inv = (float)(1.0 / (double)s_out); /* float outputdequantScale = 1.0 / mOutputScale, :340 */
    float fmin = (float)(relu ? z_out : clamp_min), fmax = (float)clamp_max;
    for (int b = 0; b < n; ++b)
        for (int hy = 0; hy < hU; ++hy)
            for (int wx = 0; wx < wU; ++wx) {
                int sy0 = hy * unit - pad_h, sx0 = wx * unit - pad_w;
                for (int c = 0; c < ic; ++c) {
                    float d[64], t1[64], t2[64];
                    for (int yy = 0; yy < alpha; ++yy)
                        for (int xx = 0; xx < alpha; ++xx) {
                            int iy = sy0 + yy, ix = sx0 + xx;
                            float f = 0.0f; /* zero padded in float, :483 */
                            if (iy >= 0 && iy < ih && ix >= 0 && ix < iw) {
                                /* MNNInt8ScaleToFloat (avx/GemmInt8.cpp:1545-1590): (u8 - (zero + 128)) * scale */
                                f = ((float)((int)x[(((size_t)b * ic + c) * ih + iy) * iw + ix] + 128) - ((float)z_in + 128.f)) * s_in;
                            }
                            d[yy * alpha + xx] = f;
                        }
                    /* srcTransXFunc: along x for every row; then srcTransYFunc: along y for every column (:499-500) */
                    for (int yy = 0; yy < alpha; ++yy) wino_src(alpha, d + yy * alpha, t1 + yy * alpha);
                    for (int k = 0; k < alpha; ++k) {
                        float col[8], res[8];
                        for (int yy = 0; yy < alpha; ++yy) col[yy] = t1[yy * alpha + k];
                        wino_src(alpha, col, res);
                        for (int j = 0; j < alpha; ++j) t2[j * alpha + k] = res[j];
                    }
                    for (int a = 0; a < alpha2; ++a) {
                        /* MNNFloat2Int8(scale = 1/inputScale[a], -127, 127, zero = inputZero[a]) (:553) */
                        float inv = 1.0f / in_scales[a];
                        float f = t2[a] * inv + (float)in_zeros[a];
                        v[(size_t)a * ic + c] = (uint8_t)(post_round(f, -127.f, 127.f) + 128);
                    }
                }
                for (int a = 0; a < alpha2; ++a)
                    for (int o = 0; o < oc; ++o) {
                        int32_t acc = 0;
                        for (int c = 0; c < ic; ++c) acc += (int32_t)v[(size_t)a * ic + c] * (int32_t)wq[((size_t)a * oc + o) * ic + c];
                        /* _AVX_MNNGemmInt8AddBiasScale_16x4_Unit float-output branch (avx/GemmInt8.cpp:672-772):
                         * f = float(acc)*scale; *= inputScale(1.0); += (1*-128)*wKernelSum(0); += srcSum(0)*wBias(0); += offset */
                        float f = (float)acc * sc[a * oc + o];
                        f = f * 1.0f;
                        f = f + (1.0f * -128.f) * 0.0f;
                        f = f + 0.0f * 0.0f;
                        f = f + of[a * oc + o];
                        mo[(size_t)a * oc + o] = f;
                    }
                for (int o = 0; o < oc; ++o) {
                    float t1[64], t2[64];
                    /* dstTransYFunc[alphaX]: along y for every column k; dstTransXFunc: along x for every output row (:623-624) */
                    for (int k = 0; k < alpha; ++k) {
                        float col[8], res[8];
                        for (int j = 0; j < alpha; ++j) col[j] = mo[(size_t)(j * alpha + k) * oc + o];
                        wino_dst(alpha, col, res);
                        for (int j = 0; j < unit; ++j) t1[j * alpha + k] = res[j];
                    }
                    for (int j = 0; j < unit; ++j) wino_dst(alpha, t1 + j * alpha, t2 + j * unit);
                    float fused = (bias ? bias[o] : 0.f) / s_out + (float)z_out; /* mFusedBias, :215-217 */
                    for (int j = 0; j < unit; ++j)
                        for (int i = 0; i < unit; ++i) {
                            int oy = hy * unit + j, ox = wx * unit + i;
                            if (oy >= oh || ox >= ow) continue;
                            float f = t2[j * unit + i] * out_inv + fused; /* MNNFloat2Int8 mode 2, :255-258 */
                            y[(((size_t)b * oc + o) * oh + oy) * ow + ox] = (int8_t)post_round(f, fmin, fmax);
                        }
                }
            }
    free(wq); free(sc); free(of); free(v); free(mo);
}

/* The transforms above as matrices (applied to unit vectors): bt [alpha][alpha], at [unit][alpha], g [alpha][r].
 * Used by the tests to calibrate per-position quantisation scales (the reference has no calibration on this path:
 * the quantisation tool writes the attr offline). */
ORACLE_API void mnn_oracle_wino_matrices(int unit, int r, float* bt, float* at, float* g) {
    int alpha = unit + r - 1;
    for (int i = 0; i < alpha; ++i) {
        float e[8] = {0}, o[8];
        e[i] = 1.0f;
        wino_src(alpha, e, o);
        for (int j = 0; j < alpha; ++j) bt[j * alpha + i] = o[j];
        wino_dst(alpha, e, o);
        for (int j = 0; j < unit; ++j) at[j * alpha + i] = o[j];
    }
    wino_make_g(unit, r, g);
}

/* ==========================================================================================
 * int8 pooling when input and output share their quant attrs (CPUBackend::onSetQuantInfo keeps the op in int8,
 * CPUBackend.cpp:930-941) -- CPUPoolInt8 (source/backend/cpu/CPUPoolInt8.cpp:19-190) with the x86 kernels
 * (x86_x64/FunctionDispatcher.cpp:122-168).  x86 stores int8 tensors as u = q + 128 and these two kernels work on the stored
 * bytes:
 *   AVE: out_u = (sum_u * floor(2^24 / count)) >> 24 in uint32, count = taps inside the image (padding excluded);
 *   MAX: the stored bytes are compared as SIGNED int8 (so q >= 0, stored 128..255, ranks below every q < 0) -- restated as is.
 * x, y: [n][c][h][w] int8 (logical values).  Window geometry as CPUPoolInt8::onResize (:180-215).
 * ========================================================================================== */
ORACLE_API void mnn_oracle_pool_int8_x86(const int8_t* x, int n, int c, int ih, int iw, int kh, int kw, int sh, int sw,
                                         int ph, int pw, int is_avg, int8_t* y, int oh, int ow) {
    for (int b = 0; b < n; ++b)
        for (int ch = 0; ch < c; ++ch)
            for (int oy = 0; oy < oh; ++oy)
                for (int ox = 0; ox < ow; ++ox) {
                    int iy0 = oy * sh - ph, ix0 = ox * sw - pw;
                    int ys = iy0 < 0 ? 0 : iy0, ye = iy0 + kh < ih ? iy0 + kh : ih;
                    int xs = ix0 < 0 ? 0 : ix0, xe = ix0 + kw < iw ? ix0 + kw : iw;
                    const int8_t* xp = x + ((size_t)b * c + ch) * ih * iw;
                    uint8_t out_u;
                    if (is_avg) {
                        uint32_t sum = 0;
                        for (int yy = ys; yy < ye; ++yy)
                            for (int xx = xs; xx < xe; ++xx) sum += (uint8_t)(xp[yy * iw + xx] + 128);
                        int count = (ye - ys) * (xe - xs);
                        uint32_t f = (uint32_t)((1 << 24) / count);
                        out_u = (uint8_t)((sum * f) >> 24);
                    } else {
                        int8_t best = INT8_MIN;
                        for (int yy = ys; yy < ye; ++yy)
                            for (int xx = xs; xx < xe; ++xx) {
                                int8_t s = (int8_t)(uint8_t)(xp[yy * iw + xx] + 128);   /* stored byte read as signed */
                                best = s > best ? s : best;
                            }
                        out_u = (uint8_t)best;
                    }
                    y[(((size_t)b * c + ch) * oh + oy) * ow + ox] = (int8_t)((int)out_u - 128);
                }
}
