// Decode-time form of the MNN-LLM linear layer ("quantized MatMul", SURVEY a7 / a8): <= 8 tokens against an int8 weight matrix
// [oc][ic].  The reference CPU backend runs the same DenseConvInt8TiledExecutor dynamic-quant branch for one token as for 4096
// (source/backend/cpu/compute/ConvInt8TiledExecutor.cpp:1990-2096, CommonOptFunction.cpp:79-94); the reference CUDA backend has a
// separate GEMV family for it (execution/weight_only_quant/ConvFpAIntBExecution.cu:433-1190).  ONE kernel per layer here:
//   * every block quantises the <= 8 token rows itself (abs-max -> 127/absmax -> round, the dynamic_quant kernel's arithmetic
//     operation for operation; 8-22 KB of fp32 per token out of L2) into shared memory -- no separate quantise launch, no
//     int8 activation round trip;
//   * every warp streams R weight rows with 16-byte non-allocating loads (each weight byte is read exactly once: HBM-bound),
//     dp4a into int32, butterfly reduce, then the SAME fp32 epilogue as gemm_i8_wgmma's EPI 1 -- int32 sums are
//     order-independent, so the result is bit-identical to the tensor-core path;
//   * K-blocked weight scales (p.bs != 0, MNN-LLM's quant_block export) take a run-time branch of the same kernel: exact int32
//     sums per block, finished in block order as gemm_i8_wgmma's blocked EPI 1 does, so again bit-identical to it;
//   * 4-bit weights (p.w4) take another run-time branch: a 16-byte load brings 32 packed weights (K 2kb..2kb+31 for byte
//     offset kb, the first 16 in the low nibbles), a mask and a shift per dword expand them to bytes u = q + 8, and everything
//     after the dp4a is the 8-bit code with the tables of mnnb200_linear_w4_create_blocked.  Only in the instantiations with
//     two or more tokens and at most two rows per warp (see stream_rows);
//   * programmatic dependent launch: the first weight chunk is requested before griddepcontrol.wait, so the next layer's blocks
//     are resident and loading while this layer drains (a decode step is ~120 dependent launches of 2-10 us each).
#include "common.cuh"
#include "kernels.h"

#include <algorithm>
#include <type_traits>

namespace mnnb200 {
namespace {

// two blocks per SM: at most 128 registers, which the per-channel path fits in on its own; the blocked path's extra values
// would otherwise lift <2, 4, 4> past it and halve its occupancy
template <int T, int R, int U>
__global__ void __launch_bounds__(256, 2) linear_w8_gemv_kernel(GemvW8Params p) {
    extern __shared__ __align__(16) uint8_t smem_x[];      // [T][icp] int8
    __shared__ float s_max[8];
    __shared__ int s_sum[8];
    __shared__ float s_dq[T], s_ss[T];
    __shared__ float s_min[8], s_izf;      // single-token (decode) branch: row minimum per warp, folded input zero
    asm volatile("griddepcontrol.launch_dependents;\n" ::: "memory");
    auto dot16 = [](const int4& xv, const int4& w, int a) {
        a = __dp4a(xv.x, w.x, a);
        a = __dp4a(xv.y, w.y, a);
        a = __dp4a(xv.z, w.z, a);
        return __dp4a(xv.w, w.w, a);
    };
    auto lo4 = [](const int4& v) { return make_int4(v.x & 0x0F0F0F0F, v.y & 0x0F0F0F0F, v.z & 0x0F0F0F0F, v.w & 0x0F0F0F0F); };
    auto hi4 = [](const int4& v) {
        return make_int4((v.x >> 4) & 0x0F0F0F0F, (v.y >> 4) & 0x0F0F0F0F, (v.z >> 4) & 0x0F0F0F0F, (v.w >> 4) & 0x0F0F0F0F);
    };
    const int icp = p.icp, ic = p.ic;
    const int w4 = T > 1 && R < 4 ? p.w4 : 0, rowb = icp >> w4;       // weight bytes per row
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int warps = blockDim.x >> 5;
    int n0 = (blockIdx.x * warps + warp) * R;
    // the first U chunks (U * 512 bytes of K) of this warp's first rows are requested right away: weights are constants, so they
    // may be in flight while the producer of x is still running and while this block quantises x
    const int8_t* wrow[R];
    int4 wv[R][U];
#pragma unroll
    for (int r = 0; r < R; ++r) {
        wrow[r] = p.w + (size_t)min(n0 + r, p.ocp - 1) * rowb;
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int k = lane * 16 + u * 512;
            wv[r][u] = (n0 < p.oc && k < rowb) ? ld_nc_16(wrow[r] + k) : make_int4(0, 0, 0, 0);
        }
    }
    // ... and so are the epilogue constants of the output this lane will finish (lane = token * R + row)
    float c_alpha = 0.f, c_wsumf = 0.f, c_wzero = 0.f, c_bias = 0.f;
    int c_wsum128 = 0;
    {
        const int n = n0 + lane % R;
        if (lane < T * R && n < p.oc && !p.bs) {
            c_alpha = __ldg(p.alpha + n); c_wsumf = __ldg(p.wsumf + n); c_wsum128 = __ldg(p.wsum128 + n);
            if (p.wzero) c_wzero = __ldg(p.wzero + n);
            if (p.bias) c_bias = __ldg(p.bias + n);
        }
    }
    asm volatile("griddepcontrol.wait;\n" ::: "memory");

    // ---- per-token dynamic quantisation into shared memory (elementwise.cu: dynamic_quant_vec_kernel, same operations);
    //      the token row stays in registers between the abs-max and the quantise pass when it fits (ic <= 8192)
    const bool vec = (ic & 3) == 0 && (reinterpret_cast<uintptr_t>(p.x) & 15) == 0;
    const bool in_regs = vec && ic <= 8192;
    for (int t = 0; t < T; ++t) {
        uint32_t* qrow = reinterpret_cast<uint32_t*>(smem_x + t * icp);
        if (t >= p.tokens) {
            for (int i = threadIdx.x; i < (icp >> 2); i += blockDim.x) qrow[i] = 0u;
            continue;
        }
        const float* xr = p.x + (size_t)t * ic;
        const float4* x4 = reinterpret_cast<const float4*>(xr);
        float4 v[8];
        float amax = 0.f;
        if (p.tokens == 1) {
            // ---- ONE token: the reference switches to its single-quant arithmetic (ConvInt8TiledExecutor.cpp:1033-1035 leaves
            //      mUseBatchQuan false for inputPlane == 1; :1432 / :2016-2050 mToFuseInputbias2Bias): asymmetric quantisation with
            //      min / max over the row INCLUDING the zero padding of the last 16-channel pack (_AVX512_MNNAsyQuantInfo,
            //      x86_x64/avx512/PackedFunction.cpp:133-165), the fma-contracted FloatToInt8 into [-128, 127], and the input zero
            //      point folded into the bias (MNNDynamicUpdateConvBiasScale, CommonOptFunction.cpp:96-103) in the epilogue below
            float mn = 3.4028234663852886e38f, mx = -3.4028234663852886e38f;
            if (in_regs) {      // all loads of the row in flight at once, the row stays in registers for the quantise pass
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int i = threadIdx.x + j * 256;
                    if (i < (ic >> 2)) {
                        v[j] = __ldg(x4 + i);
                        mn = fminf(mn, fminf(fminf(v[j].x, v[j].y), fminf(v[j].z, v[j].w)));
                        mx = fmaxf(mx, fmaxf(fmaxf(v[j].x, v[j].y), fmaxf(v[j].z, v[j].w)));
                    }
                }
            } else {
                for (int i = threadIdx.x; i < ic; i += blockDim.x) {
                    const float q = __ldg(xr + i);
                    mn = fminf(mn, q);
                    mx = fmaxf(mx, q);
                }
            }
            if (ic & 15) { mn = fminf(mn, 0.f); mx = fmaxf(mx, 0.f); }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
            }
            if (lane == 0) { s_max[warp] = mx; s_min[warp] = mn; }
            __syncthreads();
            mx = s_max[0]; mn = s_min[0];
#pragma unroll
            for (int i = 1; i < 8; ++i) { mx = fmaxf(mx, s_max[i]); mn = fminf(mn, s_min[i]); }
            const float range = __fsub_rn(mx, mn);
            float scale = 1.f, qscale = 1.f, qbias = -mx;
            if (!((double)range <= 1e-7)) {
                qscale = __fdiv_rn(255.f, range);
                scale = __fdiv_rn(range, 255.f);
                qbias = __fsub_rn(roundf(__fdiv_rn(__fmul_rn(-mn, 255.f), range)), 128.0f);
            }
            int lsum = 0;
            auto quant1 = [&](float xv) -> int {
                float f = __fmaf_rn(xv, qscale, qbias);
                f = fminf(fmaxf(f, -128.f), 127.f);
                f = __fadd_rn(f, f < 0.f ? -0.5f : 0.5f);
                const int q = __float2int_rz(f);
                lsum += q + 128;
                return q;
            };
            if (in_regs) {
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int i = threadIdx.x + j * 256;
                    if (i < (icp >> 2)) {
                        uint32_t packed = 0;
                        if (i < (ic >> 2)) {
                            const int q0 = quant1(v[j].x), q1 = quant1(v[j].y), q2 = quant1(v[j].z), q3 = quant1(v[j].w);
                            packed = (uint32_t)(q0 & 0xff) | ((uint32_t)(q1 & 0xff) << 8) | ((uint32_t)(q2 & 0xff) << 16) | ((uint32_t)(q3 & 0xff) << 24);
                        }
                        qrow[i] = packed;
                    }
                }
            } else {
                int8_t* qb = reinterpret_cast<int8_t*>(qrow);
                for (int i = threadIdx.x; i < icp; i += blockDim.x) qb[i] = i < ic ? (int8_t)quant1(__ldg(xr + i)) : (int8_t)0;
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) lsum += __shfl_xor_sync(0xffffffffu, lsum, o);
            if (lane == 0) s_sum[warp] = lsum;
            __syncthreads();
            if (threadIdx.x == 0) {
                int tot = 0;
#pragma unroll
                for (int i = 0; i < 8; ++i) tot += s_sum[i];
                s_dq[0] = scale;
                s_ss[0] = __fmul_rn(__int2float_rn(tot), scale);
                s_izf = __fmul_rn(-qbias, scale);
            }
            continue;
        }
        if (in_regs) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int i = threadIdx.x + j * 256;
                v[j] = i < (ic >> 2) ? __ldg(x4 + i) : make_float4(0.f, 0.f, 0.f, 0.f);
                amax = fmaxf(amax, fmaxf(fmaxf(fabsf(v[j].x), fabsf(v[j].y)), fmaxf(fabsf(v[j].z), fabsf(v[j].w))));
            }
        } else if (vec) {
            for (int i = threadIdx.x; i < (ic >> 2); i += blockDim.x) {
                const float4 q = __ldg(x4 + i);
                amax = fmaxf(amax, fmaxf(fmaxf(fabsf(q.x), fabsf(q.y)), fmaxf(fabsf(q.z), fabsf(q.w))));
            }
        } else {
            for (int i = threadIdx.x; i < ic; i += blockDim.x) amax = fmaxf(amax, fabsf(__ldg(xr + i)));
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
        __syncthreads();                 // s_max / s_sum of the previous token are consumed
        if (lane == 0) s_max[warp] = amax;
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
        auto quant4 = [&](const float4& q) -> uint32_t {
            const int q0 = __float2int_rn(__fmul_rn(q.x, qs)), q1 = __float2int_rn(__fmul_rn(q.y, qs));
            const int q2 = __float2int_rn(__fmul_rn(q.z, qs)), q3 = __float2int_rn(__fmul_rn(q.w, qs));
            lsum += q0 + q1 + q2 + q3 + 512;
            return (uint32_t)(q0 & 0xff) | ((uint32_t)(q1 & 0xff) << 8) | ((uint32_t)(q2 & 0xff) << 16) | ((uint32_t)(q3 & 0xff) << 24);
        };
        if (in_regs) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int i = threadIdx.x + j * 256;
                if (i < (icp >> 2)) qrow[i] = i < (ic >> 2) ? quant4(v[j]) : 0u;
            }
        } else if (vec) {
            for (int i = threadIdx.x; i < (icp >> 2); i += blockDim.x) qrow[i] = i < (ic >> 2) ? quant4(__ldg(x4 + i)) : 0u;
        } else {
            int8_t* qb = reinterpret_cast<int8_t*>(qrow);
            for (int i = threadIdx.x; i < icp; i += blockDim.x) {
                int q = 0;
                if (i < ic) { q = __float2int_rn(__fmul_rn(__ldg(xr + i), qs)); lsum += q + 128; }
                qb[i] = (int8_t)q;
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) lsum += __shfl_xor_sync(0xffffffffu, lsum, o);
        if (lane == 0) s_sum[warp] = lsum;
        __syncthreads();
        if (threadIdx.x == 0) {
            int tot = 0;
#pragma unroll
            for (int i = 0; i < 8; ++i) tot += s_sum[i];
            s_dq[t] = dqv;
            s_ss[t] = __fmul_rn(__int2float_rn(tot), dqv);
        }
    }
    __syncthreads();

    // everything after the quantisation once per weight format, W4 a constant in each.  The 4-bit branch is not in the
    // one-token and the four-row instantiations at all: next to it the 8-bit decode step of Qwen-1.8B took 0.924 ms instead of
    // 0.882 (H100 80GB HBM3, 700 W), so 4-bit layers run one token on the two-token kernel and at most two rows per warp
    auto stream_rows = [&](auto w4c) {
        constexpr int W4 = decltype(w4c)::value;
        const int row_bytes = icp >> W4;
        bool first = true;
        if (p.bs) {
            // ---- K-blocked weight scales (mnn_oracle_linear_w8_dynamic_blocks): every output sums, block after block, the fp32
            //      finish of its exact int32 block accumulator.  The quantisation above is unchanged; the per-block input sums
            //      xsum_b * scale come from the quantised rows in shared memory.  In a 512-byte window of K the G = bs / 16 lanes of a
            //      block reduce its int32 sums with a butterfly, the group's first lane finishes the block (sum_b w is dp4a'd from the
            //      streamed weights, not stored) into shared memory, and the lane owning the output adds the parts in block order.
            //      4-bit: a lane covers 32 channels, so G = bs / 32 and a 1024-channel window holds up to 32 blocks (SL slots); ws_b
            //      is the layer's weightKernelSum for the first block and 0 after it (the reference's 4-bit kernel adds it once).
            const int bs = p.bs, G = bs >> (4 + W4), nb = ic / bs, SL = 16 << W4;
            float* s_xs = reinterpret_cast<float*>(smem_x + T * icp);                 // [T][nb]
            float* s_part = s_xs + T * nb + warp * (T * R + R) * SL;                 // [T * R][SL] parts, then [R][SL] ws_b
            float* s_wsb = s_part + T * R * SL;
            for (int i = threadIdx.x; i < T * nb; i += blockDim.x) {
                const int t = i / nb, b = i - t * nb;
                float v = 0.f;
                if (t < p.tokens) {
                    const int4* q4 = reinterpret_cast<const int4*>(smem_x + t * icp + b * bs);
                    int sum = 0;
                    for (int j = 0; j < (bs >> 4); ++j) {
                        const int4 q = q4[j];
                        sum = __dp4a(q.x, 0x01010101, sum); sum = __dp4a(q.y, 0x01010101, sum);
                        sum = __dp4a(q.z, 0x01010101, sum); sum = __dp4a(q.w, 0x01010101, sum);
                    }
                    v = __fmul_rn(__int2float_rn(sum + 128 * bs), s_dq[t]);
                }
                s_xs[i] = v;
            }
            __syncthreads();
            for (; n0 < p.oc; n0 += gridDim.x * warps * R) {
                if (!first) {
#pragma unroll
                    for (int r = 0; r < R; ++r) wrow[r] = p.w + (size_t)min(n0 + r, p.ocp - 1) * row_bytes;
                }
                float f = 0.f, wtot = 0.f;
                for (int kbase = 0; kbase < row_bytes; kbase += 512 * U) {
                    if (!(first && kbase == 0)) {
#pragma unroll
                        for (int r = 0; r < R; ++r)
#pragma unroll
                            for (int u = 0; u < U; ++u) {
                                const int k = kbase + lane * 16 + u * 512;
                                wv[r][u] = k < row_bytes ? ld_nc_16(wrow[r] + k) : make_int4(0, 0, 0, 0);
                            }
                    }
#pragma unroll
                    for (int u = 0; u < U; ++u) {
                        const int kw = kbase + u * 512, k = kw + lane * 16;     // bytes of the weight row
                        if (kw >= row_bytes) break;
                        // one weight row at a time: its T block sums and sum_b w are the only new values live next to the weights
#pragma unroll
                        for (int r = 0; r < R; ++r) {
                            const int4 ones = make_int4(0x01010101, 0x01010101, 0x01010101, 0x01010101);
                            const int4 w = W4 ? lo4(wv[r][u]) : wv[r][u], wh = hi4(wv[r][u]);
                            int sw = dot16(ones, w, 0);
                            if (W4) sw = dot16(ones, wh, sw);
                            int a[T];
#pragma unroll
                            for (int t = 0; t < T; ++t) {
                                const uint8_t* xr = smem_x + t * icp + (k << W4);
                                a[t] = k < row_bytes ? dot16(*reinterpret_cast<const int4*>(xr), w, 0) : 0;
                                if (W4 && k < row_bytes) a[t] = dot16(*reinterpret_cast<const int4*>(xr + 16), wh, a[t]);
                            }
                            for (int o = 1; o < G; o <<= 1) {
                                sw += __shfl_xor_sync(0xffffffffu, sw, o);
#pragma unroll
                                for (int t = 0; t < T; ++t) a[t] += __shfl_xor_sync(0xffffffffu, a[t], o);
                            }
                            if ((lane & (G - 1)) == 0 && k < row_bytes) {
                                const int g = lane / G, b = (k << W4) / bs;
                                const size_t ci = (size_t)min(n0 + r, p.ocp - 1) * nb + b;   // alpha_b / wzero_b (zero past oc)
                                const float c_al = __ldg(p.balpha + ci), c_wz = __ldg(p.bwzero + ci);
                                // ws_b = float(sum_b w) * alpha_b + bs * wzero_b;  the block's accumulator includes the +128 offset
                                const float ws = W4 ? (b == 0 ? __ldg(p.wsumf + min(n0 + r, p.ocp - 1)) : 0.f)
                                                    : __fadd_rn(__fmul_rn(__int2float_rn(sw), c_al), __fmul_rn((float)bs, c_wz));
                                s_wsb[r * SL + g] = ws;
#pragma unroll
                                for (int t = 0; t < T; ++t) {
                                    const float sc = s_dq[t];
                                    float part = __fmul_rn(__int2float_rn(a[t] + 128 * sw), c_al);
                                    part = __fmul_rn(part, sc);
                                    part = __fadd_rn(part, __fmul_rn(__fmul_rn(sc, -128.f), ws));
                                    part = __fadd_rn(__fmul_rn(s_xs[t * nb + b], c_wz), part);
                                    s_part[(t * R + r) * SL + g] = part;
                                }
                            }
                        }
                        __syncwarp();
                        if (lane < T * R) {
                            const int nbw = min(32 / G, nb - (kw << W4) / bs);     // blocks in this window, in order
                            for (int g = 0; g < nbw; ++g) {
                                f = __fadd_rn(f, s_part[lane * SL + g]);
                                wtot = __fadd_rn(wtot, s_wsb[(lane % R) * SL + g]);
                            }
                        }
                        __syncwarp();
                    }
                }
                first = false;
                if (lane < T * R) {
                    const int n = n0 + lane % R, m = lane / R;
                    if (n < p.oc && m < p.tokens) {
                        const float bias = p.bias ? __ldg(p.bias + n) : 0.f;
                        if (p.tokens == 1) f = __fadd_rn(f, __fadd_rn(bias, __fmul_rn(wtot, s_izf)));   // bias' = bias + sum_b ws_b * izf
                        else if (p.bias) f = __fadd_rn(f, bias);
                        if (p.relu | p.relu6) { f = fminf(f, p.relu6 ? 6.0f : 3.4028234663852886e38f); f = fmaxf(f, 0.f); }
                        p.y[(size_t)m * p.ldy + n] = f;
                    }
                }
            }
            return;
        }
        for (; n0 < p.oc; n0 += gridDim.x * warps * R) {
            int acc[T][R];
#pragma unroll
            for (int t = 0; t < T; ++t)
#pragma unroll
                for (int r = 0; r < R; ++r) acc[t][r] = 0;
            if (!first) {
#pragma unroll
                for (int r = 0; r < R; ++r) wrow[r] = p.w + (size_t)min(n0 + r, p.ocp - 1) * row_bytes;
            }
            for (int k0 = lane * 16; k0 < row_bytes; k0 += 512 * U) {
                if (!(first && k0 == lane * 16)) {
#pragma unroll
                    for (int r = 0; r < R; ++r)
#pragma unroll
                        for (int u = 0; u < U; ++u) {
                            const int k = k0 + u * 512;
                            wv[r][u] = k < row_bytes ? ld_nc_16(wrow[r] + k) : make_int4(0, 0, 0, 0);
                        }
                }
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const int k = k0 + u * 512;
                    if (W4 && k < row_bytes) {
                        // one row at a time, so that only one row's expanded weights are live next to the packed ones
#pragma unroll
                        for (int r = 0; r < R; ++r) {
                            const int4 lo = lo4(wv[r][u]), hi = hi4(wv[r][u]);
#pragma unroll
                            for (int t = 0; t < T; ++t) {
                                const uint8_t* xr = smem_x + t * icp + 2 * k;
                                acc[t][r] = dot16(*reinterpret_cast<const int4*>(xr + 16), hi, dot16(*reinterpret_cast<const int4*>(xr), lo, acc[t][r]));
                            }
                        }
                    } else if (k < row_bytes) {
#pragma unroll
                        for (int t = 0; t < T; ++t) {
                            const int4 xv = *reinterpret_cast<const int4*>(smem_x + t * icp + k);
#pragma unroll
                            for (int r = 0; r < R; ++r) {
                                int a = acc[t][r];
                                a = __dp4a(xv.x, wv[r][u].x, a);
                                a = __dp4a(xv.y, wv[r][u].y, a);
                                a = __dp4a(xv.z, wv[r][u].z, a);
                                a = __dp4a(xv.w, wv[r][u].w, a);
                                acc[t][r] = a;
                            }
                        }
                    }
                }
            }
            if (!first) {
                const int n = n0 + lane % R;
                if (lane < T * R && n < p.oc) {
                    c_alpha = __ldg(p.alpha + n); c_wsumf = __ldg(p.wsumf + n); c_wsum128 = __ldg(p.wsum128 + n);
                    c_wzero = p.wzero ? __ldg(p.wzero + n) : 0.f;
                    c_bias = p.bias ? __ldg(p.bias + n) : 0.f;
                }
            }
            first = false;
#pragma unroll
            for (int t = 0; t < T; ++t)
#pragma unroll
                for (int r = 0; r < R; ++r) {
                    int a = acc[t][r];
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
                    // lane (t * R + r) finishes output (token t, row n0 + r): gemm_i8_wgmma.cu EPI 1, operation for operation
                    if (lane == t * R + r) {
                        const int n = n0 + r, m = t;
                        if (n < p.oc && m < p.tokens) {
                            const float dqm = s_dq[m], ss = s_ss[m];
                            const float corr = __fmul_rn(dqm, -128.f);
                            float f = __fmul_rn(__int2float_rn(a + c_wsum128), c_alpha);
                            f = __fmul_rn(f, dqm);
                            f = __fadd_rn(f, __fmul_rn(corr, c_wsumf));
                            f = __fadd_rn(__fmul_rn(ss, c_wzero), f);
                            if (p.tokens == 1) f = __fadd_rn(f, __fadd_rn(c_bias, __fmul_rn(c_wsumf, s_izf)));   // bias' = bias + weightKernelSum * (-qbias * scale)
                            else if (p.bias) f = __fadd_rn(f, c_bias);
                            if (p.relu | p.relu6) { f = fminf(f, p.relu6 ? 6.0f : 3.4028234663852886e38f); f = fmaxf(f, 0.f); }
                            p.y[(size_t)m * p.ldy + n] = f;
                        }
                    }
                }
        }
    };
    if constexpr (T > 1 && R < 4) {
        if (w4) return stream_rows(std::integral_constant<int, 1>{});
    }
    stream_rows(std::integral_constant<int, 0>{});
}

template <int T, int R, int U>
cudaError_t launch_t(const GemvW8Params& p, const GemvW8Launch& l, cudaStream_t stream) {
    if (l.smem > 40 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(linear_w8_gemv_kernel<T, R, U>, cudaFuncAttributeMaxDynamicSharedMemorySize, l.smem);
        if (e != cudaSuccess) return e;
    }
    ++g_launch_count;
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3((unsigned)l.grid);
    cfg.blockDim = dim3(256);
    cfg.dynamicSmemBytes = l.smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, linear_w8_gemv_kernel<T, R, U>, p);
}

// the instantiation linear_w8_gemv_launch picked; <4, 4, 4> and <8, 4, 4> are not instantiated at all
template <int T>
cudaError_t launch_r(const GemvW8Params& p, const GemvW8Launch& l, cudaStream_t stream) {
    if constexpr (T <= 2) {
        if (l.r == 4) return launch_t<T, 4, 4>(p, l, stream);
    }
    if (l.r == 2) return launch_t<T, 2, 4>(p, l, stream);
    return launch_t<T, 1, 4>(p, l, stream);
}

}  // namespace

// blocked (bs > 0): the shared memory also holds the per-block input sums and every warp's block parts (launch_t)
bool linear_w8_gemv_supported(int tokens, int icp, int bs, int w4) {
    const size_t extra = bs ? ((size_t)8 * (icp / bs) + 8 * 18 * (16 << w4)) * sizeof(float) : 0;
    return tokens >= 1 && tokens <= 8 && (size_t)8 * icp + extra <= 200 * 1024;
}

GemvW8Launch linear_w8_gemv_launch(const GemvW8Params& p, int sms) {
    GemvW8Launch l;
    // 4-bit layers run one token on the two-token instantiation (the one-token kernel carries no 4-bit branch: stream_rows)
    l.t = p.tokens <= 1 && !p.w4 ? 1 : p.tokens <= 2 ? 2 : p.tokens <= 4 ? 4 : 8;
    // rows per warp: as many as keep >= ~2 blocks per SM (the small layers are latency-bound: more blocks = more loads in
    // flight).  Four rows only for <= 2 tokens and 8-bit weights
    l.r = l.t <= 2 && !p.w4 && p.oc >= sms * 2 * 8 * 4 ? 4 : p.oc >= sms * 2 * 8 * 2 ? 2 : 1;
    const int rows_per_block = 8 * l.r;
    l.grid = std::min((p.oc + rows_per_block - 1) / rows_per_block, sms * 8);
    l.passes = (p.oc + l.grid * rows_per_block - 1) / (l.grid * rows_per_block);
    // blocked: + the per-block input sums [T][ic / bs] and each warp's block parts
    const size_t smem = (size_t)l.t * p.icp +
                        (p.bs ? ((size_t)l.t * (p.ic / p.bs) + 8 * (l.t * l.r + l.r) * (16 << p.w4)) * sizeof(float) : 0);
    l.smem = (int)smem;
    l.w4 = l.t > 1 && l.r < 4 ? p.w4 : 0;      // the kernel's own rule
    return l;
}

cudaError_t launch_linear_w8_gemv(const GemvW8Params& p, cudaStream_t stream, int sms) {
    const GemvW8Launch l = linear_w8_gemv_launch(p, sms);
    switch (l.t) {
        case 1: return launch_r<1>(p, l, stream);
        case 2: return launch_r<2>(p, l, stream);
        case 4: return launch_r<4>(p, l, stream);
        default: return launch_r<8>(p, l, stream);
    }
}

}  // namespace mnnb200
