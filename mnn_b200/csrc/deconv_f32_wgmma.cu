// deconv_f32_wgmma.cu -- fp32 Deconvolution (transposed conv, group 1, any kernel / stride <= 16 / dilation / padding) on
// split-TF32 wgmma, without inserted zeros or a column buffer.
//
// Phase (sub-pixel) decomposition: output row oy takes tap ky from input row iy when oy + pad_h = iy * sh + ky * dh, so the rows
// with the same r = (oy + pad_h) % sh share one set of taps (ky * dh = r mod sh), and along the phase consecutive outputs read
// consecutive input rows.  The same holds for columns.  Each of the sh * sw phases is therefore a stride-1 implicit GEMM over the
// input: M = its output pixels over the batch, N = oc, K = its taps * Cp8 (tap-major, channel-minor).  A phase without taps
// (kh < sh, a 1x1 kernel with stride 2) has K = 0: its outputs are the bias, then the activation.
//
// One persistent launch over the work items (phase, 128-row M tile of the phase, n chunk), phase-major, with the structure of
// conv_f32_wgmma_kernel: a loader warpgroup gathers the pixel-minor activation tile with 4-byte cp.async (taps outside the image
// zero-filled) while its thread 0 loads the phase's hi / lo weight tiles by TMA; two consumer warpgroups split the activations
// into a_hi + a_lo and issue register-A wgmma m64nNk8 tf32, acc += a_lo*w_hi + a_hi*w_lo + a_hi*w_hi.  The epilogue adds the bias,
// applies ReLU / ReLU6 and stores at the phase's strided output positions.  The weights are split once at create, per phase.
#include <cuda.h>
#include "common.cuh"
#include "hopper_common.cuh"
#include "split_tf32.cuh"
#include "host_util.h"
#include "deconv_ops.h"

namespace mnnb200 {

namespace {
using namespace hop;

// the phase of work item w, advanced from the thread's previous item (a CTA's items only increase)
__device__ __forceinline__ int phase_of(const DeconvF32Params& p, int w, int ph) {
    while (w >= p.item_end[ph]) ++ph;
    return ph;
}

template <int BN>
__global__ void __launch_bounds__(kConvThreads, 1)
deconv_f32_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_hi, const __grid_constant__ CUtensorMap tmap_lo,
                        const __grid_constant__ DeconvF32Params p) {
    using L = Layout<BN>;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    const float* sbase = reinterpret_cast<const float*>(smem_raw + (base - raw));
    constexpr int S = L::stages;
    const uint32_t bar0 = base + S * L::stage_bytes;
    auto full_bar = [&](int s) { return bar0 + 8u * s; };
    auto empty_bar = [&](int s) { return bar0 + 8u * (kMaxStages + s); };
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == kConsumerThreads) {
        prefetch_tmap(&tmap_hi);
        prefetch_tmap(&tmap_lo);
        for (int s = 0; s < S; ++s) { mbar_init(full_bar(s), kLoaderThreads + 1); mbar_init(empty_bar(s), 8); }
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    }
    __syncthreads();

    int ph = 0;
    if (threadIdx.x >= kConsumerThreads) {
        // ---- loader warpgroup
        const int t = threadIdx.x - kConsumerThreads;
        const int HW = p.IH * p.IW;
        int stage = 0, phase = 0;
        for (int w = blockIdx.x; w < p.items; w += gridDim.x) {
            ph = phase_of(p, w, ph);
            const int local = w - (ph ? p.item_end[ph - 1] : 0);
            const int nc = local % p.n_chunks, mt = local / p.n_chunks;
            const int ry = ph / p.sw, rx = ph - ry * p.sw;
            const DeconvAxis Y = p.ay[ry], X = p.ax[rx];
            const int plane = Y.len * X.len;
            const int num_kb = (Y.nk * X.nk * p.Cp8 + kBK - 1) / kBK;
            const int m = mt * kBM + t;
            const bool row_ok = m < p.N * plane;
            int qy = 0, qx = 0;
            const float* xn = p.x;
            if (row_ok) {
                const int n = m / plane, r = m - n * plane, j = r / X.len, i = r - j * X.len;
                qy = Y.q0 + j - Y.off0;
                qx = X.q0 + i - X.off0;
                xn = p.x + (size_t)n * p.IC * HW;
            }
            for (int kb = 0; kb < num_kb; ++kb) {
                mbar_wait(empty_bar(stage), phase ^ 1);
                const uint32_t st = base + stage * L::stage_bytes;
                if (t == 0) {
                    mbar_expect_tx(full_bar(stage), 2u * L::b_bytes);
                    tma_load_2d(st, &tmap_hi, full_bar(stage), kb * kBK * 4, ph * p.ocp + nc * BN);
                    tma_load_2d(st + L::b_bytes, &tmap_lo, full_bar(stage), kb * kBK * 4, ph * p.ocp + nc * BN);
                }
                const uint32_t a_dst = st + 2 * L::b_bytes + t * 4;
#pragma unroll
                for (int g = 0; g < kBK / 8; ++g) {
                    const int k0 = kb * kBK + g * 8;
                    const int tap = k0 / p.Cp8, c0 = k0 - tap * p.Cp8;
                    const int ty = tap / X.nk, tx = tap - ty * X.nk;
                    const int iy = qy - ty * p.istep_h, ix = qx - tx * p.istep_w;
                    const bool ok = row_ok && ty < Y.nk && (unsigned)iy < (unsigned)p.IH && (unsigned)ix < (unsigned)p.IW;
                    const float* src = ok ? xn + ((size_t)c0 * p.IH + iy) * p.IW + ix : p.x;
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const bool v = ok && c0 + j < p.IC;
                        cp_async4(a_dst + (g * 8 + j) * kLdA * 4, v ? src + (size_t)j * HW : p.x, v ? 4 : 0);
                    }
                }
                cp_async_arrive_noinc(full_bar(stage));
                if (++stage == S) { stage = 0; phase ^= 1; }
            }
        }
    } else {
        // ---- consumer warpgroups
        const int wg = threadIdx.x >> 7;
        const int row0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
        const int q = lane & 3;
        const int OHW = p.OH * p.OW;
        int stage = 0, phase = 0;
        float acc[BN / 2];
        for (int w = blockIdx.x; w < p.items; w += gridDim.x) {
            ph = phase_of(p, w, ph);
            const int local = w - (ph ? p.item_end[ph - 1] : 0);
            const int nc = local % p.n_chunks, mt = local / p.n_chunks;
            const int ry = ph / p.sw, rx = ph - ry * p.sw;
            const DeconvAxis Y = p.ay[ry], X = p.ax[rx];
            const int plane = Y.len * X.len;
            const int num_kb = (Y.nk * X.nk * p.Cp8 + kBK - 1) / kBK;
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
            for (int kb = 0; kb < num_kb; ++kb) {
                mbar_wait(full_bar(stage), phase);
                const float* A = sbase + (stage * L::stage_bytes + 2 * L::b_bytes) / 4;
                uint32_t ahi[kBK / 8][4], alo[kBK / 8][4];
#pragma unroll
                for (int s = 0; s < kBK / 8; ++s) {
                    const float* a0 = A + (s * 8 + q) * kLdA + row0;
                    const float v[4] = {a0[0], a0[8], a0[4 * kLdA], a0[4 * kLdA + 8]};
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        ahi[s][i] = tf32_rna(v[i]);
                        alo[s][i] = tf32_rna(v[i] - __uint_as_float(ahi[s][i]));
                    }
                }
                const uint32_t b_hi = base + stage * L::stage_bytes, b_lo = b_hi + L::b_bytes;
                fence_acc(acc);
                wgmma_fence();
#pragma unroll
                for (int s = 0; s < kBK / 8; ++s) {   // small terms first
                    wgmma_rs<BN>(acc, alo[s], gdesc_sw128(b_hi + s * 32), 1);
                    wgmma_rs<BN>(acc, ahi[s], gdesc_sw128(b_lo + s * 32), 1);
                    wgmma_rs<BN>(acc, ahi[s], gdesc_sw128(b_hi + s * 32), 1);
                }
                wgmma_commit();
                // the A registers are rewritten next stage: retire this stage's wgmmas before they are
                wgmma_wait<0>();
                fence_acc(acc);
                __syncwarp();
                if (lane == 0) mbar_arrive(empty_bar(stage));
                if (++stage == S) { stage = 0; phase ^= 1; }
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = mt * kBM + row0 + 8 * h;
                if (m >= p.N * plane) continue;
                const int n = m / plane, r = m - n * plane, j = r / X.len, i = r - j * X.len;
                float* yb = p.y + (size_t)n * p.OC * OHW + (size_t)(Y.o0 + j * p.sh) * p.OW + X.o0 + i * p.sw;
#pragma unroll
                for (int j8 = 0; j8 < BN / 8; ++j8) {
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int oc = nc * BN + j8 * 8 + 2 * q + e;
                        if (oc < p.OC) {
                            float v = __fadd_rn(acc[j8 * 4 + 2 * h + e], p.bias[oc]);
                            if (p.act >= 1) v = fmaxf(v, 0.f);
                            if (p.act == 2) v = fminf(v, 6.f);
                            yb[(size_t)oc * OHW] = v;
                        }
                    }
                }
            }
        }
    }
}

// w [ic][oc][kh][kw] fp32 -> hi / lo [phase][ocp][kp]: phase (ry, rx) holds its taps (ky, kx) = (k0y + ty * kstep_y, k0x + tx *
// kstep_x) at k = (ty * nkx + tx) * cp8 + c, zero padded; w = hi + lo, each rounded to TF32
__global__ void pack_deconv_w_f32_kernel(const float* __restrict__ w, int ic, int oc, int kh, int kw, int sh, int sw, int dh, int dw,
                                         int cp8, int kp, int ocp, float* __restrict__ hi, float* __restrict__ lo) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)sh * sw * ocp * kp) return;
    const int k = (int)(i % kp);
    const size_t r = i / kp;
    const int o = (int)(r % ocp), ph = (int)(r / ocp);
    const DeconvAxisTaps ay = deconv_axis_taps(ph / sw, sh, dh, kh), ax = deconv_axis_taps(ph % sw, sw, dw, kw);
    const int tap = k / cp8, c = k - tap * cp8;
    const int ty = ax.nk ? tap / ax.nk : 0, tx = tap - ty * ax.nk;
    float v = 0.f;
    if (o < oc && c < ic && ty < ay.nk && ax.nk) {
        const int ky = ay.k0 + ty * ay.kstep, kx = ax.k0 + tx * ax.kstep;
        v = w[(((size_t)c * oc + o) * kh + ky) * kw + kx];
    }
    const uint32_t h = tf32_rna(v);
    hi[i] = __uint_as_float(h);
    lo[i] = __uint_as_float(tf32_rna(v - __uint_as_float(h)));
}

template <int BN>
cudaError_t launch_bn(const DeconvF32Params& p, const CUtensorMap& hi, const CUtensorMap& lo, cudaStream_t s, int sm_count) {
    using L = Layout<BN>;
    cudaError_t e = ensure_max_dynamic_smem((const void*)deconv_f32_wgmma_kernel<BN>, L::smem);
    if (e != cudaSuccess) return e;
    const int grid = p.items < sm_count ? p.items : sm_count;
    ++g_launch_count;
    deconv_f32_wgmma_kernel<BN><<<grid, kConvThreads, L::smem, s>>>(hi, lo, p);
    return cudaGetLastError();
}

// ---- fp32 transposed depthwise conv (CPUDeconvolutionDepthwise) as a gather: one thread per output element, over the taps of its
//      phase only (deconv_axis_taps: oy + ph = iy * sh + ky * dh); bias, then ReLU / ReLU6
__global__ void __launch_bounds__(256) dwdeconv_f32_kernel(const DwF32Params p) {
    const size_t total = (size_t)p.N * p.C * p.OH * p.OW;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int ow = (int)(i % p.OW);
        const size_t r = i / p.OW;
        const int oh = (int)(r % p.OH);
        const size_t nc = r / p.OH;
        const int c = (int)(nc % p.C);
        const float* xp = p.x + nc * p.IH * p.IW;
        const float* wp = p.w + (size_t)c * p.KH * p.KW;
        const int uy = oh + p.ph, ux = ow + p.pw;
        const DeconvAxisTaps ay = deconv_axis_taps(uy % p.sh, p.sh, p.dh, p.KH), ax = deconv_axis_taps(ux % p.sw, p.sw, p.dw, p.KW);
        const int qy = uy / p.sh - ay.off0, qx = ux / p.sw - ax.off0;
        float acc = 0.f;
        for (int ty = 0; ty < ay.nk; ++ty) {
            const int ih = qy - ty * ay.istep;
            if ((unsigned)ih >= (unsigned)p.IH) continue;
            const float* wr = wp + (ay.k0 + ty * ay.kstep) * p.KW + ax.k0;
            for (int tx = 0; tx < ax.nk; ++tx) {
                const int iw = qx - tx * ax.istep;
                if ((unsigned)iw < (unsigned)p.IW) acc = fmaf(xp[(size_t)ih * p.IW + iw], wr[tx * ax.kstep], acc);
            }
        }
        float v = acc + p.bias[c];
        if (p.act >= 1) v = fmaxf(v, 0.f);
        if (p.act == 2) v = fminf(v, 6.f);
        p.y[i] = v;
    }
}

}  // namespace

cudaError_t launch_pack_deconv_w_f32(const float* w, int ic, int oc, int kh, int kw, int sh, int sw, int dh, int dw, int cp8,
                                     int kp, int ocp, float* hi, float* lo, cudaStream_t s) {
    const size_t n = (size_t)sh * sw * ocp * kp;
    pack_deconv_w_f32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(w, ic, oc, kh, kw, sh, sw, dh, dw, cp8, kp, ocp, hi, lo);
    ++g_launch_count;
    return cudaGetLastError();
}

cudaError_t launch_deconv_f32_wgmma(const DeconvF32Params& p, const void* tmap_hi, const void* tmap_lo, int bn, cudaStream_t s,
                                    int sm_count) {
    const CUtensorMap& hi = *reinterpret_cast<const CUtensorMap*>(tmap_hi);
    const CUtensorMap& lo = *reinterpret_cast<const CUtensorMap*>(tmap_lo);
    switch (bn) {
        case 32: return launch_bn<32>(p, hi, lo, s, sm_count);
        case 64: return launch_bn<64>(p, hi, lo, s, sm_count);
        case 128: return launch_bn<128>(p, hi, lo, s, sm_count);
        default: return cudaErrorInvalidValue;
    }
}

int deconv_f32_stages(int bn) {
    switch (bn) {
        case 32: return Layout<32>::stages;
        case 64: return Layout<64>::stages;
        case 128: return Layout<128>::stages;
        default: return 0;
    }
}

cudaError_t launch_dwdeconv_f32(const DwF32Params& p, cudaStream_t s) {
    const size_t total = (size_t)p.N * p.C * p.OH * p.OW;
    dwdeconv_f32_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(p);
    ++g_launch_count;
    return cudaGetLastError();
}

}  // namespace mnnb200
