// conv_f32_wgmma.cu -- fp32 Conv2D (any group, kernel, stride, dilation, padding) on split-TF32 wgmma.
//
// Implicit GEMM: M = output pixels (N*OH*OW), N = output channels, K = taps * Cp8 (tap-major, channel-minor, Cp8 = the input
// channels of one n chunk rounded up to 8 so that every k8 step of wgmma reads one tap).  Activations and outputs are NCHW-linear
// fp32.  Groups: an n chunk covers P consecutive whole groups (ocg <= bn) or one bn-wide slice of one group (Q chunks per group),
// so its input and output channels are both contiguous ranges and its weight tile is block-diagonal (the zeros add exact zeros).
// Group 1 is G = 1, P = 1, Q = n_chunks: every chunk reads all input channels, the K order and MMAs of a dense conv.
//
// One persistent, warp-specialised kernel:
//   warps 8-11  loader warpgroup.  Thread t gathers pixel row t of the 128-row M tile: 32 K values per stage with 4-byte cp.async
//               into a pixel-minor shared-memory tile [32 k][136] (out-of-image taps and padded channels are zero-filled: float
//               padding is a true zero).  An NCHW map is pixel-minor and its 7- / 14-wide rows break TMA's 16-byte stride rule, so
//               the activation operand is gathered by threads; thread 0 also loads the two weight tiles (hi, lo) with TMA.
//   warps 0-7   two consumer warpgroups, 64 rows each.  TF32 wgmma reads a shared-memory A operand only K-major, so the consumers
//               build the A fragments from the pixel-minor tile themselves and issue the register-A form (m64nNk8, four .b32 A
//               registers), splitting each activation into a_hi + a_lo on the way.
// Split TF32 (3xTF32): a = a_hi + a_lo, w = w_hi + w_lo, each part rounded to TF32; acc += a_lo*w_hi + a_hi*w_lo + a_hi*w_hi in fp32.
// The dropped a_lo*w_lo term and the TF32 rounding of the low parts leave an error near fp32's (about 2^-21 of |a||w| per product).
// The weights are split once at create (pack_conv_w_f32_kernel).  Epilogue: + bias, then ReLU / ReLU6, stored NCHW from the
// accumulator fragments.  The tile width BN (32 / 64 / 128) is a template parameter chosen once per layer: at resize for group 1,
// at create for a grouped layer (its packed K layout depends on it).
#include <cuda.h>
#include "common.cuh"
#include "hopper_common.cuh"
#include "split_tf32.cuh"
#include "host_util.h"
#include "kernels.h"

namespace mnnb200 {

namespace {
using namespace hop;

// epilogue: + bias, then ReLU (ACT 1) / ReLU6 (ACT 2), stored NCHW; column j of the tile is channel oc0 + j, stored iff j < ncols
template <int BN, int ACT>
__device__ __forceinline__ void store_tile(const float (&acc)[BN / 2], const ConvF32Params& p, int mt, int row0, int q, int oc0,
                                           int ncols) {
    const int OHW = p.OH * p.OW;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int m = mt * kBM + row0 + 8 * h;
        if (m >= p.M) continue;
        const int n = m / OHW, pix = m - n * OHW;
        float* yb = p.y + (size_t)n * p.OC * OHW + pix;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int col = j * 8 + 2 * q + e, oc = oc0 + col;
                if (col < ncols) {
                    float v = __fadd_rn(acc[j * 4 + 2 * h + e], p.bias[oc]);
                    if (ACT >= 1) v = fmaxf(v, 0.f);
                    if (ACT == 2) v = fminf(v, 6.f);
                    yb[(size_t)oc * OHW] = v;
                }
            }
        }
    }
}

template <int BN>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_f32_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_hi, const __grid_constant__ CUtensorMap tmap_lo, const ConvF32Params p) {
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
    const int work_total = p.m_tiles * p.n_chunks;

    if (threadIdx.x == kConsumerThreads) {
        prefetch_tmap(&tmap_hi);
        prefetch_tmap(&tmap_lo);
        for (int s = 0; s < S; ++s) { mbar_init(full_bar(s), kLoaderThreads + 1); mbar_init(empty_bar(s), 8); }
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    }
    __syncthreads();

    if (threadIdx.x >= kConsumerThreads) {
        // ---- loader warpgroup
        const int t = threadIdx.x - kConsumerThreads;
        const int HW = p.IH * p.IW, OHW = p.OH * p.OW;
        int stage = 0, phase = 0;
        for (int w = blockIdx.x; w < work_total; w += gridDim.x) {
            const int nc = w % p.n_chunks, mt = w / p.n_chunks;
            const int g0 = nc / p.Q * p.P, ng = min(p.P, p.G - g0);
            const int cin = ng * p.icg;            // this chunk's input channels: [g0 icg, g0 icg + cin)
            const int m = mt * kBM + t;
            const bool row_ok = m < p.M;
            int ih0 = 0, iw0 = 0;
            const float* xn = p.x;
            if (row_ok) {
                const int n = m / OHW, r = m - n * OHW, oh = r / p.OW, ow = r - oh * p.OW;
                ih0 = oh * p.sh - p.ph;
                iw0 = ow * p.sw - p.pw;
                xn = p.x + ((size_t)n * p.IC + g0 * p.icg) * HW;
            }
            for (int kb = 0; kb < p.num_kb; ++kb) {
                mbar_wait(empty_bar(stage), phase ^ 1);
                const uint32_t st = base + stage * L::stage_bytes;
                if (t == 0) {
                    mbar_expect_tx(full_bar(stage), 2u * L::b_bytes);
                    tma_load_2d(st, &tmap_hi, full_bar(stage), kb * kBK * 4, nc * BN);
                    tma_load_2d(st + L::b_bytes, &tmap_lo, full_bar(stage), kb * kBK * 4, nc * BN);
                }
                const uint32_t a_dst = st + 2 * L::b_bytes + t * 4;
#pragma unroll
                for (int g = 0; g < kBK / 8; ++g) {
                    const int k0 = kb * kBK + g * 8;
                    const int tap = k0 / p.Cp8, c0 = k0 - tap * p.Cp8;
                    const int kh = tap / p.KW, kw = tap - kh * p.KW;
                    const int ih = ih0 + kh * p.dh, iw = iw0 + kw * p.dw;
                    const bool ok = row_ok && tap < p.taps && (unsigned)ih < (unsigned)p.IH && (unsigned)iw < (unsigned)p.IW;
                    const float* src = ok ? xn + ((size_t)c0 * p.IH + ih) * p.IW + iw : p.x;
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const bool v = ok && c0 + j < cin;
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
        int stage = 0, phase = 0;
        float acc[BN / 2];
        for (int w = blockIdx.x; w < work_total; w += gridDim.x) {
            const int nc = w % p.n_chunks, mt = w / p.n_chunks;
            const int g0 = nc / p.Q * p.P, sub = nc - nc / p.Q * p.Q, ng = min(p.P, p.G - g0);
            const int oc0 = g0 * p.ocg + sub * BN;           // column j of this chunk is channel oc0 + j, stored iff j < ncols
            const int ncols = min(BN, ng * p.ocg - sub * BN);
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
            for (int kb = 0; kb < p.num_kb; ++kb) {
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
            // one epilogue per activation, chosen once per tile
            if (p.act == 0) store_tile<BN, 0>(acc, p, mt, row0, q, oc0, ncols);
            else if (p.act == 1) store_tile<BN, 1>(acc, p, mt, row0, q, oc0, ncols);
            else store_tile<BN, 2>(acc, p, mt, row0, q, oc0, ncols);
        }
    }
}

// w [oc][icg][taps] fp32 -> hi / lo [ocp][kp], block-diagonal per n chunk of g.bn rows: row nc * bn + j holds channel oc0 + j's
// taps at k = tap * cp8 + (c - ic0) (c an input channel of its group, ic0 the chunk's first), zeros elsewhere; w = hi + lo, each
// rounded to TF32.  Group 1 is G = P = Q = 1, bn = ocp: row o is channel o, k = tap * cp8 + c.
__global__ void pack_conv_w_f32_kernel(const float* __restrict__ w, int oc, int taps, int cp8, int kp, int ocp, ConvF32Groups g,
                                       float* __restrict__ hi, float* __restrict__ lo) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)ocp * kp) return;
    const int o = (int)(i / kp), k = (int)(i - (size_t)o * kp);
    const int nc = o / g.bn, j = o - nc * g.bn;
    const int g0 = nc / g.Q * g.P, sub = nc - nc / g.Q * g.Q, ng = min(g.P, g.G - g0);
    const int ch = g0 * g.ocg + sub * g.bn + j;                                  // the row's output channel
    const int tap = k / cp8, c = k - tap * cp8 - (ch / g.ocg - g0) * g.icg;      // input channel within the row's group
    const bool in = j < ng * g.ocg - sub * g.bn && ch < oc && tap < taps && c >= 0 && c < g.icg;
    const float v = in ? w[((size_t)ch * g.icg + c) * taps + tap] : 0.f;
    const uint32_t h = tf32_rna(v);
    hi[i] = __uint_as_float(h);
    lo[i] = __uint_as_float(tf32_rna(v - __uint_as_float(h)));
}

template <int BN>
cudaError_t launch_bn(const ConvF32Params& p, const CUtensorMap& hi, const CUtensorMap& lo, cudaStream_t s, int sm_count) {
    using L = Layout<BN>;
    cudaError_t e = ensure_max_dynamic_smem((const void*)conv_f32_wgmma_kernel<BN>, L::smem);
    if (e != cudaSuccess) return e;
    const int work = p.m_tiles * p.n_chunks;
    const int grid = work < sm_count ? work : sm_count;
    ++g_launch_count;
    conv_f32_wgmma_kernel<BN><<<grid, kConvThreads, L::smem, s>>>(hi, lo, p);
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_pack_conv_w_f32(const float* w, int oc, int taps, int cp8, int kp, int ocp, const ConvF32Groups& g, float* hi,
                                   float* lo, cudaStream_t s) {
    const size_t n = (size_t)ocp * kp;
    pack_conv_w_f32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(w, oc, taps, cp8, kp, ocp, g, hi, lo);
    ++g_launch_count;
    return cudaGetLastError();
}

cudaError_t launch_conv_f32_wgmma(const ConvF32Params& p, const void* tmap_hi, const void* tmap_lo, int bn, cudaStream_t s,
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

int conv_f32_stages(int bn) {
    switch (bn) {
        case 32: return Layout<32>::stages;
        case 64: return Layout<64>::stages;
        case 128: return Layout<128>::stages;
        default: return 0;
    }
}

}  // namespace mnnb200
