// conv_f32_wgmma.cu -- fp32 Conv2D (group 1, any kernel / stride / dilation / padding) on split-TF32 wgmma.
//
// Implicit GEMM: M = output pixels (N*OH*OW), N = output channels, K = taps * Cp8 (tap-major, channel-minor, Cp8 = ic rounded up
// to 8 so that every k8 step of wgmma reads one tap).  Activations and outputs are NCHW-linear fp32.
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
// accumulator fragments.  The tile width BN (32 / 64 / 128) is a template parameter chosen once per layer at resize.
#include <cuda.h>
#include "common.cuh"
#include "hopper_common.cuh"
#include "host_util.h"
#include "kernels.h"

namespace mnnb200 {

namespace {
using namespace hop;

constexpr int kBM = 128, kBK = 32 /* floats = 128 bytes */, kLdA = kBM + 8 /* conflict-free fragment reads */, kMaxStages = 8;
constexpr int kLoaderThreads = 128;
constexpr int kConvThreads = kConsumerThreads + kLoaderThreads;

template <int BN>
struct Layout {
    static constexpr int b_bytes = BN * kBK * 4;                         // one weight tile (hi or lo), 128B-swizzled rows
    static constexpr int a_bytes = kBK * kLdA * 4;
    static constexpr int stage_bytes = (2 * b_bytes + a_bytes + 1023) & ~1023;
    static constexpr int stages_fit = (227 * 1024 - 1024 - 256) / stage_bytes;
    static constexpr int stages = stages_fit > kMaxStages ? kMaxStages : stages_fit;
    static constexpr int smem = stages * stage_bytes + 1024 + 256;
};

__device__ __forceinline__ uint32_t tf32_rna(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ void cp_async4(uint32_t dst, const void* src, int src_bytes) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;\n" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
// arrives on bar once every cp.async this thread issued before has landed (counts as one of the barrier's expected arrivals)
__device__ __forceinline__ void cp_async_arrive_noinc(uint32_t bar) {
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];\n" ::"r"(bar) : "memory");
}

// wgmma m64nNk8 tf32 with A from registers: a[0..3] = A[r][q], A[r + 8][q], A[r][q + 4], A[r + 8][q + 4] with r = 16 * (warp % 4) +
// lane / 4, q = lane % 4 (the per-warp layout of mma.m16n8k8.tf32); B K-major in shared memory.
template <int N>
__device__ __forceinline__ void wgmma_rs(float* d, const uint32_t (&a)[4], uint64_t b, int scale_d);
template <> __device__ __forceinline__ void wgmma_rs<32>(float* d, const uint32_t (&a)[4], uint64_t b, int scale_d) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %21, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_rs<64>(float* d, const uint32_t (&a)[4], uint64_t b, int scale_d) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_rs<128>(float* d, const uint32_t (&a)[4], uint64_t b, int scale_d) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %69, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(scale_d));
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
            const int m = mt * kBM + t;
            const bool row_ok = m < p.M;
            int ih0 = 0, iw0 = 0;
            const float* xn = p.x;
            if (row_ok) {
                const int n = m / OHW, r = m - n * OHW, oh = r / p.OW, ow = r - oh * p.OW;
                ih0 = oh * p.sh - p.ph;
                iw0 = ow * p.sw - p.pw;
                xn = p.x + (size_t)n * p.IC * HW;
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
        for (int w = blockIdx.x; w < work_total; w += gridDim.x) {
            const int nc = w % p.n_chunks, mt = w / p.n_chunks;
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
                        const int oc = nc * BN + j * 8 + 2 * q + e;
                        if (oc < p.OC) {
                            float v = __fadd_rn(acc[j * 4 + 2 * h + e], p.bias[oc]);
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

// w [oc][ic][taps] fp32 -> hi / lo [ocp][kp], k = tap * cp8 + c, zero padded; w = hi + lo, each rounded to TF32
__global__ void pack_conv_w_f32_kernel(const float* __restrict__ w, int oc, int ic, int taps, int cp8, int kp, int ocp,
                                       float* __restrict__ hi, float* __restrict__ lo) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)ocp * kp) return;
    const int o = (int)(i / kp), k = (int)(i - (size_t)o * kp);
    const int tap = k / cp8, c = k - tap * cp8;
    const float v = (o < oc && tap < taps && c < ic) ? w[((size_t)o * ic + c) * taps + tap] : 0.f;
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

cudaError_t launch_pack_conv_w_f32(const float* w, int oc, int ic, int taps, int cp8, int kp, int ocp, float* hi, float* lo,
                                   cudaStream_t s) {
    const size_t n = (size_t)ocp * kp;
    pack_conv_w_f32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(w, oc, ic, taps, cp8, kp, ocp, hi, lo);
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
