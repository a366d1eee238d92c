// conv_int8_mma.cu -- int8 Conv2D as an IMPLICIT GEMM (no im2col buffer in HBM).
//
// Replaces the reference's Im2Col_packC_16 + CUTLASS GemmBiasScale pair
// (source/backend/cuda/execution/int8/ConvInt8CutlassExecution.cu:16-68, 381-445): the im2col gather is done
// by cp.async straight into swizzled shared memory (padded taps are filled with the INPUT ZERO POINT, as the
// CPU backend does -- compute/ConvInt8TiledExecutor.cpp:2269-2271 -- not with 0 as the reference CUDA kernel),
// the MMA is mma.sync.m16n8k32.s8 and the epilogue is the CPU backend's fp32 sequence, bit for bit.
// This is the general kernel (any kernel size / stride / dilation / pad): it takes the convs that the wgmma kernel in
// conv_group_wgmma.cu does not (stride_w > 2, the largest feature maps).
//
// GEMM view: M = N*OH*OW output pixels, N = oc, K = KH*KW*Cp (tap-major, channel-minor; Cp = p16(ic)).
// Roofline: HBM-bound for MobileNet-class layers; algorithmic bytes = |x| + |w| + |y| (SURVEY 8d).
#include "common.cuh"
#include "host_util.h"
#include "kernels.h"

namespace mnnb200 {

constexpr int BK = 64;      // bytes of K per pipeline stage (= 4 x 16-byte chunks)
constexpr int STAGES = 4;   // cp.async ring depth

template <int BM, int BN, int WM, int WN>
__global__ void __launch_bounds__(WM * WN * 32) conv_int8_igemm_kernel(const ConvParams p) {
    constexpr int THREADS = WM * WN * 32;
    constexpr int WTM = BM / WM, WTN = BN / WN;  // warp tile
    constexpr int MI = WTM / 16, NI = WTN / 8;
    static_assert(NI % 2 == 0, "B fragments are loaded two n8 tiles at a time");
    constexpr int A_ITERS = BM * 4 / THREADS;
    static_assert(A_ITERS * THREADS == BM * 4, "A tile must divide evenly");
    constexpr int B_ITERS = (BN * 4 + THREADS - 1) / THREADS;
    constexpr int CPITCH = BN + 16;

    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* sA = smem;                          // [STAGES][BM][64]
    uint8_t* sB = smem + STAGES * BM * BK;       // [STAGES][BN][64]

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm0 = (warp / WN) * WTM, wn0 = (warp % WN) * WTN;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    const int cpc = p.Cp >> 4;  // 16-byte chunks per tap
    const int c = tid & 3;      // this thread's chunk column inside a K tile

    // ---- per-row gather state (each thread owns A_ITERS rows, always the same chunk column)
    int iy0[A_ITERS], ix0[A_ITERS];
    const int8_t* xb[A_ITERS];
    bool rvalid[A_ITERS];
#pragma unroll
    for (int i = 0; i < A_ITERS; ++i) {
        int r = (tid >> 2) + i * (THREADS / 4);
        int m = m0 + r;
        rvalid[i] = m < p.M;
        int mm = rvalid[i] ? m : 0;
        int ox = mm % p.OW;
        int t = mm / p.OW;
        int oy = t % p.OH;
        int n = t / p.OH;
        iy0[i] = oy * p.sh - p.ph;
        ix0[i] = ox * p.sw - p.pw;
        xb[i] = p.x + (size_t)n * p.IH * p.IW * p.Cp;
    }
    // ---- K decode state for the chunk this thread loads in the NEXT tile to be issued
    int kc = c;
    int c16 = kc % cpc;
    int tap = kc / cpc;
    int ky = tap / p.KW, kx = tap % p.KW;

    const int KT = (p.Kc + 3) >> 2;
    asm volatile("griddepcontrol.wait;\n" ::: "memory");          // PDL: previous kernel's writes are visible from here
    asm volatile("griddepcontrol.launch_dependents;\n" ::: "memory");

    auto load_tile = [&](int stage) {
        const bool kvalid = kc < p.Kc;
        uint8_t* a_st = sA + stage * BM * BK;
#pragma unroll
        for (int i = 0; i < A_ITERS; ++i) {
            int r = (tid >> 2) + i * (THREADS / 4);
            uint32_t dst = smem_u32(a_st + r * BK + ((c ^ ((r >> 1) & 3)) << 4));
            if (kvalid && rvalid[i]) {
                int iy = iy0[i] + ky * p.dh, ix = ix0[i] + kx * p.dw;
                if ((unsigned)iy < (unsigned)p.IH && (unsigned)ix < (unsigned)p.IW) {
                    cp_async16(dst, xb[i] + ((size_t)iy * p.IW + ix) * p.Cp + (c16 << 4), true);
                } else {  // padded tap: the CPU im2col buffer holds the input zero point there
                    asm volatile("st.shared.v4.b32 [%0], {%1,%1,%1,%1};\n" ::"r"(dst), "r"(p.zin_splat));
                }
            } else {
                cp_async16(dst, p.x, false);
            }
        }
        uint8_t* b_st = sB + stage * BN * BK;
#pragma unroll
        for (int i = 0; i < B_ITERS; ++i) {
            int id = tid + i * THREADS;
            if (id < BN * 4) {
                int r = id >> 2;
                int n = n0 + r;
                uint32_t dst = smem_u32(b_st + r * BK + ((c ^ ((r >> 1) & 3)) << 4));
                bool v = kvalid && n < p.OCw;
                cp_async16(dst, v ? (const void*)(p.w + ((size_t)n * p.Kc + kc) * 16) : (const void*)p.w, v);
            }
        }
        // advance to the chunk of the next tile
        kc += 4;
        c16 += 4;
        while (c16 >= cpc) {
            c16 -= cpc;
            if (++kx == p.KW) { kx = 0; ++ky; }
        }
    };

    int acc[MI][NI][4];
#pragma unroll
    for (int i = 0; i < MI; ++i)
#pragma unroll
        for (int j = 0; j < NI; ++j)
#pragma unroll
            for (int k = 0; k < 4; ++k) acc[i][j][k] = 0;

    // ---- prologue
#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s) {
        if (s < KT) load_tile(s);
        cp_async_commit();
    }

    for (int kt = 0; kt < KT; ++kt) {
        cp_async_wait<STAGES - 2>();
        __syncthreads();
        {
            int nt = kt + STAGES - 1;
            if (nt < KT) load_tile(nt % STAGES);
            cp_async_commit();
        }
        const uint8_t* a_st = sA + (kt % STAGES) * BM * BK;
        const uint8_t* b_st = sB + (kt % STAGES) * BN * BK;
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) {
            uint32_t a[MI][4];
#pragma unroll
            for (int mi = 0; mi < MI; ++mi) {
                int row = wm0 + mi * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
                int ch = ks * 2 + (lane >> 4);
                ldmatrix_x4(a[mi][0], a[mi][1], a[mi][2], a[mi][3],
                            smem_u32(a_st + row * BK + ((ch ^ ((row >> 1) & 3)) << 4)));
            }
#pragma unroll
            for (int nj = 0; nj < NI / 2; ++nj) {
                int row = wn0 + nj * 16 + (lane & 7) + (lane >> 4) * 8;
                int ch = ks * 2 + ((lane >> 3) & 1);
                uint32_t b0, b1, b2, b3;
                ldmatrix_x4(b0, b1, b2, b3, smem_u32(b_st + row * BK + ((ch ^ ((row >> 1) & 3)) << 4)));
#pragma unroll
                for (int mi = 0; mi < MI; ++mi) {
                    mma_s8_16832(acc[mi][nj * 2], a[mi], b0, b1);
                    mma_s8_16832(acc[mi][nj * 2 + 1], a[mi], b2, b3);
                }
            }
        }
    }
    cp_async_wait<0>();
    __syncthreads();

    const int g = lane >> 2, t4 = lane & 3;
    // ---- epilogue: CPU-exact requantisation, staged through smem for 16-byte NHWC16 stores
    uint8_t* sC = smem;  // [BM][CPITCH]
#pragma unroll
    for (int ni = 0; ni < NI; ++ni) {
        int col = wn0 + ni * 8 + t4 * 2;
        int n = n0 + col;
        float ws0 = 0.f, ws1 = 0.f, bf0 = 0.f, bf1 = 0.f;
        int k0 = 0, k1 = 0;
        if (n < p.OC) { ws0 = p.wscale[n]; bf0 = p.bias[n]; k0 = p.wsum128[n]; }
        if (n + 1 < p.OC) { ws1 = p.wscale[n + 1]; bf1 = p.bias[n + 1]; k1 = p.wsum128[n + 1]; }
#pragma unroll
        for (int mi = 0; mi < MI; ++mi) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                int row = wm0 + mi * 16 + g + h * 8;
                int q0 = requant_cpu_exact(acc[mi][ni][h * 2] + k0, ws0, p.scale_x, bf0, p.minv, p.maxv);
                int q1 = requant_cpu_exact(acc[mi][ni][h * 2 + 1] + k1, ws1, p.scale_x, bf1, p.minv, p.maxv);
                if (n >= p.OC) q0 = 0;       // channel padding of NHWC16 stays zero
                if (n + 1 >= p.OC) q1 = 0;
                *reinterpret_cast<uint16_t*>(sC + row * CPITCH + col) =
                    (uint16_t)((q0 & 0xff) | ((q1 & 0xff) << 8));
            }
        }
    }
    __syncthreads();
    constexpr int CCH = BN / 16;
    for (int i = tid; i < BM * CCH; i += THREADS) {
        int r = i / CCH, ch = i % CCH;
        int m = m0 + r, n = n0 + ch * 16;
        if (m < p.M && n < p.OCp) {
            *reinterpret_cast<int4*>(p.y + (size_t)m * p.OCp + n) = *reinterpret_cast<const int4*>(sC + r * CPITCH + ch * 16);
        }
    }
}

template <int BM, int BN, int WM, int WN>
static cudaError_t launch_cfg(const ConvParams& p, cudaStream_t stream) {
    constexpr int THREADS = WM * WN * 32;
    const int smem_pipe = STAGES * (BM + BN) * BK;
    const int smem_epi = BM * (BN + 16);
    const int smem = smem_pipe > smem_epi ? smem_pipe : smem_epi;
    auto kern = conv_int8_igemm_kernel<BM, BN, WM, WN>;
    {
        cudaError_t e = ensure_max_dynamic_smem((const void*)kern, smem);
        if (e != cudaSuccess) return e;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((p.M + BM - 1) / BM, (p.OCp + BN - 1) / BN);
    cfg.blockDim = dim3(THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    ++g_launch_count;
    return cudaLaunchKernelEx(&cfg, kern, p);
}

void conv_tile_shape(int tile, int* bm, int* bn) {
    static const int s[TILE_COUNT][2] = {{128, 64}, {128, 32}, {128, 16}, {64, 64}, {64, 32}, {128, 128}};
    *bm = s[tile][0];
    *bn = s[tile][1];
}

cudaError_t launch_conv_int8_igemm(const ConvParams& p, int tile, cudaStream_t stream) {
    switch (tile) {
        case TILE_128x64: return launch_cfg<128, 64, 4, 2>(p, stream);
        case TILE_128x32: return launch_cfg<128, 32, 8, 1>(p, stream);
        case TILE_128x16: return launch_cfg<128, 16, 8, 1>(p, stream);
        case TILE_64x64: return launch_cfg<64, 64, 2, 2>(p, stream);
        case TILE_64x32: return launch_cfg<64, 32, 4, 1>(p, stream);
        case TILE_128x128: return launch_cfg<128, 128, 4, 2>(p, stream);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace mnnb200
