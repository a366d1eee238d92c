// gemm_f16_wgmma.cu -- float (batched) MatMul on wgmma:  C[b][e][h] (fp32) = A[b][e][l] * B[b][l][h] (+ bias)
//
// SURVEY a9: the attention QK^T / PV matmuls MNN-LLM leaves outside its fused attention op, and every other MatMul /
// BatchMatMul the geometry stage emits.  Replaces MatMulExecution's 18 CUTLASS mma.sync variants
// (source/backend/cuda/execution/MatMulExecution.cu:306-1050) with one persistent TMA + wgmma kernel:
//   1. pack kernels bring an operand that is not K-major already to K-major form in its own type ([b][e][lp], [b][h][lp],
//      lp = l padded to 16 bytes; the transposes that transposeA / !transposeB imply are done in the same pass through smem);
//   2. gemm_f16_wgmma_kernel: warp 8 = TMA producer (128B-swizzled stages), warps 0-7 = two consumer warpgroups
//      (wgmma.mma_async m64nNk16 f16 or m64nNk8 tf32, fp32 accumulators in registers, 64 rows of the 128-row tile each)
//      whose epilogue adds the bias and stores fp32 straight from the accumulator fragments.
// Accuracy contract (BASELINE north_star): max|C - C_cpu| / max|C_cpu| <= 1e-3 against the CPU backend's fp32 matmul.
#include <cuda.h>
#include <cuda_fp16.h>
#include "common.cuh"
#include "hopper_common.cuh"
#include "host_util.h"
#include "kernels.h"

namespace mnnb200 {

namespace {
using namespace hop;

constexpr int kBM = 128, kBK = 128 /* bytes = 64 halves */, kMaxStages = 6, kMaxBN = 256;

struct FParams {
    int M, N, K;           // K in BYTES of one operand row (multiple of 16)
    int bn, n_chunks, m_tiles, batch;
    int a_batch_rows, b_batch_rows;
    const int* batch_map;  // [batch][2]: the A and B batch of each output batch (broadcast), or nullptr: both are the output's
    float* c;              // [batch][M][N]
    const float* bias;     // [N] or nullptr
    int stages;
};

// TF32 = false: fp16 operands (K16 per wgmma), true: fp32 operands read as tf32 (K8 per wgmma); both 32 bytes of K
template <bool TF32>
__global__ void __launch_bounds__(kThreads, 1)
gemm_f16_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, const FParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    const int stage_bytes = kBM * kBK + p.bn * kBK;
    const int S = p.stages;
    const uint32_t bar0 = base + S * stage_bytes;
    auto full_bar = [&](int s) { return bar0 + 8u * s; };
    auto empty_bar = [&](int s) { return bar0 + 8u * (kMaxStages + s); };
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int num_kb = (p.K + kBK - 1) / kBK;
    const int work_total = p.batch * p.m_tiles * p.n_chunks;

    if (warp == 8 && lane == 0) {
        prefetch_tmap(&tmap_a);
        prefetch_tmap(&tmap_b);
        for (int s = 0; s < S; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 8); }
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            int stage = 0, phase = 0;
            for (int w = blockIdx.x; w < work_total; w += gridDim.x) {
                const int nc = w % p.n_chunks, wq = w / p.n_chunks, mt = wq % p.m_tiles, bt = wq / p.m_tiles;
                const int ab = p.batch_map ? p.batch_map[2 * bt] : bt, bb = p.batch_map ? p.batch_map[2 * bt + 1] : bt;
                const int a_row = ab * p.a_batch_rows + mt * kBM, b_row = bb * p.b_batch_rows + nc * p.bn;
                for (int kb = 0; kb < num_kb; ++kb) {
                    mbar_wait(empty_bar(stage), phase ^ 1);
                    mbar_expect_tx(full_bar(stage), (uint32_t)stage_bytes);
                    const uint32_t a_dst = base + stage * stage_bytes;
                    tma_load_2d(a_dst, &tmap_a, full_bar(stage), kb * kBK, a_row);
                    tma_load_2d(a_dst + kBM * kBK, &tmap_b, full_bar(stage), kb * kBK, b_row);
                    if (++stage == S) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        const int wg = threadIdx.x >> 7;
        const int r_base = wg * 64 + (warp & 3) * 16 + (lane >> 2);
        const int q4 = lane & 3;
        const int nblk = p.bn >> 3;
        const bool vec_ok = (p.N & 1) == 0;
        int stage = 0, phase = 0;
        float acc[kMaxBN / 2];
#pragma unroll
        for (int i = 0; i < kMaxBN / 2; ++i) acc[i] = 0.f;
        for (int w = blockIdx.x; w < work_total; w += gridDim.x) {
            const int nc = w % p.n_chunks, wq = w / p.n_chunks, mt = wq % p.m_tiles, bt = wq / p.m_tiles;
            const int n0 = nc * p.bn;
            int prev = -1;
            for (int kb = 0; kb < num_kb; ++kb) {
                mbar_wait(full_bar(stage), phase);
                const uint32_t a_addr = base + stage * stage_bytes + wg * 64 * kBK, b_addr = base + stage * stage_bytes + kBM * kBK;
                const int kleft = p.K - kb * kBK;                     // bytes of K left
                const int nmma = kleft >= kBK ? 4 : (kleft + 31) / 32;
                fence_acc(acc);
                wgmma_fence();
                for (int k = 0; k < nmma; ++k)
                    wgmma_bn<TF32 ? Kind::TF32 : Kind::F16, kMaxBN>(acc, p.bn, gdesc_sw128(a_addr + k * 32), gdesc_sw128(b_addr + k * 32),
                                                                   kBK, (kb | k) != 0);
                wgmma_commit();
                wgmma_wait<1>();
                fence_acc(acc);
                if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(empty_bar(prev)); }
                prev = stage;
                if (++stage == S) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
            fence_acc(acc);
            __syncwarp();
            if (lane == 0) mbar_arrive(empty_bar(prev));
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = mt * kBM + r_base + 8 * h;
                if (m >= p.M) continue;
                float* crow = p.c + ((size_t)bt * p.M + m) * p.N;
#pragma unroll
                for (int j = 0; j < kMaxBN / 8; ++j) {
                    if (j < nblk) {
                        const int n = n0 + j * 8 + 2 * q4;
                        if (n < p.N) {
                            float f0 = acc[j * 4 + 2 * h], f1 = acc[j * 4 + 2 * h + 1];
                            if (p.bias) {
                                f0 = __fadd_rn(f0, p.bias[n]);
                                if (n + 1 < p.N) f1 = __fadd_rn(f1, p.bias[n + 1]);
                            }
                            if (vec_ok && n + 1 < p.N) {
                                *reinterpret_cast<float2*>(crow + n) = make_float2(f0, f1);
                            } else {
                                crow[n] = f0;
                                if (n + 1 < p.N) crow[n + 1] = f1;
                            }
                        }
                    }
                }
            }
        }
    }
}

// ---- operand pack: src fp16, logical [b][rows][k] (trans = 0: memory is [rows][k]; trans = 1: memory is [k][rows])
//      -> dst fp16 [b][rows][kp], zero padded along k.  32x32 smem tile transpose when trans = 1.
template <typename T>
__global__ void pack_kmajor_f16_kernel(const T* __restrict__ src, __half* __restrict__ dst, int rows, int k, int kp, int trans) {
    __shared__ float tile[32][33];
    const int b = blockIdx.z;
    const T* s = src + (size_t)b * rows * k;
    __half* d = dst + (size_t)b * rows * kp;
    const int r0 = blockIdx.y * 32, k0 = blockIdx.x * 32;
    const int tx = threadIdx.x, ty = threadIdx.y;   // 32 x 8
    if (!trans) {
        for (int i = ty; i < 32; i += 8) {
            int r = r0 + i, kk = k0 + tx;
            if (r < rows && kk < kp) d[(size_t)r * kp + kk] = kk < k ? __float2half_rn((float)s[(size_t)r * k + kk]) : __float2half_rn(0.f);
        }
    } else {
        for (int i = ty; i < 32; i += 8) {          // read [k][rows] coalesced along rows
            int kk = k0 + i, r = r0 + tx;
            tile[i][tx] = (kk < k && r < rows) ? (float)s[(size_t)kk * rows + r] : 0.f;
        }
        __syncthreads();
        for (int i = ty; i < 32; i += 8) {
            int r = r0 + i, kk = k0 + tx;
            if (r < rows && kk < kp) d[(size_t)r * kp + kk] = __float2half_rn(tile[tx][i]);
        }
    }
}

}  // namespace

template <typename T>
__global__ void pack_kmajor_f32_kernel(const T* __restrict__ src, float* __restrict__ dst, int rows, int k, int kp, int trans) {
    __shared__ float tile[32][33];
    const int b = blockIdx.z;
    const T* s = src + (size_t)b * rows * k;
    float* d = dst + (size_t)b * rows * kp;
    const int r0 = blockIdx.y * 32, k0 = blockIdx.x * 32;
    const int tx = threadIdx.x, ty = threadIdx.y;
    if (!trans) {
        for (int i = ty; i < 32; i += 8) {
            int r = r0 + i, kk = k0 + tx;
            if (r < rows && kk < kp) d[(size_t)r * kp + kk] = kk < k ? (float)s[(size_t)r * k + kk] : 0.f;
        }
    } else {
        for (int i = ty; i < 32; i += 8) {
            int kk = k0 + i, r = r0 + tx;
            tile[i][tx] = (kk < k && r < rows) ? (float)s[(size_t)kk * rows + r] : 0.f;
        }
        __syncthreads();
        for (int i = ty; i < 32; i += 8) {
            int r = r0 + i, kk = k0 + tx;
            if (r < rows && kk < kp) d[(size_t)r * kp + kk] = tile[tx][i];
        }
    }
}

cudaError_t launch_pack_kmajor_f32(const float* src, float* dst, int batch, int rows, int k, int kp, int trans, cudaStream_t s) {
    dim3 grid((kp + 31) / 32, (rows + 31) / 32, batch), block(32, 8);
    pack_kmajor_f32_kernel<float><<<grid, block, 0, s>>>(src, dst, rows, k, kp, trans);
    ++g_launch_count;
    return cudaGetLastError();
}

cudaError_t launch_pack_kmajor_f16(const void* src, void* dst, int batch, int rows, int k, int kp, int trans, cudaStream_t s) {
    dim3 grid((kp + 31) / 32, (rows + 31) / 32, batch), block(32, 8);
    pack_kmajor_f16_kernel<__half><<<grid, block, 0, s>>>((const __half*)src, (__half*)dst, rows, k, kp, trans);
    ++g_launch_count;
    return cudaGetLastError();
}

cudaError_t launch_gemm_f16_wgmma(const void* tmap_a, const void* tmap_b, int batch, int M, int N, int k_bytes, int tf32,
                                  int a_batch_rows, int b_batch_rows, int bn, float* c, const float* bias, cudaStream_t stream,
                                  int sm_count, const int* batch_map) {
    if (bn < 16 || bn > kMaxBN || (bn & 15)) return cudaErrorInvalidValue;
    FParams p;
    p.M = M; p.N = N; p.K = k_bytes; p.bn = bn; p.n_chunks = (N + bn - 1) / bn; p.m_tiles = (M + kBM - 1) / kBM; p.batch = batch;
    p.a_batch_rows = a_batch_rows; p.b_batch_rows = b_batch_rows; p.batch_map = batch_map; p.c = c; p.bias = bias;
    const int stage_bytes = kBM * kBK + bn * kBK;
    int st = (227 * 1024 - 256 - 1024) / stage_bytes;
    p.stages = st > kMaxStages ? kMaxStages : st;
    const int smem = p.stages * stage_bytes + 256 + 1024;
    const void* kern = tf32 ? (const void*)gemm_f16_wgmma_kernel<true> : (const void*)gemm_f16_wgmma_kernel<false>;
    {
        cudaError_t e = ensure_max_dynamic_smem(kern, 227 * 1024);
        if (e != cudaSuccess) return e;
    }
    const int work = p.batch * p.m_tiles * p.n_chunks;
    const int grid = work < sm_count ? work : sm_count;
    ++g_launch_count;
    const CUtensorMap& ta = *reinterpret_cast<const CUtensorMap*>(tmap_a);
    const CUtensorMap& tb = *reinterpret_cast<const CUtensorMap*>(tmap_b);
    if (tf32) gemm_f16_wgmma_kernel<true><<<grid, kThreads, smem, stream>>>(ta, tb, p);
    else gemm_f16_wgmma_kernel<false><<<grid, kThreads, smem, stream>>>(ta, tb, p);
    return cudaGetLastError();
}

}  // namespace mnnb200
