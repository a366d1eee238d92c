// gemm_f16_wgmma.cu -- float (batched) MatMul on wgmma:  C[b][e][h] (fp32) = A[b][e][l] * B[b][l][h] (+ bias)
//
// SURVEY a9: the attention QK^T / PV matmuls MNN-LLM leaves outside its fused attention op, and every other MatMul /
// BatchMatMul the geometry stage emits.  Replaces MatMulExecution's 18 CUTLASS mma.sync variants
// (source/backend/cuda/execution/MatMulExecution.cu:306-1050) with one persistent TMA + wgmma kernel:
//   1. pack kernels bring both operands to K-major form ([b][e][lp], [b][h][lp], lp = l padded to 16 bytes; the transposes
//      that transposeA / !transposeB imply are done in the same pass through smem): fp16 operands stay fp16, fp32 operands
//      are split into two TF32 planes x = hi + lo (split_tf32);
//   2. gemm_f16_wgmma_kernel: warp 8 = TMA producer (128B-swizzled stages), warps 0-7 = two consumer warpgroups
//      (fp32 accumulators in registers, 64 rows of the 128-row tile each) whose epilogue adds the bias and stores fp32 straight
//      from the accumulator fragments.  fp16: one wgmma m64nNk16 f16 per 32 bytes of K.  fp32: a stage holds the hi and lo
//      tiles of both operands and each k8 step issues three wgmma m64nNk8 tf32, a_hi*b_hi + a_hi*b_lo + a_lo*b_hi.
// Accuracy: fp32 operands err by about 3 * 2^-22 of |a||b| per product plus the fp32 accumulation (tests/test_gpu_matmul_f32.py
// bounds every output); fp16 operands by the accumulation alone.
#include <cuda.h>
#include <cuda_fp16.h>
#include "common.cuh"
#include "hopper_common.cuh"
#include "host_util.h"
#include "kernels.h"
#include "split_tf32.cuh"

namespace mnnb200 {

namespace {
using namespace hop;

// tile rows, K block bytes (64 halves / 32 floats), stage ring, widest n chunk of the fp16 and of the split fp32 kernel (the
// split stage holds four tiles: 128 columns keep three stages in shared memory)
constexpr int kMmBM = 128, kMmBK = 128, kMmStages = 6, kMmMaxBN = 256, kMmMaxBNSplit = 128;

struct FParams {
    int M, N, K;           // K in BYTES of one operand row (multiple of 16)
    int bn, n_chunks, m_tiles, batch;
    int a_batch_rows, b_batch_rows;
    int a_lo_row, b_lo_row; // split: the lo plane's first row in each operand's tensor map
    const int* batch_map;  // [batch][2]: the A and B batch of each output batch (broadcast), or nullptr: both are the output's
    float* c;              // [batch][M][N]
    const float* bias;     // [N] or nullptr
    int stages;
    int vec_ok;            // N even and c 8-byte aligned: column pairs are stored as float2
};

// SPLIT = false: fp16 operands (K16 per wgmma); true: fp32 operands as TF32 hi / lo planes (K8 per wgmma, three per step)
template <bool SPLIT>
__global__ void __launch_bounds__(kThreads, 1)
gemm_f16_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, const FParams p) {
    constexpr int kPlanes = SPLIT ? 2 : 1, kMaxBN = SPLIT ? kMmMaxBNSplit : kMmMaxBN;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    const int a_tile = kMmBM * kMmBK, b_tile = p.bn * kMmBK;
    const int stage_bytes = kPlanes * (a_tile + b_tile);    // [A hi][A lo][B hi][B lo]
    const int S = p.stages;
    const uint32_t bar0 = base + S * stage_bytes;
    auto full_bar = [&](int s) { return bar0 + 8u * s; };
    auto empty_bar = [&](int s) { return bar0 + 8u * (kMmStages + s); };
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int num_kb = (p.K + kMmBK - 1) / kMmBK;
    const int work_total = p.batch * p.m_tiles * p.n_chunks;   // < 2^31: matmul_create refuses more

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
                const int a_row = ab * p.a_batch_rows + mt * kMmBM, b_row = bb * p.b_batch_rows + nc * p.bn;
                for (int kb = 0; kb < num_kb; ++kb) {
                    mbar_wait(empty_bar(stage), phase ^ 1);
                    mbar_expect_tx(full_bar(stage), (uint32_t)stage_bytes);
                    const uint32_t a_dst = base + stage * stage_bytes, b_dst = a_dst + kPlanes * a_tile;
                    tma_load_2d(a_dst, &tmap_a, full_bar(stage), kb * kMmBK, a_row);
                    tma_load_2d(b_dst, &tmap_b, full_bar(stage), kb * kMmBK, b_row);
                    if constexpr (SPLIT) {
                        tma_load_2d(a_dst + a_tile, &tmap_a, full_bar(stage), kb * kMmBK, p.a_lo_row + a_row);
                        tma_load_2d(b_dst + b_tile, &tmap_b, full_bar(stage), kb * kMmBK, p.b_lo_row + b_row);
                    }
                    if (++stage == S) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        const int wg = threadIdx.x >> 7;
        const int r_base = wg * 64 + (warp & 3) * 16 + (lane >> 2);
        const int q4 = lane & 3;
        const int nblk = p.bn >> 3;
        const bool vec_ok = p.vec_ok != 0;
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
                const uint32_t a_addr = base + stage * stage_bytes + wg * 64 * kMmBK, b_addr = base + stage * stage_bytes + kPlanes * a_tile;
                const int kleft = p.K - kb * kMmBK;                   // bytes of K left
                const int nmma = kleft >= kMmBK ? 4 : (kleft + 31) / 32;
                fence_acc(acc);
                wgmma_fence();
                for (int k = 0; k < nmma; ++k) {
                    const int first = (kb | k) == 0 ? 0 : 1;
                    if constexpr (SPLIT) {
                        // the small terms first: a_hi*b_lo and a_lo*b_hi, then a_hi*b_hi
                        wgmma_bn<Kind::TF32, kMaxBN>(acc, p.bn, gdesc_sw128(a_addr + k * 32), gdesc_sw128(b_addr + b_tile + k * 32),
                                                     kMmBK, first);
                        wgmma_bn<Kind::TF32, kMaxBN>(acc, p.bn, gdesc_sw128(a_addr + a_tile + k * 32), gdesc_sw128(b_addr + k * 32),
                                                     kMmBK, 1);
                        wgmma_bn<Kind::TF32, kMaxBN>(acc, p.bn, gdesc_sw128(a_addr + k * 32), gdesc_sw128(b_addr + k * 32), kMmBK, 1);
                    } else {
                        wgmma_bn<Kind::F16, kMaxBN>(acc, p.bn, gdesc_sw128(a_addr + k * 32), gdesc_sw128(b_addr + k * 32), kMmBK,
                                                    first);
                    }
                }
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
                const int m = mt * kMmBM + r_base + 8 * h;
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

__device__ __forceinline__ void pack_put(__half* d, size_t, size_t i, float v) { d[i] = __float2half_rn(v); }
__device__ __forceinline__ void pack_put(float* d, size_t lo_off, size_t i, float v) {
    float hi, lo;
    split_tf32(v, hi, lo);
    d[i] = hi;
    d[lo_off + i] = lo;
}

// ---- operand pack: src logical [b][rows][k] (trans = 0: memory is [rows][k]; trans = 1: memory is [k][rows])
//      -> dst [b][rows][kp], zero padded along k: fp16 for an fp16 src; for an fp32 src the TF32 hi plane, and the lo plane
//      lo_off floats further.  32x32 tiles (smem transpose when trans = 1), grid-stride over every batch's tiles, so any
//      batch and row count is covered by a one-dimensional grid.  One body, two entry points (fp16 copy, fp32 split).
template <typename T>
__device__ __forceinline__ void pack_kmajor_tiles(const T* __restrict__ src, T* __restrict__ dst, size_t lo_off, int batches,
                                                  int rows, int k, int kp, int trans) {
    __shared__ float tile[32][33];
    const int k_tiles = (kp + 31) / 32, r_tiles = (rows + 31) / 32;
    const long long tiles = (long long)batches * r_tiles * k_tiles;
    const int tx = threadIdx.x, ty = threadIdx.y;   // 32 x 8
    for (long long t = blockIdx.x; t < tiles; t += gridDim.x) {
        const long long q = t / k_tiles, b = q / r_tiles;
        const int k0 = (int)(t - q * k_tiles) * 32, r0 = (int)(q - b * r_tiles) * 32;
        const T* s = src + (size_t)b * rows * k;
        const size_t d0 = (size_t)b * rows * kp;
        if (!trans) {
            for (int i = ty; i < 32; i += 8) {
                int r = r0 + i, kk = k0 + tx;
                if (r < rows && kk < kp) pack_put(dst, lo_off, d0 + (size_t)r * kp + kk, kk < k ? (float)s[(size_t)r * k + kk] : 0.f);
            }
        } else {
            for (int i = ty; i < 32; i += 8) {          // read [k][rows] coalesced along rows
                int kk = k0 + i, r = r0 + tx;
                tile[i][tx] = (kk < k && r < rows) ? (float)s[(size_t)kk * rows + r] : 0.f;
            }
            __syncthreads();
            for (int i = ty; i < 32; i += 8) {
                int r = r0 + i, kk = k0 + tx;
                if (r < rows && kk < kp) pack_put(dst, lo_off, d0 + (size_t)r * kp + kk, tile[tx][i]);
            }
            __syncthreads();
        }
    }
}

template <typename T>
__global__ void pack_kmajor_f16_kernel(const T* __restrict__ src, __half* __restrict__ dst, int batches, int rows, int k, int kp,
                                       int trans) {
    pack_kmajor_tiles<__half>(src, dst, 0, batches, rows, k, kp, trans);
}
template <typename T>
__global__ void pack_kmajor_f32_kernel(const T* __restrict__ src, float* __restrict__ dst, size_t lo_off, int batches, int rows,
                                       int k, int kp, int trans) {
    pack_kmajor_tiles<float>(src, dst, lo_off, batches, rows, k, kp, trans);
}

int pack_grid(int batch, int rows, int kp) {
    const long long tiles = (long long)batch * ((rows + 31) / 32) * ((kp + 31) / 32);
    return (int)(tiles < (1 << 20) ? tiles : (1 << 20));
}

}  // namespace

cudaError_t launch_pack_split_tf32(const float* src, float* dst, size_t lo_off, int batch, int rows, int k, int kp, int trans,
                                   cudaStream_t s) {
    pack_kmajor_f32_kernel<float><<<pack_grid(batch, rows, kp), dim3(32, 8), 0, s>>>(src, dst, lo_off, batch, rows, k, kp, trans);
    ++g_launch_count;
    return cudaGetLastError();
}

cudaError_t launch_pack_kmajor_f16(const void* src, void* dst, int batch, int rows, int k, int kp, int trans, cudaStream_t s) {
    pack_kmajor_f16_kernel<__half><<<pack_grid(batch, rows, kp), dim3(32, 8), 0, s>>>((const __half*)src, (__half*)dst, batch, rows,
                                                                                     k, kp, trans);
    ++g_launch_count;
    return cudaGetLastError();
}

int gemm_f16_wgmma_max_bn(int split) { return split ? kMmMaxBNSplit : kMmMaxBN; }

cudaError_t launch_gemm_f16_wgmma(const void* tmap_a, const void* tmap_b, int batch, int M, int N, int k_bytes, int split,
                                  int a_batch_rows, int b_batch_rows, int a_lo_row, int b_lo_row, int bn, float* c,
                                  const float* bias, cudaStream_t stream, int sm_count, const int* batch_map) {
    if (bn < 16 || bn > gemm_f16_wgmma_max_bn(split) || (bn & 15)) return cudaErrorInvalidValue;
    FParams p;
    p.M = M; p.N = N; p.K = k_bytes; p.bn = bn; p.n_chunks = (N + bn - 1) / bn; p.m_tiles = (M + kMmBM - 1) / kMmBM; p.batch = batch;
    p.a_batch_rows = a_batch_rows; p.b_batch_rows = b_batch_rows; p.a_lo_row = a_lo_row; p.b_lo_row = b_lo_row;
    p.batch_map = batch_map; p.c = c; p.bias = bias;
    p.vec_ok = (N & 1) == 0 && ((uintptr_t)c & 7) == 0;
    const int stage_bytes = (split ? 2 : 1) * (kMmBM + bn) * kMmBK;
    int st = (227 * 1024 - 256 - 1024) / stage_bytes;
    p.stages = st > kMmStages ? kMmStages : st;
    const int smem = p.stages * stage_bytes + 256 + 1024;
    const void* kern = split ? (const void*)gemm_f16_wgmma_kernel<true> : (const void*)gemm_f16_wgmma_kernel<false>;
    {
        cudaError_t e = ensure_max_dynamic_smem(kern, 227 * 1024);
        if (e != cudaSuccess) return e;
    }
    const long long work = (long long)p.batch * p.m_tiles * p.n_chunks;
    if (work > 0x7fffffffLL) return cudaErrorInvalidValue;
    const int grid = work < sm_count ? (int)work : sm_count;
    ++g_launch_count;
    const CUtensorMap& ta = *reinterpret_cast<const CUtensorMap*>(tmap_a);
    const CUtensorMap& tb = *reinterpret_cast<const CUtensorMap*>(tmap_b);
    if (split) gemm_f16_wgmma_kernel<true><<<grid, kThreads, smem, stream>>>(ta, tb, p);
    else gemm_f16_wgmma_kernel<false><<<grid, kThreads, smem, stream>>>(ta, tb, p);
    return cudaGetLastError();
}

}  // namespace mnnb200
