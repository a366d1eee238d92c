// gemm_i8_wgmma.cu -- Hopper int8 GEMM  D[M,N] = A[M,K] * B[N,K]^T  (s8 x s8 -> s32), fp32 out
//
// The LLM linear layer after dynamic activation quantisation and the Winograd position GEMMs.  Replaces the
// dequantise-then-fp16-GEMM of ConvFpAIntBExecution (weight_only_quant/ConvFpAIntBExecution.cu:1884-1924).  Int8 convolutions
// with int8 outputs run on conv_group_wgmma.cu, 1x1 ones included.
//
//   * operands: TMA (cp.async.bulk.tensor.2d) into 128B-swizzled shared memory, up to 8-stage mbarrier ring, issued by
//               warp 8; a weight matrix that fits stays resident for the whole launch
//   * math:     wgmma.mma_async m64nNk32 s8, two consumer warpgroups, each owning 64 rows of the 128-row tile
//   * epilogue: straight from the accumulator registers: the CPU backend's dynamic-quant linear or Winograd position fp32
//               forms, bit for bit
//   * persistent: grid = #SMs, static round-robin over (batch, m_tile, n_chunk) work items
//   * 4-bit weights (EPI 1, single CTA): TMA brings the packed nibbles (half the bytes of B), the consumer warpgroups expand
//               them into the int8 B tile of the stage (or the resident B once) before the wgmmas read it
//   * pair mode (launch_gemm_i8_2cta): a 2-CTA cluster computes 256 x bn; each CTA loads its own 128 rows of A and HALF of
//     the B tile, multicast into both CTAs' shared memory, so each SM ingests 3/4 of the operand bytes of a lone CTA
#include <cuda.h>
#include "common.cuh"
#include "hopper_common.cuh"
#include "host_util.h"
#include "kernels.h"

namespace mnnb200 {

namespace {
using namespace hop;

constexpr int kBM = 128;
constexpr int kBK = 128;          // bytes of K per pipeline stage = one 128B swizzle row
constexpr int kMaxStages = 8;
constexpr int kMaxBN = 256;
constexpr int kStageBytesA = kBM * kBK;          // 16 KB
constexpr int kConstBytes = kMaxBN * 4 * 5;      // per-column epilogue constants
constexpr int kSmemBudget = 227 * 1024 - 1024;   // minus the 1024B alignment slack

struct SmemPlan {
    int stages, stage_bytes, resident_b;   // resident_b: B (weights) loaded once per CTA
    int off_resb, off_resp, off_consts, off_bars, total;   // off_resp: the packed resident B of 4-bit weights
};
// w4: B arrives as packed nibbles (bn * kBK / 2 bytes per K block) next to the int8 tile they are expanded into
__host__ __device__ inline SmemPlan make_plan(int bn, int n_chunks, int num_kb, bool pair, int w4 = 0) {
    SmemPlan pl;
    const int resb_bytes = bn * kBK * num_kb;
    const int packed = w4 ? bn * kBK / 2 : 0;
    pl.resident_b = (!pair && n_chunks == 1 && resb_bytes <= 72 * 1024) ? 1 : 0;
    pl.stage_bytes = kStageBytesA + (pl.resident_b ? 0 : bn * kBK + packed);
    const int fixed = (pl.resident_b ? resb_bytes + packed * num_kb : 0) + kConstBytes + 256;
    const int st = (kSmemBudget - fixed) / pl.stage_bytes;
    pl.stages = st > kMaxStages ? kMaxStages : (st < 2 ? 2 : st);
    pl.off_resb = pl.stages * pl.stage_bytes;
    pl.off_resp = pl.off_resb + (pl.resident_b ? resb_bytes : 0);
    pl.off_consts = pl.off_resp + (pl.resident_b ? packed * num_kb : 0);
    pl.off_bars = pl.off_consts + kConstBytes;
    pl.total = pl.off_bars + 256;
    return pl;
}

struct KParams {
    int M, N, K;          // N = valid (padded-to-16) output columns
    int bn;               // columns per work item (multiple of 16, <= 256)
    int n_chunks, m_tiles;   // pair mode: m_tiles counts 256-row tiles
    const float* wscale;
    const float* bias;
    const int32_t* wsum128;
    int OC, ldy;
    // fp32 out; dq / srcsum / wsumf / wzero: dynamic-quant linear only
    float* y_f32;
    const float* dq;
    const float* srcsum;
    const float* wsumf;
    const float* wzero;
    int relu, relu6, has_bias;
    // K-blocked weight scales (EPI 1, single CTA, bn <= 128): bsteps = 32-byte k-steps per block (0: per channel)
    int bsteps, blocks;
    const float *balpha, *bwzero, *bws, *xsb;
    const int32_t* bw128;
    // batched mode (Winograd: one GEMM per transform position): work item = (batch, m_tile, n_chunk)
    int batch, a_batch_rows, b_batch_rows, c_batch_stride;
    int one_tile;   // grid == number of work items: every CTA owns exactly one (batch, m tile, n chunk)
    int w4;         // B holds 4-bit weights, packed as GemmI8Params::w4 describes
};

// EPI 1: fp32 dynamic-quant linear, 2: fp32 Winograd position GEMM.  PAIR: 2-CTA cluster (EPI 1).
// MAXBN bounds the tile width (and the accumulator registers).  p is __grid_constant__ so its fields are read from the
// parameter bank where they are used: as a plain by-value struct of <= 128 bytes it is copied into registers and the fp32
// epilogue is duplicated (the Qwen linear layers ran 4 % slower on an H100 80GB HBM3 at 700 W).
template <int EPI, bool PAIR, int MAXBN>
__global__ void __launch_bounds__(kThreads, 1)
gemm_i8_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                     const __grid_constant__ KParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // dynamic smem base is only guaranteed 16B aligned: round up to 1024 (SWIZZLE_128B requirement)
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    uint8_t* smem = smem_raw + (base - raw);
    const int num_kb = (p.K + kBK - 1) / kBK;
    // "fixed tile": the CTA's n chunk (and batch) never changes, so its weights can stay resident and its per-column
    // constants are loaded once -- and, since neither depends on the previous layer, BEFORE griddepcontrol.wait.
    const bool fixed_tile = !PAIR && (p.one_tile || p.n_chunks * p.batch == 1);
    const int w4 = (EPI == 1 && !PAIR && p.w4) ? 1 : 0;
    const SmemPlan pl = make_plan(p.bn, fixed_tile ? 1 : p.n_chunks * p.batch, num_kb, PAIR, w4);
    int nc0 = 0, bt0 = 0;
    if (p.one_tile) { nc0 = blockIdx.x % p.n_chunks; bt0 = (blockIdx.x / p.n_chunks) / p.m_tiles; }
    const int S = pl.stages;

    const uint32_t bar0 = base + pl.off_bars;
    auto full_bar = [&](int s) { return bar0 + 8u * s; };
    auto empty_bar = [&](int s) { return bar0 + 8u * (kMaxStages + s); };
    const uint32_t bres_bar = bar0 + 8u * (2 * kMaxStages);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t rank = PAIR ? cluster_rank() : 0u;
    const int unit = PAIR ? (int)(blockIdx.x >> 1) : (int)blockIdx.x;
    const int units = PAIR ? (int)(gridDim.x >> 1) : (int)gridDim.x;
    const int work_total = p.batch * p.m_tiles * p.n_chunks;
    const int tile_rows = PAIR ? 2 * kBM : kBM;

    if (warp == 8 && lane == 0) {
        prefetch_tmap(&tmap_a);
        prefetch_tmap(&tmap_b);
        for (int s = 0; s < S; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), PAIR ? 16 : 8); }
        mbar_init(bres_bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    }
    __syncthreads();
    if (PAIR) cluster_sync_all();    // the peer's barriers are initialised before anyone signals them

    if (warp == 8) {
        // ================= TMA producer =================
        if (lane == 0 && pl.resident_b) {    // weights: once per CTA, all K blocks (4-bit: packed, expanded by the consumers)
            mbar_expect_tx(bres_bar, (uint32_t)((p.bn * kBK * num_kb) >> w4));
            for (int kb = 0; kb < num_kb; ++kb)
                tma_load_2d(base + (w4 ? pl.off_resp : pl.off_resb) + ((kb * p.bn * kBK) >> w4), &tmap_b, bres_bar, kb * (kBK >> w4),
                            bt0 * p.b_batch_rows + nc0 * p.bn);
        }
        pdl_wait();
        if (lane == 0) {
            const int half_bn = p.bn >> 1;
            int stage = 0, phase = 0;
            for (int w = unit; w < work_total; w += units) {
                const int nc = w % p.n_chunks, wq = w / p.n_chunks;
                const int mt = wq % p.m_tiles, bt = wq / p.m_tiles;
                const int a_row = bt * p.a_batch_rows + mt * tile_rows + (int)rank * kBM, b_row = bt * p.b_batch_rows + nc * p.bn;
                for (int kb = 0; kb < num_kb; ++kb) {
                    mbar_wait(empty_bar(stage), phase ^ 1);
                    mbar_expect_tx(full_bar(stage), (uint32_t)(kStageBytesA + (PAIR || !pl.resident_b ? (p.bn * kBK) >> w4 : 0)));
                    const uint32_t a_dst = base + stage * pl.stage_bytes;
                    tma_load_2d(a_dst, &tmap_a, full_bar(stage), kb * kBK, a_row);
                    if (PAIR)
                        tma_load_2d_multicast(a_dst + kStageBytesA + rank * half_bn * kBK, &tmap_b, full_bar(stage), kb * kBK,
                                              b_row + (int)rank * half_bn, (uint16_t)3);
                    else if (!pl.resident_b)
                        tma_load_2d(a_dst + kStageBytesA + (w4 ? p.bn * kBK : 0), &tmap_b, full_bar(stage), kb * (kBK >> w4), b_row);
                    if (++stage == S) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        // ================= two consumer warpgroups: wgmma main loop + epilogue =================
        const int ct = threadIdx.x;                  // 0..255
        const int wg = ct >> 7;                      // rows [64 wg, 64 wg + 64) of the tile
        const int r_base = wg * 64 + (warp & 3) * 16 + (lane >> 2);
        const int q4 = lane & 3;
        float* cst = reinterpret_cast<float*>(smem + pl.off_consts);
        const bool blocked = EPI == 1 && !PAIR && p.bsteps != 0;   // K-blocked weight scales (finish_block below)
        const int* wsum = reinterpret_cast<const int*>(cst) + 2 * kMaxBN;
        auto load_consts = [&](int n0, int cb) {
            for (int j = ct; j < p.bn; j += kConsumerThreads) {
                int n = n0 + j;
                const bool v = n < p.OC;
                n += cb;
                if (blocked) {                   // the per-block tables are read from global memory by finish_block
                    cst[kMaxBN + j] = (v && p.has_bias) ? p.bias[n] : 0.f;
                    continue;
                }
                cst[j] = v ? p.wscale[n] : 0.f;
                cst[kMaxBN + j] = (v && p.has_bias) ? p.bias[n] : 0.f;
                reinterpret_cast<int*>(cst)[2 * kMaxBN + j] = v ? p.wsum128[n] : 0;
                if (EPI == 1) {
                    cst[3 * kMaxBN + j] = v ? p.wsumf[n] : 0.f;
                    cst[4 * kMaxBN + j] = (v && p.wzero) ? p.wzero[n] : 0.f;
                }
            }
        };
        if (fixed_tile) {                            // per-column constants are the same for every tile: load once
            load_consts(nc0 * p.bn, bt0 * p.c_batch_stride);
            named_sync(1, kConsumerThreads);
        }
        // 4-bit weights: rows of 64 packed bytes (K block of 128), 16-byte group g holding K 32 g + j in its low nibbles and
        // K 32 g + 16 + j in its high ones, become rows of the 128B-swizzled int8 tile the TMA would have written (u = q + 8 in
        // 0..15; the epilogue's wsum128 / wsumf / wzero carry the offset).  Written through the generic proxy, so fenced for
        // the wgmmas' async proxy; both warpgroups read every row, so both expand and meet at named barrier 2.
        auto expand_w4 = [&](uint32_t pk, uint32_t dst, int rows) {     // shared-memory addresses
#pragma unroll 1
            for (int i = ct; i < rows * 4; i += kConsumerThreads) {
                const uint32_t r = (uint32_t)i >> 2, g = (uint32_t)i & 3u, m = 0x0F0F0F0Fu;
                uint32_t v0, v1, v2, v3;
                asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];\n" : "=r"(v0), "=r"(v1), "=r"(v2), "=r"(v3)
                             : "r"(pk + r * (kBK / 2) + g * 16));
                const uint32_t row = dst + r * kBK;
                asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};\n" ::"r"(row + (((2 * g) ^ (r & 7)) << 4)),
                             "r"(v0 & m), "r"(v1 & m), "r"(v2 & m), "r"(v3 & m) : "memory");
                asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};\n" ::"r"(row + (((2 * g + 1) ^ (r & 7)) << 4)),
                             "r"((v0 >> 4) & m), "r"((v1 >> 4) & m), "r"((v2 >> 4) & m), "r"((v3 >> 4) & m) : "memory");
            }
            asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
            named_sync(2, kConsumerThreads);
        };
        pdl_wait();
        if (pl.resident_b) mbar_wait(bres_bar, 0);
        if (w4 && pl.resident_b) expand_w4(base + pl.off_resp, base + pl.off_resb, p.bn * num_kb);
        auto release = [&](int s) {                  // this warp's MMAs on stage s have completed
            __syncwarp();
            if (lane == 0) {
                mbar_arrive(empty_bar(s));
                if (PAIR) mbar_arrive_cluster(mapa(empty_bar(s), rank ^ 1u));
            }
        };
        const int nblk = p.bn >> 3;
        int stage = 0, phase = 0;
        int acc[MAXBN / 2];
#pragma unroll
        for (int i = 0; i < MAXBN / 2; ++i) acc[i] = 0;
        // K-blocked weight scales: the MMAs use acc[0, bn / 2) (bn <= MAXBN / 2), acc[MAXBN / 4 + i] holds the fp32 running sum
        // of accumulator i as bits.  Block b's int32 accumulators are finished in the order of mnn_oracle_linear_w8_dynamic_blocks:
        //   part = float(acc + 128 sum_b w) * alpha_b;  part *= dq;  part += (dq * -128) * ws_b;  part = xsb * wzero_b + part;  f += part
        auto finish_block = [&](int b, int mt, int n0) {
            float dqm[2], corr[2], xs[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = mt * kBM + r_base + 8 * h;
                const bool v = m < p.M;
                dqm[h] = v ? p.dq[m] : 0.f;
                xs[h] = v ? p.xsb[(size_t)m * p.blocks + b] : 0.f;
                corr[h] = __fmul_rn(dqm[h], -128.f);
            }
            const size_t tb = (size_t)b * p.N;
#pragma unroll
            for (int j = 0; j < MAXBN / 16; ++j) {
                if (j < nblk) {
                    const int n = n0 + j * 8 + 2 * q4;
                    float2 al = make_float2(0.f, 0.f), wz = al, ws = al;
                    int2 w128 = make_int2(0, 0);
                    if (n < p.N) {
                        al = __ldg(reinterpret_cast<const float2*>(p.balpha + tb + n));
                        wz = __ldg(reinterpret_cast<const float2*>(p.bwzero + tb + n));
                        ws = __ldg(reinterpret_cast<const float2*>(p.bws + tb + n));
                        w128 = __ldg(reinterpret_cast<const int2*>(p.bw128 + tb + n));
                    }
#pragma unroll
                    for (int h = 0; h < 2; ++h)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int i = j * 4 + 2 * h + e;
                            float part = __fmul_rn(__int2float_rn(acc[i] + (e ? w128.y : w128.x)), e ? al.y : al.x);
                            part = __fmul_rn(part, dqm[h]);
                            part = __fadd_rn(part, __fmul_rn(corr[h], e ? ws.y : ws.x));
                            part = __fadd_rn(__fmul_rn(xs[h], e ? wz.y : wz.x), part);
                            acc[MAXBN / 4 + i] = __float_as_int(__fadd_rn(__int_as_float(acc[MAXBN / 4 + i]), part));
                        }
                }
            }
        };
        for (int w = unit; w < work_total; w += units) {
            const int nc = w % p.n_chunks, wq = w / p.n_chunks;
            const int mt = wq % p.m_tiles, bt = wq / p.m_tiles;
            const int n0 = nc * p.bn;
            if (!fixed_tile) {
                named_sync(1, kConsumerThreads);     // the previous tile's readers of the constants are done
                load_consts(n0, bt * p.c_batch_stride);
                named_sync(1, kConsumerThreads);
            }
            int prev = -1;
            if (blocked) {
#pragma unroll
                for (int i = MAXBN / 4; i < MAXBN / 2; ++i) acc[i] = 0;   // the fp32 running sums (+0.0f)
            }
            for (int kb = 0; kb < num_kb; ++kb) {
                mbar_wait(full_bar(stage), phase);  // TMA bytes have landed
                if (w4 && !pl.resident_b)
                    expand_w4(base + stage * pl.stage_bytes + kStageBytesA + p.bn * kBK, base + stage * pl.stage_bytes + kStageBytesA, p.bn);
                const uint32_t a_addr = base + stage * pl.stage_bytes + wg * 64 * kBK;
                const uint32_t b_addr = pl.resident_b ? base + pl.off_resb + kb * p.bn * kBK : base + stage * pl.stage_bytes + kStageBytesA;
                const int kleft = p.K - kb * kBK;
                const int nmma = kleft >= kBK ? 4 : (kleft + 31) / 32;
                fence_acc(acc);
                wgmma_fence();
                if (blocked) {
                    // every block's first k-step starts its int32 accumulators from zero; its last one is waited for and the
                    // block finished into the fp32 sums before the next block's MMAs are issued
                    for (int k = 0; k < nmma; ++k) {
                        const int ks = kb * 4 + k;
                        wgmma_bn<Kind::S8, MAXBN>(acc, p.bn, gdesc_sw128(a_addr + k * 32), gdesc_sw128(b_addr + k * 32), kBK,
                                                  ks % p.bsteps != 0);
                        if ((ks + 1) % p.bsteps == 0) {
                            wgmma_commit();
                            wgmma_wait<0>();
                            fence_acc(acc);
                            finish_block(ks / p.bsteps, mt, n0);
                            fence_acc(acc);
                            wgmma_fence();
                        }
                    }
                } else {
                    for (int k = 0; k < nmma; ++k)
                        wgmma_bn<Kind::S8, MAXBN>(acc, p.bn, gdesc_sw128(a_addr + k * 32), gdesc_sw128(b_addr + k * 32), kBK, (kb | k) != 0);
                }
                wgmma_commit();
                wgmma_wait<1>();                     // the previous stage's MMAs are done: hand its slot back
                fence_acc(acc);
                if (prev >= 0) release(prev);
                prev = stage;
                if (++stage == S) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
            fence_acc(acc);
            release(prev);

            // ---- epilogue from the accumulator fragments: register i = row r_base + 8 * ((i >> 1) & 1),
            //      column 8 * (i >> 2) + 2 * q4 + (i & 1)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = mt * tile_rows + (int)rank * kBM + r_base + 8 * h;
                if (m >= p.M) continue;
                float dqm = 0.f, ss = 0.f, corr = 0.f;
                if (EPI == 1 && !blocked) { dqm = p.dq[m]; ss = p.srcsum[m]; corr = __fmul_rn(dqm, -128.f); }
                float* yrow = p.y_f32 + ((size_t)bt * p.a_batch_rows + m) * p.ldy;
                // float2 stores need an 8-byte aligned row: an even ldy and y itself 8-byte aligned (y need only be 4-byte aligned)
                const bool vec_ok = (p.ldy & 1) == 0 && ((uintptr_t)p.y_f32 & 7) == 0;
#pragma unroll
                for (int j = 0; j < MAXBN / 8; ++j) {
                    if (j < nblk) {
                        const int c = j * 8 + 2 * q4, n = n0 + c;
                        if (n < p.OC) {
                            float o[2];
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                const int jj = c + e;
                                float f;
                                if (blocked) {
                                    f = __int_as_float(acc[(MAXBN / 4 + j * 4 + 2 * h + e) & (MAXBN / 2 - 1)]);
                                } else {
                                    f = __fmul_rn(__int2float_rn(acc[j * 4 + 2 * h + e] + wsum[jj]), cst[jj]);
                                    if (EPI == 1) {
                                        f = __fmul_rn(f, dqm);
                                        f = __fadd_rn(f, __fmul_rn(corr, cst[3 * kMaxBN + jj]));
                                        f = __fadd_rn(__fmul_rn(ss, cst[4 * kMaxBN + jj]), f);
                                    }
                                }
                                if (EPI == 1) {
                                    if (p.has_bias) f = __fadd_rn(f, cst[kMaxBN + jj]);
                                    if (p.relu | p.relu6) { f = fminf(f, p.relu6 ? 6.0f : 3.4028234663852886e38f); f = fmaxf(f, 0.f); }
                                } else {
                                    // Winograd position GEMM (avx/GemmInt8.cpp:672-772 float branch): acc*scale[a][oc] + offset[a][oc]
                                    f = __fadd_rn(f, cst[kMaxBN + jj]);
                                }
                                o[e] = f;
                            }
                            if (vec_ok && n + 1 < p.OC) {
                                *reinterpret_cast<float2*>(yrow + n) = make_float2(o[0], o[1]);
                            } else {
                                yrow[n] = o[0];
                                if (n + 1 < p.OC) yrow[n + 1] = o[1];
                            }
                        }
                    }
                }
            }
        }
    }
    __syncthreads();
    if (PAIR) cluster_sync_all();    // the peer may still multicast into this CTA's smem / signal its barriers until here
}

template <class Kern>
cudaError_t launch(Kern kern, const CUtensorMap* ta, const CUtensorMap* tb, const KParams& p, int grid, int smem, int smem_cap,
                   bool pair, cudaStream_t stream) {
    cudaError_t e = ensure_max_dynamic_smem((const void*)kern, smem_cap);
    if (e != cudaSuccess) return e;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    if (pair) {
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = 2;
        attr[0].val.clusterDim.y = 1;
        attr[0].val.clusterDim.z = 1;
    } else {
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[0].val.programmaticStreamSerializationAllowed = 1;
    }
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    ++g_launch_count;
    return cudaLaunchKernelEx(&cfg, kern, *ta, *tb, p);
}

KParams make_params(const GemmI8Params& g, int bn) {
    KParams p;
    p.M = g.M; p.N = g.N; p.K = g.K; p.bn = bn;
    p.n_chunks = (g.N + bn - 1) / bn;
    p.m_tiles = (g.M + kBM - 1) / kBM;
    p.wscale = g.wscale; p.bias = g.bias; p.wsum128 = g.wsum128; p.OC = g.OC; p.ldy = g.ldy;
    p.y_f32 = g.y_f32; p.dq = g.dq; p.srcsum = g.srcsum; p.wsumf = g.wsumf; p.wzero = g.wzero;
    p.relu = g.relu; p.relu6 = g.relu6; p.has_bias = g.bias != nullptr;
    p.bsteps = g.bs / 32; p.blocks = g.blocks;
    p.balpha = g.balpha; p.bwzero = g.bwzero; p.bws = g.bws; p.xsb = g.xsb; p.bw128 = g.bw128;
    p.batch = g.batch > 0 ? g.batch : 1;
    p.a_batch_rows = g.a_batch_rows; p.b_batch_rows = g.b_batch_rows; p.c_batch_stride = g.c_batch_stride;
    p.one_tile = 0;
    p.w4 = g.w4;
    return p;
}

}  // namespace

GemmI8Launch gemm_i8_wgmma_launch(const GemmI8Params& g, int bn, int sm_count) {
    const KParams p = make_params(g, bn);
    GemmI8Launch l;
    l.n_chunks = p.n_chunks;
    l.m_tiles = p.m_tiles;
    l.num_kb = (g.K + kBK - 1) / kBK;
    l.items = p.batch * p.m_tiles * p.n_chunks;
    l.grid = l.items < sm_count ? l.items : sm_count;
    l.one_tile = l.grid == l.items ? 1 : 0;
    const bool fixed_tile = l.one_tile || p.n_chunks * p.batch == 1;
    const SmemPlan pl = make_plan(bn, fixed_tile ? 1 : p.n_chunks * p.batch, l.num_kb, false, g.w4);
    l.resident_b = pl.resident_b;
    l.stages = pl.stages;
    l.smem = pl.total + 1024;
    return l;
}

cudaError_t launch_gemm_i8_wgmma(const GemmI8Params& g, const void* tmap_a, const void* tmap_b, int bn, cudaStream_t stream,
                                 int sm_count) {
    if (bn < 16 || bn > kMaxBN || (bn & 15) || g.y_f32 == nullptr) return cudaErrorInvalidValue;
    if (g.bs && (g.wino || bn > kMaxBN / 2 || g.bs % 32 || g.K % g.bs || g.blocks != g.K / g.bs)) return cudaErrorInvalidValue;
    if (g.w4 && (g.wino || g.K % 32)) return cudaErrorInvalidValue;
    KParams p = make_params(g, bn);
    const GemmI8Launch l = gemm_i8_wgmma_launch(g, bn, sm_count);
    p.one_tile = l.one_tile;
    const CUtensorMap* ta = reinterpret_cast<const CUtensorMap*>(tmap_a);
    const CUtensorMap* tb = reinterpret_cast<const CUtensorMap*>(tmap_b);
    if (g.wino) return launch(gemm_i8_wgmma_kernel<2, false, 256>, ta, tb, p, l.grid, l.smem, 227 * 1024, false, stream);
    return launch(gemm_i8_wgmma_kernel<1, false, 256>, ta, tb, p, l.grid, l.smem, 227 * 1024, false, stream);
}

cudaError_t launch_gemm_i8_2cta(const GemmI8Params& g, const void* tmap_a, const void* tmap_b_half, int bn, cudaStream_t stream,
                                int sm_count) {
    if (bn < 32 || bn > kMaxBN || (bn & 31) || g.y_f32 == nullptr || g.wino || g.bs || g.w4) return cudaErrorInvalidValue;
    KParams p = make_params(g, bn);
    const GemmI8Launch l = gemm_i8_2cta_launch(g, bn, sm_count);
    p.batch = 1;
    p.m_tiles = l.m_tiles;
    return launch(gemm_i8_wgmma_kernel<1, true, 256>, reinterpret_cast<const CUtensorMap*>(tmap_a),
                  reinterpret_cast<const CUtensorMap*>(tmap_b_half), p, l.grid, l.smem, 227 * 1024, true, stream);
}

GemmI8Launch gemm_i8_2cta_launch(const GemmI8Params& g, int bn, int sm_count) {
    GemmI8Launch l;
    l.n_chunks = (g.N + bn - 1) / bn;
    l.m_tiles = (g.M + 2 * kBM - 1) / (2 * kBM);
    l.num_kb = (g.K + kBK - 1) / kBK;
    l.items = l.m_tiles * l.n_chunks;
    const int pairs = l.items < sm_count / 2 ? l.items : sm_count / 2;
    l.grid = 2 * pairs;
    l.one_tile = 0;
    const SmemPlan pl = make_plan(bn, l.n_chunks, l.num_kb, true);
    l.resident_b = pl.resident_b;
    l.stages = pl.stages;
    l.smem = pl.total + 1024;
    return l;
}

}  // namespace mnnb200
