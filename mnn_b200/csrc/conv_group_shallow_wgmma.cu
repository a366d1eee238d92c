// conv_group_shallow_wgmma.cu -- the conv-group launch for 1x1 layers of ONE K block (K <= 128): four consumer warpgroups,
// each on its own stream of 64-row tiles.
//
// conv_group_wgmma.cu runs a 128-row tile at a time on two consumer warpgroups in lockstep (full-barrier wait -> wgmma -> wait
// -> epilogue -> release).  A one-K-block layer has one wgmma chain per tile and an epilogue of a few thousand cycles that is
// latency-bound at two warps per SM sub-partition, so most of the SM idles.  Here the 128-row M tiles of the CTA's schedule row
// (group_schedule, capi.cu, the same schedule over this launch's members) are split into 64-row halves dealt to four consumer
// warpgroups in turn: half g goes to warpgroup g % 4.  Each warpgroup has its own ring of activation stages and full / empty
// mbarriers, so the four chains run independently and one warpgroup's epilogue overlaps the others' loads, MMAs and
// epilogues.  There is one accumulator set per thread and no next-tile probe.
//
// The weights and the epilogue constants of a run of items with the same (layer, n chunk) are resident in shared memory for
// the whole run, in one of two slots: the producer loads run r into slot r % 2 once every consumer warp has released run r - 2.
// Every consumer warpgroup walks every run (also one that deals it no half), so each slot's barriers see every warp once per
// run.  The epilogue is the conv-group kernel's (conv_group_epilogue.cuh), so both kernels write the same bytes.
//
//   warps 16-19: producer warpgroup (setmaxnreg.dec); one thread issues the TMA loads
//   warps 0-15: four consumer warpgroups: wgmma.mma_async m64nBNk32 s8 -> CPU-exact requant -> 8-byte stores to NHWC16 rows
#include <cuda.h>
#include "common.cuh"
#include "conv_group_epilogue.cuh"
#include "hopper_common.cuh"
#include "host_util.h"
#include "kernels.h"

namespace mnnb200 {

namespace {
using namespace hop;

constexpr int kWGs = 4;                              // consumer warpgroups
constexpr int kStages = 4;                           // activation stages per consumer warpgroup
constexpr int kStageBytes = 64 * 128;                // one 64-row half of a K block of at most 128 bytes
constexpr int kWSlotBytes = kGroupMaxBN * 128;       // one run's weight tile (bn x cb)
constexpr int kConstBytes = 3 * kGroupMaxBN * 4;     // one run's epilogue constants: wscale, biasFloat, preset per column
constexpr int kOffW = kWGs * kStages * kStageBytes;
constexpr int kOffConsts = kOffW + 2 * kWSlotBytes;
constexpr int kOffLayers = kOffConsts + 2 * kConstBytes;
constexpr int kOffBars = kOffLayers + kGroupMaxLayers * (int)sizeof(GroupLayerParams);
constexpr int kNumBars = 2 * kWGs * kStages + 4;     // full / empty per (warpgroup, stage), then wfull[2], wempty[2]
constexpr int kOffSched = kOffBars + ((kNumBars * 8 + 127) & ~127);
constexpr int kSchedSmemWords = 512;
constexpr int kSmemTotal = kOffSched + kSchedSmemWords * 4;
static_assert(kOffW % 1024 == 0 && kStageBytes % 1024 == 0, "swizzled tiles need 1 KB alignment");
static_assert(kSmemTotal + 1024 <= 227 * 1024, "shallow conv group kernel: shared memory plan does not fit");

// widths up to this one keep a run's epilogue constants in registers, as conv_group_wgmma.cu's kConstRegsMaxBN
constexpr int kConstRegsMaxBN = 64;

// setmaxnreg.inc only takes registers that setmaxnreg.dec gave back in the same CTA, so the split has to fit what the CTA
// was launched with: ptxas gives 640 threads 96 registers each (65536 / 640, in steps of 8), 20 warps x 96 = 4 x 32 + 16 x 112.
// (A split above that leaves the consumers waiting in setmaxnreg.inc for good.)
constexpr int kThreadsTotal = (kWGs + 1) * 128;
constexpr int kLaunchRegs = 96;
constexpr int kProducerRegs = 32, kConsumerRegs = 112;
static_assert(kLaunchRegs * kThreadsTotal <= 65536, "shallow conv group kernel: launch register count does not fit");
static_assert(kProducerRegs + kWGs * kConsumerRegs <= (kWGs + 1) * kLaunchRegs, "shallow conv group kernel: register split does not fit");

__device__ __forceinline__ void decode_item(uint32_t w, int& layer, int& nc, int& mt, int& cnt) {
    layer = (int)(w >> kGroupItemLayerShift);
    nc = (int)((w >> kGroupItemChunkShift) & kGroupItemChunkMask);
    cnt = (int)((w >> kGroupItemCountShift) & kGroupItemCountMask) + 1;
    mt = (int)(w & kGroupItemTileMask);
}
__device__ __forceinline__ void bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(dst), "l"(src),
                 "r"(bytes), "r"(bar)
                 : "memory");
}

// One RUN on one consumer warpgroup: the items my[i], my[i + 1], ... with the same (layer, n chunk), whose 64-row halves this
// warpgroup takes every fourth of, counting from the CTA row's half `g`; on return i is the run's last item and g counts the
// run's halves.  BN is a compile-time constant (see conv_group_wgmma.cu's consume_run).
template <int BN>
__device__ __forceinline__ void shallow_run(const GroupLayerParams& lp, int n0, int ncols, const uint32_t* __restrict__ my, int& i,
                                            int& g, uint32_t base, const uint8_t* smem, int slot) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wg = warp >> 2;
    const int r_base = (warp & 3) * 16 + (lane >> 2);
    const int q4 = lane & 3;
    const int cb = __shfl_sync(0xffffffffu, lp.cb, 0);
    const float* cst = reinterpret_cast<const float*>(smem + kOffConsts + slot * kConstBytes);
    const float* wscale = cst;
    const float* bias = cst + BN;
    const int* preset = reinterpret_cast<const int*>(cst) + 2 * BN;
    const uint32_t b_addr = base + kOffW + slot * kWSlotBytes;
    const uint32_t bar0 = base + kOffBars;
    const float scale_x = lp.scale_x;
    const int minv = lp.minv, maxv = lp.maxv;
    const uint32_t min2 = (uint32_t)(minv & 0xffff) * 0x10001u, max2 = (uint32_t)(maxv & 0xffff) * 0x10001u;
    constexpr int kGroups = (BN + 31) / 32;
    uint32_t mlo[kGroups], mhi[kGroups];
    group_pad_masks<BN>(lp.OC, n0, ncols, minv, maxv, q4, mlo, mhi);
    constexpr bool kRegConsts = BN <= kConstRegsMaxBN;
    float2 ws[kRegConsts ? BN / 8 : 1], bs[kRegConsts ? BN / 8 : 1];
    if constexpr (kRegConsts) {
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            ws[j] = *reinterpret_cast<const float2*>(wscale + 8 * j + 2 * q4);
            bs[j] = *reinterpret_cast<const float2*>(bias + 8 * j + 2 * q4);
        }
    }
    // |sum (x + 128) w| <= 128 * 255 * 128 < 2^22: one K block of at most 128 bytes is always the small-accumulator case
    const int M = lp.M, ldy = lp.ldy;
    int8_t* const y = lp.y;
    const uint32_t key = my[i] >> kGroupItemChunkShift;
    int acc[BN / 2];
    for (;; ++i) {
        int L, nc, mt0, cnt;
        decode_item(my[i], L, nc, mt0, cnt);
        for (int t = 2 * mt0; t < 2 * (mt0 + cnt); ++t, ++g) {
            if ((g & (kWGs - 1)) != wg) continue;
            // half t of the layer: rows [64 t, 64 t + 64); this warpgroup's j-th half
            const int j = g >> 2, stage = j % kStages;
            const uint32_t phase = (uint32_t)(j / kStages) & 1u;
            const uint32_t full = bar0 + 8u * (wg * kStages + stage);
            const uint32_t a_addr = base + (wg * kStages + stage) * kStageBytes;
#pragma unroll
            for (int jj = 0; jj < BN / 8; ++jj) {
                const int2 v = *reinterpret_cast<const int2*>(preset + 8 * jj + 2 * q4);
                acc[4 * jj] = v.x; acc[4 * jj + 1] = v.y; acc[4 * jj + 2] = v.x; acc[4 * jj + 3] = v.y;
            }
            mbar_wait(full, phase);
            fence_acc(acc);
            wgmma_fence();
            if (cb == 128) {
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    wgmma_span<Kind::S8, BN, 0>(acc, gdesc_sw128(a_addr + k * 32), gdesc_sw128(b_addr + k * 32), 128, 1);
            } else if (cb == 64) {
#pragma unroll
                for (int k = 0; k < 2; ++k)
                    wgmma_span<Kind::S8, BN, 0>(acc, gdesc(a_addr + k * 32, kSw64, 16, 512), gdesc(b_addr + k * 32, kSw64, 16, 512), 64, 1);
            } else {
                wgmma_span<Kind::S8, BN, 0>(acc, gdesc(a_addr, kSw32, 16, 256), gdesc(b_addr, kSw32, 16, 256), 32, 1);
            }
            wgmma_commit();
            wgmma_wait<0>();
            fence_acc(acc);
            __syncwarp();
            if (lane == 0) mbar_arrive(full + 8u * (kWGs * kStages));     // this warp is done with the stage
            int8_t* yrow[2];
            int lim[2];
            const int32_t* corrp[2] = {nullptr, nullptr};
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = t * 64 + r_base + 8 * h;
                yrow[h] = y + (size_t)m * ldy + n0;
                lim[h] = m < M ? ncols : 0;
            }
            group_column_run<BN, kRegConsts, true, false>(acc, ws, bs, wscale, bias, q4, scale_x, min2, max2, mlo, mhi, yrow, lim, corrp);
        }
        const uint32_t wn = my[i + 1];
        if (wn == kGroupSchedEnd || (wn >> kGroupItemChunkShift) != key) break;
    }
}

__global__ void __launch_bounds__(kThreadsTotal, 1)
conv_group_shallow_wgmma_kernel(const __grid_constant__ GroupMapsParam mp, const GroupLayerParams* __restrict__ params, int n_layers,
                                const uint32_t* __restrict__ sched, int sched_stride) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    uint8_t* smem = smem_raw + (base - raw);
    // the launch that follows (the conv-group kernel over the other members) does not read what this one writes: let it take
    // each SM as soon as this launch's CTA there is done
    asm volatile("griddepcontrol.launch_dependents;\n" ::: "memory");

    const uint32_t bar0 = base + kOffBars;
    auto full_bar = [&](int w, int s) { return bar0 + 8u * (w * kStages + s); };
    auto empty_bar = [&](int w, int s) { return bar0 + 8u * (kWGs * kStages + w * kStages + s); };
    auto wfull_bar = [&](int s) { return bar0 + 8u * (2 * kWGs * kStages + s); };
    auto wempty_bar = [&](int s) { return bar0 + 8u * (2 * kWGs * kStages + 2 + s); };
    const GroupLayerParams* sl = reinterpret_cast<const GroupLayerParams*>(smem + kOffLayers);
    const uint32_t* grow = sched + (size_t)blockIdx.x * sched_stride;
    const bool fits = sched_stride <= kSchedSmemWords;
    if (fits) {
        uint32_t* row = reinterpret_cast<uint32_t*>(smem + kOffSched);
        for (int i = threadIdx.x; i < sched_stride; i += kThreadsTotal) row[i] = grow[i];
    }
    const uint32_t* const my = fits ? reinterpret_cast<const uint32_t*>(smem + kOffSched) : grow;
    {
        const int4* src = reinterpret_cast<const int4*>(params);
        int4* dst = reinterpret_cast<int4*>(smem + kOffLayers);
        const int n16 = n_layers * (int)(sizeof(GroupLayerParams) / 16);
        for (int i = threadIdx.x; i < n16; i += kThreadsTotal) dst[i] = src[i];
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp == 4 * kWGs && lane == 0) {
        for (int w = 0; w < kWGs; ++w)
            for (int s = 0; s < kStages; ++s) { mbar_init(full_bar(w, s), 1); mbar_init(empty_bar(w, s), 4); }
        for (int s = 0; s < 2; ++s) { mbar_init(wfull_bar(s), 1); mbar_init(wempty_bar(s), 4 * kWGs); }
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    }
    __syncthreads();

    if (warp >= 4 * kWGs) {
        // ================= TMA producer =================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(kProducerRegs));
        if (warp == 4 * kWGs && lane == 0) {
            uint32_t key = 0xffffffffu;
            int run = -1, g = 0;
            for (int i = 0;; ++i) {
                const uint32_t w = my[i];
                if (w == kGroupSchedEnd) break;
                int L, nc, mt0, cnt;
                decode_item(w, L, nc, mt0, cnt);
                const GroupLayerParams& lp = sl[L];
                const int cb = lp.cb, bn = lp.bn;
                if ((w >> kGroupItemChunkShift) != key) {
                    // a new run: its weight tile and constants into slot run % 2, once every consumer warp is done with run - 2
                    key = w >> kGroupItemChunkShift;
                    const int slot = ++run & 1;
                    if (run >= 2) mbar_wait(wempty_bar(slot), (uint32_t)((run >> 1) - 1) & 1u);
                    mbar_expect_tx(wfull_bar(slot), (uint32_t)(bn * cb + 12 * bn));
                    tma_load_2d(base + kOffW + slot * kWSlotBytes, &mp.b[L], wfull_bar(slot), 0, nc * bn);
                    bulk_load(base + kOffConsts + slot * kConstBytes, lp.ep + (size_t)nc * 3 * bn, (uint32_t)(12 * bn), wfull_bar(slot));
                }
                const void* ta = &mp.a[L];
                for (int t = 2 * mt0; t < 2 * (mt0 + cnt); ++t, ++g) {
                    const int wgi = g & (kWGs - 1), j = g >> 2, s = j % kStages;
                    mbar_wait(empty_bar(wgi, s), ((uint32_t)(j / kStages) & 1u) ^ 1u);
                    mbar_expect_tx(full_bar(wgi, s), (uint32_t)(64 * cb));
                    tma_load_2d(base + (wgi * kStages + s) * kStageBytes, ta, full_bar(wgi, s), 0, t * 64);
                }
            }
        }
    } else {
        // ================= four consumer warpgroups =================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(kConsumerRegs));
        int run = -1, g = 0;
        for (int i = 0; my[i] != kGroupSchedEnd; ++i) {
            int L, nc, mt0, cnt;
            decode_item(my[i], L, nc, mt0, cnt);
            const GroupLayerParams& lp = sl[L];
            const int bn = lp.bn, n0 = nc * bn;
            const int ncols = (lp.N - n0) < bn ? (lp.N - n0) : bn;
            const int slot = ++run & 1;
            mbar_wait(wfull_bar(slot), (uint32_t)(run >> 1) & 1u);
            switch (bn >> 4) {     // the plan takes widths up to kGroupShallowMaxBN only
                case 1: shallow_run<16>(lp, n0, ncols, my, i, g, base, smem, slot); break;
                case 2: shallow_run<32>(lp, n0, ncols, my, i, g, base, smem, slot); break;
                case 3: shallow_run<48>(lp, n0, ncols, my, i, g, base, smem, slot); break;
                case 4: shallow_run<64>(lp, n0, ncols, my, i, g, base, smem, slot); break;
                case 5: shallow_run<80>(lp, n0, ncols, my, i, g, base, smem, slot); break;
                case 6: shallow_run<96>(lp, n0, ncols, my, i, g, base, smem, slot); break;
                default: __trap();
            }
            // every warp of every consumer warpgroup releases the run's slot, also one the run dealt no half
            __syncwarp();
            if (lane == 0) mbar_arrive(wempty_bar(slot));
        }
    }
}

}  // namespace

cudaError_t launch_conv_group_shallow(const GroupMapsParam* maps_host, const GroupLayerParams* params, int n_layers,
                                      const uint32_t* sched, int sched_stride, int grid, cudaStream_t stream) {
    cudaError_t e = ensure_max_dynamic_smem((const void*)conv_group_shallow_wgmma_kernel, kSmemTotal + 1024);
    if (e != cudaSuccess) return e;
    conv_group_shallow_wgmma_kernel<<<grid, kThreadsTotal, kSmemTotal + 1024, stream>>>(*maps_host, params, n_layers, sched, sched_stride);
    return cudaGetLastError();
}

}  // namespace mnnb200
