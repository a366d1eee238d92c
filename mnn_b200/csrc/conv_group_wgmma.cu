// conv_group_wgmma.cu -- ONE persistent launch for a whole LIST of int8 convolutions.
//
// One launch per 1x1 convolution pays the launch -> barrier init -> cold TMA -> epilogue -> teardown chain for a few MB of
// traffic per layer.  Here the per-layer state (TMA descriptors + epilogue constants) lives in a device-side layer table
// and the tiles of ALL layers form one host-built schedule that gives every CTA, one per SM, an equal share of every layer's
// tiles in list order (group_schedule, capi.cu), so barriers are set up once per step, the TMA producer runs ahead across layer boundaries (the next
// layer's operands are already in flight while the current tile's epilogue drains) and there is no per-layer tail.
//
// Replaces (structure) the per-op Execution::onExecute walk of Pipeline::execute (source/core/Pipeline.cpp:1069-1140)
// over ConvInt8CutlassExecution::onExecute (source/backend/cuda/execution/int8/ConvInt8CutlassExecution.cu:381-445)
// for runs of int8 convolutions; a conv executed alone runs here as a one-layer list.  Arithmetic = the CPU backend's
// (requant_cpu_exact, common.cuh).
//
// Layer modes (kernels.h): 0 = GEMM-shaped 1x1 conv (A is the activation itself); 1 = implicit GEMM for any kernel size /
// stride <= 2 / dilation / padding: the A tile of a K block (tap, channel chunk) is gathered by R TMA boxes of BH output rows x
// TWp pixels from a 4D {C, W, H, N} view of the input -- no im2col buffer (the reference writes and re-reads one:
// Im2Col_packC_16, ConvInt8CutlassExecution.cu:16-68), out-of-image taps are zero-filled by the TMA unit and, when the input
// zero point is not 0, put back in the epilogue as z_in * sum_{OOB taps} w from a small per-border-class table.
//
// Weight tiles are CACHED in shared memory across work items (4 slots tagged (layer, n chunk, K block) + a 36 KB resident set
// for layers whose K blocks all fit): the schedule keeps all CTAs on the same layer at the same time, and
// re-fetching the same few weight lines for every item from every SM serialises in L2.
//
//   warps 8-11: producer warpgroup (setmaxnreg.dec); one thread issues the TMA loads (cp.async.bulk.tensor.2d/4d, 128B / 64B / 32B swizzle or 16-byte interleaved chunks, 6-stage ring of
//              16 KB activation tiles)
//   warps 0-7: two consumer warpgroups, 64 rows of the 128-row tile each: wgmma.mma_async m64nNk32 s8 (N = bn <= 128,
//              accumulators in registers; the per-run work is instantiated per bn, see consume_run) -> CPU-exact requant
//              -> 8-byte stores straight to the NHWC16 output rows; per-column constants staged in shared memory per
//              (layer, n chunk), the next one copied in with cp.async while the current item runs
#include <cuda.h>
#include <cstdlib>
#include "common.cuh"
#include "conv_group_epilogue.cuh"
#include "hopper_common.cuh"
#include "host_util.h"
#include "kernels.h"

namespace mnnb200 {

namespace {
using namespace hop;

constexpr int kBM = 128;
constexpr int kBK = 128;                          // bytes of K per stage (one 128B swizzle row)
constexpr int kStages = 6;                        // activation-tile ring
constexpr int kMaxBN = kGroupMaxBN;               // 128
constexpr int kStageA = kBM * kBK;                // 16 KB
constexpr int kStageB = kMaxBN * kBK;             // 16 KB
constexpr int kStageBytes = kStageA;               // the stage ring holds ACTIVATION tiles only
constexpr int kBSlots = 4;                        // weight-tile cache: (layer, n chunk, K block) -> slot
constexpr int kOffB = kStages * kStageA;
constexpr int kConstBytes = 3 * kMaxBN * 4;       // one slot: wscale, biasFloat, preset per column

constexpr int kOffResident = kOffB + kBSlots * kStageB;  // the RESIDENT weight set
constexpr int kResidentBytes = 36 * 1024;
static_assert(kOffResident % 1024 == 0, "resident weight tiles need 1 KB alignment");
constexpr int kOffConsts = kOffResident + kResidentBytes;
constexpr int kOffLayers = kOffConsts + 2 * kConstBytes;
constexpr int kOffRbTab = kOffLayers + kGroupMaxLayers * (int)sizeof(GroupLayerParams);   // producer: [3][16] row-box coordinates
constexpr int kOffBSlot = kOffRbTab + 3 * 16 * 4;                                          // [kStages] weight slot of the block in each stage
constexpr int kOffBars = kOffBSlot + 32;                                                   // (kStages ints, padded)
constexpr int kOffSched = kOffBars + 256;                                                  // the CTA's schedule row
constexpr int kSchedSmemWords = 512;
constexpr int kSmemTotal = kOffSched + kSchedSmemWords * 4;
static_assert(kSmemTotal + 1024 <= 227 * 1024, "conv group kernel: shared memory plan does not fit");
static_assert(sizeof(GroupLayerParams) % 16 == 0, "layer params are copied with 16-byte loads");
// Two consumer warpgroups and a producer WARPGROUP (warps 8-11, one thread of warp 8 issues the TMA loads).  With nine warps
// ptxas caps a thread at 168 registers (three warps share one of the SM's four 64 KB register files), too few for two
// accumulator sets; with whole warpgroups setmaxnreg moves the producer's registers to the consumers: per register file one
// producer warp at 88 and two consumer warps at 208, 504 x 32 <= 16 K registers.  (The TMA thread's bookkeeping spills below
// 88; two bn-96 sets and the epilogue fit 208.)
constexpr int kCgThreads = kConsumerThreads + 128;
constexpr int kProducerRegs = 88, kConsumerRegs = 208;
static_assert(kProducerRegs + 2 * kConsumerRegs <= 512, "conv group kernel: register split does not fit");

// work item = `cnt` consecutive M tiles of one (layer, n chunk), encoded as kernels.h describes.
// The producer pays its per-item bookkeeping (schedule word, layer parameters, descriptors) once per item.
__device__ __forceinline__ void decode_item(uint32_t w, int& layer, int& nc, int& mt, int& cnt) {
    layer = (int)(w >> kGroupItemLayerShift);
    nc = (int)((w >> kGroupItemChunkShift) & kGroupItemChunkMask);
    cnt = (int)((w >> kGroupItemCountShift) & kGroupItemCountMask) + 1;
    mt = (int)(w & kGroupItemTileMask);
}

// Has the phase of parity `parity` of barrier `bar` completed, in EVERY thread of this consumer warpgroup?  test_wait does not
// block; the AND over the warpgroup's 128 threads (named barrier 2 + wg) makes the answer the same in every warp, as the wgmmas
// it decides about need.  A completed phase stays completed until this warpgroup releases the stage, so a 'no' from one warp
// only means the stage is taken through the blocking wait later.  The barrier id is a register, so ptxas reserves all 16
// named barriers (harmless at one CTA per SM): immediate ids behind a branch or a predicate on wg make it serialise the wgmmas.
__device__ __forceinline__ bool stage_landed(uint32_t bar, uint32_t parity, int wg) {
    uint32_t all;
    asm volatile(
        "{\n"
        ".reg .pred p, q;\n"
        "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "bar.red.and.pred q, %3, 128, p;\n"
        "selp.u32 %0, 1, 0, q;\n"
        "}\n"
        : "=r"(all)
        : "r"(bar), "r"(parity), "r"(2 + wg)
        : "memory");
    return all != 0;
}

// Widths up to this one keep a second accumulator set: the next tile's first K block is issued into it before the current
// tile's epilogue, so the tensor core works while the epilogue runs.  Two sets of a wider tile do not fit the registers; such
// layers have few tiles per CTA, so there is little to overlap.
constexpr int kOverlapMaxBN = 64;

// widths up to this one keep a run's epilogue constants in registers (consume_run)
constexpr int kConstRegsMaxBN = 64;

// One RUN on one consumer warpgroup: the consecutive items my[i], my[i + 1], ... of the CTA's schedule row with the same
// (layer, n chunk), each `cnt` M tiles of rows [64 wg, 64 wg + 64) x BN columns; on return i is the run's last item.  BN is a
// compile-time constant so the accumulator arrays, the wgmma_span chain and the epilogue's column loop are fixed: a run-time
// switch on the tile width between two wgmma instructions would make ptxas serialise every one of them.
// cst = the (layer, n chunk)'s row of the epilogue table, [3][BN] in GEMM-column order: wscale, biasFloat, preset.
// fetch_next(w) is called once, with the item that follows the run, when the run's last item starts.
template <int BN, class FetchNext>
__device__ __forceinline__ void consume_run(const GroupLayerParams& lp, const GroupConvGeom* __restrict__ gp, int n0, int ncols,
                                            const uint32_t* __restrict__ my, int& i, uint32_t base, const uint8_t* smem,
                                            const float* cst, int& stage, int& phase, FetchNext fetch_next) {
    constexpr bool kTwoSets = BN <= kOverlapMaxBN;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wg = threadIdx.x >> 7;
    const int r_base = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int q4 = lane & 3;
    // lp lives in shared memory, so ptxas cannot tell these are the same in every lane; the broadcast makes the branches
    // around the wgmmas provably warp-uniform
    const int cb = __shfl_sync(0xffffffffu, lp.cb, 0);
    const int num_kb = __shfl_sync(0xffffffffu, lp.num_kb, 0);
    const float* wscale = cst;
    const float* bias = cst + BN;
    const int* preset = reinterpret_cast<const int*>(cst) + 2 * BN;
    const uint32_t bar0 = base + kOffBars;
    int acc[BN / 2];
    // the next tile's first K block while acc's epilogue runs.  Only wgmmas write it: a register write to an accumulator
    // while a wgmma pipeline is open makes ptxas serialise every wgmma of the kernel
    int nxt[kTwoSets ? BN / 2 : 1];
    const float scale_x = lp.scale_x;
    // The clamp runs on the rounded integers.  The reference's rounding round(f) = trunc(fadd_rn(f, copysign(0.5, f))) is
    // monotone non-decreasing and maps every integer bound to itself (|bound| < 2^23), and a monotone function commutes with
    // min and max, so max(min(round(f), maxv), minv) = round(max(min(f, maxv), minv)) bit for bit, also when minv > maxv.  The
    // saturations on the way are monotone and the identity on the bounds' range, so they change nothing: F2I.TRUNC at the
    // int32 range, the pack at the s16 range (conv_plan gives the kernel no bounds outside it).  (Only a NaN f, which needs a
    // non-finite table constant, would differ: fminf sends it to maxv, F2I to 0.)  Per 4 outputs that is two saturating packs
    // to s16 pairs, one s16x2 min and one max per pair, and one PRMT to the low bytes, instead of 8 FMNMX and 3 PRMTs.
    const int minv = lp.minv, maxv = lp.maxv;
    const uint32_t min2 = (uint32_t)(minv & 0xffff) * 0x10001u, max2 = (uint32_t)(maxv & 0xffff) * 0x10001u;
    // the chunk's pad channels (>= OC) are stored and must stay zero.  Their table constants are zero, so they requantise to
    // clamp(0): only a clamp without 0 needs their bytes cleared, and only in the chunk that holds them (all ones elsewhere).
    // The byte masks of the thread's 32-column groups are set here, once per run: one AND per 4 outputs in the column run, no
    // instruction to build them per tile and no second instantiation of the column run.
    const bool pad = lp.OC - n0 < ncols && (minv > 0 || maxv < 0);
    constexpr int kGroups = (BN + 31) / 32;
    uint32_t mlo[kGroups], mhi[kGroups];
#pragma unroll
    for (int G = 0; G < kGroups; ++G) {
        const int nv = pad ? lp.OC - n0 - (32 * G + 2 * (BN - 32 * G >= 32 ? 4 : 2) * q4) : 8;   // the group's valid channels
        mlo[G] = nv >= 4 ? 0xffffffffu : (nv <= 0 ? 0u : (1u << (8 * nv)) - 1u);
        mhi[G] = nv >= 8 ? 0xffffffffu : (nv <= 4 ? 0u : (1u << (8 * (nv - 4))) - 1u);
    }
    // the thread's wscale and biasFloat pairs, the same for every tile of the run: pair j = 4 G + s of the column run below.
    // Up to kConstRegsMaxBN they are read once, here; wider tiles read them from shared memory per tile, as their 4 BN / 8
    // registers next to BN / 2 accumulators do not fit.
    constexpr bool kRegConsts = BN <= kConstRegsMaxBN;
    float2 ws[kRegConsts ? BN / 8 : 1], bs[kRegConsts ? BN / 8 : 1];
    if constexpr (kRegConsts) {
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            ws[j] = *reinterpret_cast<const float2*>(wscale + 8 * j + 2 * q4);
            bs[j] = *reinterpret_cast<const float2*>(bias + 8 * j + 2 * q4);
        }
    }
    // |sum (x + 128) w| <= 128 * 255 * 128 < 2^22.  Broadcast like cb: the epilogue branches on it and on mode while the next
    // tile's wgmmas run, and a branch ptxas cannot prove uniform there makes it serialise the wgmmas
    const bool small_acc = __shfl_sync(0xffffffffu, lp.K, 0) <= 128;
    // the layer fields the epilogue uses, held in registers instead of read from lp (shared memory) for every row and column
    const int OC = lp.OC, M = lp.M, ldy = lp.ldy, mode = __shfl_sync(0xffffffffu, lp.mode, 0);
    int8_t* const y = lp.y;

    // the accumulators start at their column's preset (128 sum w, + 0x4B400000 for requant_round_small), so every wgmma
    // accumulates and the epilogue adds no per-column integer
    auto init = [&](int (&a)[BN / 2]) {
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            const int2 v = *reinterpret_cast<const int2*>(preset + 8 * j + 2 * q4);
            a[4 * j] = v.x; a[4 * j + 1] = v.y; a[4 * j + 2] = v.x; a[4 * j + 3] = v.y;
        }
    };
    // the wgmmas of the K block in the current stage into a (after wgmma_fence, before the commit); scale0 = 0: the first
    // k-step overwrites a instead of accumulating
    auto mma_block = [&](int (&a)[BN / 2], int scale0) {
        const uint32_t a_addr = base + stage * kStageBytes;
        const uint32_t b_addr = base + kOffB + (uint32_t)(*reinterpret_cast<const volatile int*>(smem + kOffBSlot + 4 * stage));
        // every K block runs its full count of k-steps in one straight run: a condition per k-step would make ptxas
        // serialise the wgmmas.  Past the end of a layer's K the weight tile holds zeros from the TMA unit (out-of-bounds
        // fill), so those k-steps add nothing.  A mode-0 layer's K block is as narrow as its K allows (conv_plan): 64 bytes are
        // two k-steps, 32 bytes one.
        if (cb == 128) {
#pragma unroll
            for (int k = 0; k < 4; ++k)
                wgmma_span<Kind::S8, BN, 0>(a, gdesc_sw128(a_addr + wg * 64 * 128 + k * 32), gdesc_sw128(b_addr + k * 32), 128, k ? 1 : scale0);
        } else if (cb == 64) {
#pragma unroll
            for (int k = 0; k < 2; ++k)
                wgmma_span<Kind::S8, BN, 0>(a, gdesc(a_addr + wg * 64 * 64 + k * 32, kSw64, 16, 512),
                                            gdesc(b_addr + k * 32, kSw64, 16, 512), 64, k ? 1 : scale0);
        } else if (cb == 32) {
            wgmma_span<Kind::S8, BN, 0>(a, gdesc(a_addr + wg * 64 * 32, kSw32, 16, 256), gdesc(b_addr, kSw32, 16, 256), 32, scale0);
        } else {
#pragma unroll
            for (int u = 0; u < 4; ++u)
                wgmma_span<Kind::S8, BN, 0>(a, gdesc(a_addr + 2 * u * (kBM * 16) + wg * 64 * 16, kSwNone, kBM * 16, 128),
                                            gdesc(b_addr + 2 * u * (BN * 16), kSwNone, BN * 16, 128), 16,
                                            u ? 1 : scale0);
        }
    };
    // prev = the stage whose MMAs were issued last and which is not released yet (-1: none)
    int prev = -1;
    auto release_prev = [&]() {
        if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(bar0 + 8u * (kStages + prev)); }
    };
    auto next_stage = [&]() {
        prev = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1; }
    };

    // the run's tiles: M tile mt of item my[i], `left` tiles of the item from mt on; last_item = my[i + 1] is not in the run
    // (a row ends with two end markers: my[i + 1] exists)
    const uint32_t key = my[i] >> kGroupItemChunkShift;
    int mt, left;
    bool last_item;
    auto start_item = [&]() {
        int L, nc;
        decode_item(my[i], L, nc, mt, left);
        const uint32_t wn = my[i + 1];
        last_item = wn == kGroupSchedEnd || (wn >> kGroupItemChunkShift) != key;
        if (last_item && wn != kGroupSchedEnd) fetch_next(wn);
    };
    start_item();
    init(acc);
    bool ahead = false;                      // the tile's first K block was issued (into acc) before the previous epilogue
    for (;;) {
        for (int kb = ahead ? 1 : 0; kb < num_kb; ++kb) {
            mbar_wait(bar0 + 8u * stage, phase);
            fence_acc(acc);
            wgmma_fence();
            mma_block(acc, 1);
            wgmma_commit();
            wgmma_wait<1>();                 // the previous stage's MMAs are done: hand its slot back
            fence_acc(acc);
            release_prev();
            next_stage();
        }
        const int mt_cur = mt;
        bool more = true;                    // the run has another tile: it becomes (mt, ...)
        if (--left > 0) ++mt;
        else if (!last_item) { ++i; start_item(); }
        else more = false;
        more = __shfl_sync(0xffffffffu, more, 0);      // (the schedule is the same in every lane; see cb)
        bool issued = false;                 // the next tile's first K block is in flight, into nxt
        if constexpr (kTwoSets) {
            // only if its stage has landed already: the epilogue never waits for a future stage.  Both ways commit one group
            // (empty if nothing was issued) and wait for all but it, so ptxas sees the same wgmma pipeline on either side.
            // (the result is the same in every lane; the broadcast lets ptxas see that, like cb's)
            if (more) issued = __shfl_sync(0xffffffffu, stage_landed(bar0 + 8u * stage, phase, wg), 0);
            fence_acc(nxt);
            wgmma_fence();
            if (issued) mma_block(nxt, 0);
            wgmma_commit();
            wgmma_wait<1>();                 // this tile's MMAs are done, the next tile's keep running
        } else {
            wgmma_wait<0>();
        }
        fence_acc(acc);
        release_prev();                      // this tile's last stage goes back before its epilogue
        if (issued) next_stage();
        else prev = -1;

        // ---- epilogue from the accumulator fragments: register i = row r_base + 8 * ((i >> 1) & 1),
        //      GEMM column 8 * (i >> 2) + 2 * q4 + (i & 1).  The chunk's columns are permuted (group_column_channel, kernels.h):
        //      in each 32-column group G the thread holds channels 32 G + 8 q4 ... + 7 of its rows (a 16-wide last group:
        //      32 G + 4 q4 ... + 3), stored with one 8-byte (4-byte) store per row and group.
        // Row setup first, for both rows of the thread: the output address, how many channels of the chunk the row stores (0 for
        // a row outside the layer) and, for a padded conv with z_in != 0, the row of the border-correction table.
        int8_t* yrow[2];
        int lim[2];
        const int32_t* corrp[2];
        bool corr = false;                   // some row of the warp is a border pixel: + z_in * sum_{OOB taps} w
        if (mode == 0) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = mt_cur * kBM + r_base + 8 * h;
                yrow[h] = y + (size_t)m * ldy + n0;
                lim[h] = m < M ? ncols : 0;
                corrp[h] = nullptr;
            }
        } else {
            // implicit-GEMM layers: which output pixel accumulator row r is, and its border class
            const GroupConvGeom& g = *gp;
            const int box_rows = g.BH * lp.TWp;
            const int corr_ld = lp.n_chunks * BN;   // the table's columns are in the same permuted order as the weights
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = r_base + 8 * h;
                yrow[h] = y;
                lim[h] = 0;
                // a row without a correction reads the interior class's row of the table, which holds zeros (or, outside the
                // layer, any row: nothing is stored)
                corrp[h] = g.corr == nullptr ? nullptr : g.corr + (size_t)(g.interior_cls < 0 ? 0 : g.interior_cls) * corr_ld + n0;
                const int j = r / box_rows, rem = r - j * box_rows;
                const int brow = rem / lp.TWp, pcol = rem - brow * lp.TWp;
                const int rb = mt_cur * lp.R + j;
                if (j < lp.R && rb < g.rowboxes) {
                    const int seg = rb % g.SEG, tt = rb / g.SEG;
                    const int oh = (tt % g.OHB) * g.BH + brow, n = tt / g.OHB;
                    const int ow = seg * lp.TWp + pcol;
                    if (ow < g.OW) {
                        yrow[h] = y + (size_t)((n * g.OH + oh) * g.OW + ow) * ldy + n0;
                        lim[h] = ncols;
                        if (g.corr != nullptr) {
                            const int cls = (int)g.hcls[oh] * g.wc_count + (int)g.wcls[ow];
                            if (cls != g.interior_cls) { corrp[h] = g.corr + (size_t)cls * corr_ld + n0; corr = true; }
                        }
                    }
                }
            }
            corr = __any_sync(0xffffffffu, corr);
        }
        // Then one straight run over every column group of both rows (group_column_run); the requant path and the border
        // correction are chosen once per run.
        if (corr) {
            if (small_acc) group_column_run<BN, kRegConsts, true, true>(acc, ws, bs, wscale, bias, q4, scale_x, min2, max2, mlo, mhi, yrow, lim, corrp);
            else group_column_run<BN, kRegConsts, false, true>(acc, ws, bs, wscale, bias, q4, scale_x, min2, max2, mlo, mhi, yrow, lim, corrp);
        } else {
            if (small_acc) group_column_run<BN, kRegConsts, true, false>(acc, ws, bs, wscale, bias, q4, scale_x, min2, max2, mlo, mhi, yrow, lim, corrp);
            else group_column_run<BN, kRegConsts, false, false>(acc, ws, bs, wscale, bias, q4, scale_x, min2, max2, mlo, mhi, yrow, lim, corrp);
        }
        if constexpr (kTwoSets) {
            // the next tile starts in acc: the preset, + its first K block if that was issued (into nxt, which is written by
            // wgmmas only); that block's stage goes back.  The wait comes before the run can end, so no path leaves the loop
            // with a wgmma in flight.
            wgmma_wait<0>();
            fence_acc(nxt);
            if (!more) break;
            release_prev();
            prev = -1;
            init(acc);
#pragma unroll
            for (int j = 0; j < BN / 2; ++j) acc[j] += issued ? nxt[j] : 0;
        } else {
            if (!more) break;
            init(acc);
        }
        ahead = issued;
    }
}

__global__ void __launch_bounds__(kCgThreads, 1)
conv_group_wgmma_kernel(const __grid_constant__ GroupMapsParam mp, const GroupLayerParams* __restrict__ params,
                        const GroupConvGeom* __restrict__ geom, int n_layers, const uint32_t* __restrict__ sched, int sched_stride) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    uint8_t* smem = smem_raw + (base - raw);

    const uint32_t bar0 = base + kOffBars;
    auto full_bar = [&](int s) { return bar0 + 8u * s; };
    auto empty_bar = [&](int s) { return bar0 + 8u * (kStages + s); };
    const GroupLayerParams* sl = reinterpret_cast<const GroupLayerParams*>(smem + kOffLayers);
    // every role reads its schedule row item by item, two dependent loads per tile in the consumers: a row that fits is read
    // from shared memory (contiguous multi-tile items keep rows to a few words per layer), a longer one from global memory
    const uint32_t* grow = sched + (size_t)blockIdx.x * sched_stride;
    const bool fits = sched_stride <= kSchedSmemWords;
    if (fits) {
        uint32_t* row = reinterpret_cast<uint32_t*>(smem + kOffSched);
        for (int i = threadIdx.x; i < sched_stride; i += kCgThreads) row[i] = grow[i];
    }
    const uint32_t* const my = fits ? reinterpret_cast<const uint32_t*>(smem + kOffSched) : grow;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    // layer table -> smem (read by every role for every item)
    {
        const int4* src = reinterpret_cast<const int4*>(params);
        int4* dst = reinterpret_cast<int4*>(smem + kOffLayers);
        const int n16 = n_layers * (int)(sizeof(GroupLayerParams) / 16);
        for (int i = threadIdx.x; i < n16; i += kCgThreads) dst[i] = src[i];
    }
    if (warp == 8 && lane == 0) {
        for (int s = 0; s < kStages; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 8); }
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    }
    __syncthreads();

    if (warp >= 8) {
        // ================= TMA producer =================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(kProducerRegs));
        if (warp == 8 && lane == 0) {
            int stage = 0, phase = 0;
            // weight-tile cache, all bookkeeping in registers (this thread's instruction count per K block is what bounds the kernel
            // on short K loops; a shared-memory tag table measured 8-30 % slower):
            //  * 4 slots of 16 KB tagged (layer, n chunk, K block), FIFO replacement: layers with <= 4 K blocks keep their weights
            //    across the M tiles a CTA computes;
            //  * one RESIDENT set in the 36 KB behind them for a layer whose K blocks ALL fit there although there are more than
            //    four (3x3 x 64 channels: 9 tiles of 4 KB): tile kb lives at kb * tile bytes, loaded during the first M tile only --
            //    without it such a layer reloads 4 KB per 7 KB activation block and runs 4 blocks deep instead of 6.
            uint32_t btag0 = 0xffffffffu, btag1 = 0xffffffffu, btag2 = 0xffffffffu, btag3 = 0xffffffffu;
            int buse0 = -1, buse1 = -1, buse2 = -1, buse3 = -1, bvictim = 0, blk = 0;
            uint32_t res_key = 0xffffffffu;      // (layer, n chunk) owning the resident set
            int res_loaded = 0, res_use = -1;    // K blocks of it already loaded; last block that read the set
            volatile int* stage_bslot = reinterpret_cast<volatile int*>(smem + kOffBSlot);
            // returns the byte offset (from kOffB) of the slot holding tile `key`; *miss = the tile has to be loaded into it
            auto b_lookup = [&](uint32_t key, bool* miss) -> int {
                *miss = false;
                int slot;
                if (key == btag0) slot = 0;
                else if (key == btag1) slot = 1;
                else if (key == btag2) slot = 2;
                else if (key == btag3) slot = 3;
                else {
                    *miss = true;
                    slot = bvictim;
                    bvictim = (bvictim + 1) & 3;
                    const int u = slot == 0 ? buse0 : (slot == 1 ? buse1 : (slot == 2 ? buse2 : buse3));
                    // the MMAs of block u read the old tile: wait until that block's stage was released (blocks <= blk - kStages
                    // are known to be: this thread waited on their empty barriers when it reused their stages)
                    if (u >= 0 && u > blk - kStages) mbar_wait(empty_bar(u % kStages), (uint32_t)((u / kStages) & 1));
                    if (slot == 0) btag0 = key; else if (slot == 1) btag1 = key; else if (slot == 2) btag2 = key; else btag3 = key;
                }
                if (slot == 0) buse0 = blk; else if (slot == 1) buse1 = blk; else if (slot == 2) buse2 = blk; else buse3 = blk;
                return slot * kStageB;
            };
            // the resident set: (layer, n chunk) `key`, K block kb, tile_bytes per K block
            auto b_resident = [&](uint32_t key, int kb, int tile_bytes, bool* miss) -> int {
                if (key != res_key) {
                    if (res_use >= 0 && res_use > blk - kStages) mbar_wait(empty_bar(res_use % kStages), (uint32_t)((res_use / kStages) & 1));
                    res_key = key;
                    res_loaded = 0;
                }
                *miss = kb >= res_loaded;
                if (*miss) res_loaded = kb + 1;
                res_use = blk;
                return kBSlots * kStageB + kb * tile_bytes;
            };
            for (int i = 0;; ++i) {
                const uint32_t w = my[i];
                if (w == kGroupSchedEnd) break;
                int L, nc, mt0, cnt;
                decode_item(w, L, nc, mt0, cnt);
                const GroupLayerParams& lp = sl[L];
                const void* ta = &mp.a[L];
                const void* tb = &mp.b[L];
                if (lp.mode == 0) {
                    const int num_kb = lp.num_kb, cb = lp.cb, brow = nc * lp.bn;
                    const uint32_t a_bytes = (uint32_t)(kBM * cb), b_bytes = (uint32_t)(lp.bn * cb);
                    const uint32_t key0 = ((uint32_t)L << 16) | ((uint32_t)nc << 8);
                    for (int t = 0; t < cnt; ++t) {
                        const int row0 = (mt0 + t) * kBM;
                        for (int kb = 0; kb < num_kb; ++kb) {
                            mbar_wait(empty_bar(stage), phase ^ 1);
                            bool miss;
                            const int bs = b_lookup(key0 | (uint32_t)kb, &miss);
                            stage_bslot[stage] = bs;
                            mbar_expect_tx(full_bar(stage), a_bytes + (miss ? b_bytes : 0u));
                            const uint32_t a_dst = base + stage * kStageBytes;
                            tma_load_2d(a_dst, ta, full_bar(stage), kb * cb, row0);
                            if (miss) tma_load_2d(base + kOffB + bs, tb, full_bar(stage), kb * cb, brow);
                            if (++stage == kStages) { stage = 0; phase ^= 1; }
                            ++blk;
                        }
                    }
                    continue;
                }
                // ---- implicit GEMM: the tile's R output rows -> (image, first input row, first input column)
                const GroupConvGeom& g = geom[L];
                const int R = lp.R, TWp = lp.TWp, cb = lp.cb;
                const int KW = g.KW, sw = g.sw, dh = g.dh, dw = g.dw, cpt = g.cpt, Cp = g.Cp;
                const void* ta1 = &mp.a1[L];
                int* rb_n = reinterpret_cast<int*>(smem + kOffRbTab);
                int* rb_ih0 = rb_n + 16;
                int* rb_iw0 = rb_n + 32;
                for (int t = 0; t < cnt; ++t) {
                const int mt = mt0 + t;
                const int BH = g.BH, box_rows = BH * TWp;    // a box = BH output rows x TWp pixels
                for (int j = 0; j < R; ++j) {
                    const int rb = mt * R + j;
                    int n = g.NB, oh = 0, seg = 0;          // n = NB: every coordinate of the box is out of bounds -> zeros
                    if (rb < g.rowboxes) { seg = rb % g.SEG; const int t = rb / g.SEG; oh = (t % g.OHB) * BH; n = t / g.OHB; }
                    rb_n[j] = n; rb_ih0[j] = oh * g.sh - g.ph; rb_iw0[j] = seg * TWp * sw - g.pw;
                }
                const int rows_bytes = R * box_rows;        // x cb = A bytes per chunk
                if (cb >= 64) {
                    // this loop runs on ONE thread, once per K block: everything that can be hoisted is (tap -> (kh, kw) by
                    // counters, stride 1 / 2 parity by mask and shift, the first two boxes' coordinates in registers)
                    int cc = 0, kh = 0, kw = 0, bk = 0;
                    const int swm = sw - 1;                          // sw is 1 or 2 (conv_plan)
                    const int n0 = rb_n[0], ih00 = rb_ih0[0], iw00 = rb_iw0[0];
                    const int n1 = rb_n[1], ih01 = rb_ih0[1], iw01 = rb_iw0[1];
                    const uint32_t key0 = ((uint32_t)L << 16) | ((uint32_t)nc << 8);
                    const bool untagged = lp.num_kb > 256;           // such a layer gets tags no other block has: always a miss
                    const uint32_t a_bytes = (uint32_t)(rows_bytes * cb), b_bytes = (uint32_t)(lp.bn * cb);
                    const int brow = nc * lp.bn;
                    // more than 4 K blocks, but all of them fit the resident set (tiles at 1 KB multiples: swizzle atoms stay aligned)
                    const bool resident = lp.num_kb > kBSlots && (b_bytes & 1023u) == 0 && lp.num_kb * (int)b_bytes <= kResidentBytes;
                    for (int kb = 0; kb < lp.num_kb; ++kb) {
                        mbar_wait(empty_bar(stage), phase ^ 1);
                        bool miss;
                        const int bs = resident ? b_resident(key0, kb, (int)b_bytes, &miss)
                                                : b_lookup(untagged ? (0x80000000u | (uint32_t)blk) : (key0 | (uint32_t)kb), &miss);
                        stage_bslot[stage] = bs;
                        mbar_expect_tx(full_bar(stage), a_bytes + (miss ? b_bytes : 0u));
                        const uint32_t a_dst = base + stage * kStageBytes;
                        const int dcol = kw * dw, drow = kh * dh, ccb = cc * cb;
                        {
                            const int iw = iw00 + dcol, par = iw & swm;
                            tma_load_4d(a_dst, par ? ta1 : ta, full_bar(stage), ccb, (iw - par) >> swm, ih00 + drow, n0);
                        }
                        if (R > 1) {
                            const int iw = iw01 + dcol, par = iw & swm;
                            tma_load_4d(a_dst + box_rows * cb, par ? ta1 : ta, full_bar(stage), ccb, (iw - par) >> swm, ih01 + drow, n1);
                        }
                        for (int j = 2; j < R; ++j) {
                            const int iw = rb_iw0[j] + dcol, par = iw & swm;
                            tma_load_4d(a_dst + j * box_rows * cb, par ? ta1 : ta, full_bar(stage), ccb, (iw - par) >> swm,
                                        rb_ih0[j] + drow, rb_n[j]);
                        }
                        if (miss) tma_load_2d(base + kOffB + bs, tb, full_bar(stage), bk, brow);
                        bk += cb;
                        if (++cc == cpt) { cc = 0; bk += Cp - cpt * cb; if (++kw == KW) { kw = 0; ++kh; } }
                        if (++stage == kStages) { stage = 0; phase ^= 1; }
                        ++blk;
                    }
                } else {
                    // 16-byte chunks (Cp not a multiple of 64): up to 8 chunks (128 bytes of K) per stage, no swizzle.  The consumer
                    // runs all 8 chunks of every K block, so a weight tile always holds 8: past the last one they are all-zero boxes
                    // (out of bounds), and whatever the activation stage holds there is multiplied by zero.  Only the weights get
                    // the extra boxes, and only when a tile is loaded: the activation boxes are R per chunk and would be paid for in
                    // every M tile by this thread.
                    const int taps = g.KH * KW;
                    for (int kb = 0; kb < lp.num_kb; ++kb) {
                        const int q0 = kb * 8;
                        const int nq = (g.chunks - q0) < 8 ? (g.chunks - q0) : 8;
                        mbar_wait(empty_bar(stage), phase ^ 1);
                        bool miss;
                        const int bs = b_lookup(lp.num_kb > 256 ? (0x80000000u | (uint32_t)blk)
                                                                : (((uint32_t)L << 16) | ((uint32_t)nc << 8) | (uint32_t)kb), &miss);
                        stage_bslot[stage] = bs;
                        mbar_expect_tx(full_bar(stage), (uint32_t)(nq * rows_bytes * 16 + (miss ? 8 * lp.bn * 16 : 0)));
                        const uint32_t a_dst = base + stage * kStageBytes;
                        for (int ql = 0; ql < nq; ++ql) {
                            const int q = q0 + ql;
                            const int tap = q / cpt, cc = q - tap * cpt;
                            const bool dummy = tap >= taps;          // the padding chunk of an odd chunk count: zeros
                            const int kh = tap / KW, kw = tap - kh * KW;
                            for (int j = 0; j < R; ++j) {
                                const int iw = rb_iw0[j] + kw * dw;
                                int par = iw % sw; par = par < 0 ? par + sw : par;
                                tma_load_4d(a_dst + ql * (kBM * 16) + j * box_rows * 16, par ? ta1 : ta, full_bar(stage), cc * 16,
                                            (iw - par) / sw, rb_ih0[j] + kh * dh, dummy ? g.NB : rb_n[j]);
                            }
                        }
                        if (miss)
                            for (int ql = 0; ql < 8; ++ql)
                                tma_load_2d(base + kOffB + bs + ql * (lp.bn * 16), tb, full_bar(stage), (q0 + ql) * 16, nc * lp.bn);
                        if (++stage == kStages) { stage = 0; phase ^= 1; }
                        ++blk;
                    }
                }
                }   // tiles of the item
            }
        }
    } else {
        // ================= two consumer warpgroups: wgmma main loop + epilogue =================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(kConsumerRegs));
        const int ct = threadIdx.x;                  // 0..255
        // two slots of epilogue constants: the current (layer, n chunk)'s table row, and the next distinct one in this CTA's
        // schedule, copied with cp.async while the current item runs
        const uint32_t slot0 = base + kOffConsts;
        auto fetch = [&](uint32_t w, int slot) {
            const GroupLayerParams& lp = sl[w >> kGroupItemLayerShift];
            const int nc = (int)((w >> kGroupItemChunkShift) & kGroupItemChunkMask);
            if (ct < 3 * lp.bn / 4)         // 3 x bn words, 16 bytes per thread
                cp_async16(slot0 + slot * kConstBytes + 16u * ct, lp.ep + (size_t)nc * 3 * lp.bn + 4 * ct, true);
            cp_async_commit();
        };
        int cur = 1;
        int stage = 0, phase = 0;

        uint32_t w = my[0];
        if (w != kGroupSchedEnd) fetch(w, 0);
        for (int i = 0; w != kGroupSchedEnd; w = my[++i]) {
            // a run of items with the same (layer, n chunk) starts at my[i]
            int L, nc, mt0, cnt;
            decode_item(w, L, nc, mt0, cnt);
            const GroupLayerParams& lp = sl[L];
            const int bn = lp.bn, n0 = nc * bn;
            const int ncols = (lp.N - n0) < bn ? (lp.N - n0) : bn;      // valid (16-padded) columns of this chunk
            // this run's constants were fetched into the other slot during the previous run: once every consumer's copies have
            // landed (and so every consumer is done reading the old slot), switch
            cp_async_wait<0>();
            named_sync(1, kConsumerThreads);
            cur ^= 1;
            auto fetch_next = [&](uint32_t wn) { fetch(wn, cur ^ 1); };
            const float* cst = reinterpret_cast<const float*>(smem + kOffConsts + cur * kConstBytes);
            switch (lp.bn >> 4) {     // conv_plan: bn is a multiple of 16 <= kGroupMaxBN
                case 1: consume_run<16>(lp, geom + L, n0, ncols, my, i, base, smem, cst, stage, phase, fetch_next); break;
                case 2: consume_run<32>(lp, geom + L, n0, ncols, my, i, base, smem, cst, stage, phase, fetch_next); break;
                case 3: consume_run<48>(lp, geom + L, n0, ncols, my, i, base, smem, cst, stage, phase, fetch_next); break;
                case 4: consume_run<64>(lp, geom + L, n0, ncols, my, i, base, smem, cst, stage, phase, fetch_next); break;
                case 5: consume_run<80>(lp, geom + L, n0, ncols, my, i, base, smem, cst, stage, phase, fetch_next); break;
                case 6: consume_run<96>(lp, geom + L, n0, ncols, my, i, base, smem, cst, stage, phase, fetch_next); break;
                case 7: consume_run<112>(lp, geom + L, n0, ncols, my, i, base, smem, cst, stage, phase, fetch_next); break;
                case 8: consume_run<128>(lp, geom + L, n0, ncols, my, i, base, smem, cst, stage, phase, fetch_next); break;
                default: __trap();
            }
        }
    }
    // launched programmatically after the shallow kernel (group_launch, capi.cu): this grid ends only after that one has, so
    // the launches after it on the stream see both grids' outputs (a no-op in a launch without a programmatic predecessor)
    asm volatile("griddepcontrol.wait;\n" ::: "memory");
}

}  // namespace

cudaError_t launch_conv_group(const GroupMapsParam* maps_host, const GroupLayerParams* params, const GroupConvGeom* geom, int n_layers,
                              const uint32_t* sched, int sched_stride, int grid, bool programmatic, cudaStream_t stream) {
    cudaError_t e = ensure_max_dynamic_smem((const void*)conv_group_wgmma_kernel, 227 * 1024);
    if (e != cudaSuccess) return e;
    ++g_launch_count;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(kCgThreads);
    cfg.dynamicSmemBytes = kSmemTotal + 1024;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = programmatic ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, conv_group_wgmma_kernel, *maps_host, params, geom, n_layers, sched, sched_stride);
}

}  // namespace mnnb200
