// recur_common.cuh -- what the cluster-resident recurrences of rnn.cu (LSTM / RNN) and gru.cu (GRU) share: the distributed
// shared-memory store, the bounded cluster mbarrier wait, the fixed-order gate dot product and the launch-plan search.
//
// Each recurrence runs one thread-block cluster per (direction, batch group).  The cluster's CTAs each own a slice of hidden
// units and all gate rows of R for them; every CTA holds the group's whole h_prev, double-buffered, and a step's new h slice is
// stored into every CTA's other buffer (mapa + st.shared::cluster) before an arrive on each CTA's mbarrier of that buffer.
#pragma once
#include <algorithm>

#include "hopper_common.cuh"
#include "host_util.h"
#include "rnn_ops.h"

namespace mnnb200 {
namespace {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void st_cluster(uint32_t addr, float v) {
    asm volatile("st.shared::cluster.f32 [%0], %1;\n" ::"r"(addr), "f"(v) : "memory");
}
// mbarrier wait with cluster-scope acquire (the stores it orders come from other CTAs), bounded as hop::mbar_wait is
__device__ __forceinline__ uint32_t mbar_try_wait_cluster(uint32_t bar, uint32_t parity, uint32_t hint_ns) {
    uint32_t done;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2, %3;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(done)
        : "r"(bar), "r"(parity), "r"(hint_ns)
        : "memory");
    return done;
}
__device__ __forceinline__ void mbar_wait_cluster(uint32_t bar, uint32_t parity) {
    if (mbar_try_wait_cluster(bar, parity, 0u)) return;
    long long t0 = 0;
    while (!mbar_try_wait_cluster(bar, parity, 100000u)) {
        const long long now = clock64();
        if (t0 == 0) t0 = now;
        else if (now - t0 > 8000000000ll) __trap();
    }
}

// z[q] = sum_k rrow[q * pitch + k] * hv[k] over k < n for the NG gate rows, by KS consecutive lanes (s = this lane's index
// among them): lane s keeps the partial sums of k = a mod 8 for a = s, s + KS, ..., the lanes combine bits 0 .. log2(KS) of a
// by shuffles and then each lane the remaining bits in registers, lowest bit first.  Every lane of the KS returns the sums.
// All 32 lanes of the warp call it (live or not) for the shuffles.
template <int NG, int KS>
__device__ __forceinline__ void gate_dots(float (&z)[NG], const float* __restrict__ rrow, size_t pitch,
                                          const float* __restrict__ hv, int n, int s, bool live) {
    constexpr int M = kRnnPartials / KS;
    float a[NG][M];
#pragma unroll
    for (int q = 0; q < NG; ++q)
#pragma unroll
        for (int m = 0; m < M; ++m) a[q][m] = 0.f;
    if (live) {
        for (int k0 = 0; k0 < n; k0 += kRnnPartials) {
#pragma unroll
            for (int m = 0; m < M; ++m) {
                const int k = k0 + s + KS * m;
                if (k < n) {
                    const float hk = hv[k];
#pragma unroll
                    for (int q = 0; q < NG; ++q) a[q][m] = __fmaf_rn(rrow[q * pitch + k], hk, a[q][m]);
                }
            }
        }
    }
#pragma unroll
    for (int q = 0; q < NG; ++q) {
#pragma unroll
        for (int lvl = 1; lvl < KS; lvl <<= 1)
#pragma unroll
            for (int m = 0; m < M; ++m) a[q][m] = __fadd_rn(a[q][m], __shfl_xor_sync(0xffffffffu, a[q][m], lvl));
#pragma unroll
        for (int st = 1; st < M; st <<= 1)
#pragma unroll
            for (int m = 0; m < M; m += 2 * st) a[q][m] = __fadd_rn(a[q][m], a[q][m + st]);
        z[q] = a[q][0];
    }
}

// ---- the launch plan ------------------------------------------------------------------------------------------------------
// A recurrence's shared memory per CTA: `bars` mbarriers (rounded up to 16 bytes), the double-buffered h_prev [2][rows][H],
// one float per item [rows][hs] (the LSTM's cell state, the GRU's update gate), `extra` more floats per batch row (the GRU's
// r * h_prev [rows][H] when the reset gate applies before the candidate's product), and with R resident the `ng` gate rows of
// the slice [ng][hs][rstride].
struct RecurSmem {
    int ng, bars, extra;
};

inline int recur_ks(int items) {
    int ks = kRnnPartials;
    while (ks > 1 && items * ks > kRnnThreads) ks >>= 1;
    return ks;
}

// the plan's CTA geometry and shared memory for cluster size cs
inline RnnPlan recur_shape(const RecurSmem& m, int h, int rows, int groups, int cs, bool resident) {
    RnnPlan pl;
    pl.cs = cs;
    pl.groups = groups;
    pl.rows = rows;
    pl.hs = (h + cs - 1) / cs;
    const int items = rows * pl.hs;
    pl.ks = recur_ks(items);
    pl.threads = std::min(kRnnThreads, (items * pl.ks + 31) / 32 * 32);
    pl.resident = resident ? 1 : 0;
    const long long rstride = h + (((pl.ks - h) % 32) + 32) % 32;   // rows of the resident slice pitch KS banks apart
    long long bytes = (8LL * m.bars + 15) / 16 * 16 + 4LL * (2LL * rows * h + (long long)rows * pl.hs + (long long)rows * m.extra);
    if (resident) bytes += 4LL * m.ng * pl.hs * rstride;
    pl.smem = bytes > 0x7fffffffLL ? 0x7fffffff : (int)bytes;
    pl.rstride = (int)rstride;
    return pl;
}

// The plan of a recurrence of shared memory `m` for (B, H, D) on a device of `sms` SMs with at most `smem_cap` bytes of dynamic
// shared memory per CTA; depends on nothing else, T in particular.  fits(plan): whether a cluster of the plan can be resident
// (cudaOccupancyMaxActiveClusters); a plan that cannot halves its cluster.  False when nothing fits.
template <class Fits>
bool recur_choose_plan(const RecurSmem& m, int b, int h, int d, int sms, int smem_cap, Fits fits, RnnPlan* out) {
    // batch rows of one group: their h buffers (and extra floats) within 192 KiB
    const int max_rows = std::max(1, std::min(kRnnMaxRows, 49152 / (2 * h + m.extra)));
    const int groups = (b + max_rows - 1) / max_rows, rows = (b + groups - 1) / groups;
    int top = 1;                                        // the largest power-of-two cluster with a unit per CTA
    while (top * 2 <= std::min(h, kRnnMaxCluster)) top *= 2;
    int cs = 1;                                         // enough CTAs that each has at most 32 items
    while (cs < top && (long long)rows * ((h + cs - 1) / cs) > 32) cs *= 2;
    while (cs > 1 && (long long)cs * groups * d > sms) cs /= 2;   // one CTA per SM where the card has them
    for (;;) {
        RnnPlan pl = recur_shape(m, h, rows, groups, cs, false);
        for (int c = cs; c <= top; c *= 2) {            // R resident at the smallest cluster, from cs up, whose slice fits
            const RnnPlan r = recur_shape(m, h, rows, groups, c, true);
            if (r.smem <= smem_cap) {
                pl = r;
                break;
            }
        }
        if (pl.smem <= smem_cap && fits(pl)) {
            *out = pl;
            return true;
        }
        if (cs == 1) return false;
        cs /= 2;
        top = cs;
    }
}

// the launch of one cluster per (direction, batch group): grid (cs, groups, d), cluster (cs, 1, 1)
inline cudaLaunchConfig_t recur_config(const RnnPlan& pl, int d, cudaStream_t s, cudaLaunchAttribute* attr) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(pl.cs, pl.groups, d);
    cfg.blockDim = dim3(pl.threads);
    cfg.dynamicSmemBytes = pl.smem;
    cfg.stream = s;
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = pl.cs;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cfg;
}

// cudaOccupancyMaxActiveClusters of kernel k at the plan; sets the attributes (dynamic shared memory up to smem_cap,
// non-portable cluster sizes) that the launch needs, so it precedes the plan's first launch
inline cudaError_t recur_max_active_clusters(const void* k, const RnnPlan& pl, int smem_cap, int* clusters) {
    if (!k) return cudaErrorInvalidValue;
    cudaError_t e = ensure_max_dynamic_smem(k, smem_cap);
    if (e != cudaSuccess) return e;
    if ((e = cudaFuncSetAttribute(k, cudaFuncAttributeNonPortableClusterSizeAllowed, 1)) != cudaSuccess) return e;
    cudaLaunchAttribute attr[1];
    RnnPlan one = pl;   // what fits depends on one cluster, not on the grid (whose y may pass 65535 here: resize refuses that)
    one.groups = 1;
    const cudaLaunchConfig_t cfg = recur_config(one, 1, nullptr, attr);
    return cudaOccupancyMaxActiveClusters(clusters, k, &cfg);
}

}  // namespace
}  // namespace mnnb200
