// scatter.cu -- ScatterNd and ScatterElements of fp32 (and, without a reduction, int32) models, bit for bit the reference
// CPU's sequential loop.  GeometryScatter.cpp:13-152 lowers both ops to one While loop (buildScatterND) that the CPU runs
// with parallel = false (GeometryScatter.cpp:129, CPURaster.cpp:1194-1197): y starts as data (or zeros), then for i = 0 .. n-1
// in order the slice of update i goes to destination dst_i:
//   - without a reduction (fuse < 0, CPURaster.cpp:911-962) it is copied when 0 <= dst_i < total: the last writer wins;
//   - with ADD / SUB / MUL (fuse >= 0, CPURaster.cpp:964-1186) y[dst_i + w] = y[dst_i + w] op upd[i][w] in plain fp32, so a
//     destination that several updates share takes them in update order.
// Atomics give neither result, so:
//   scatter_init_kernel<VEC>      y = data or zeros, 16-byte vectors when total % 4 == 0 and both bases are aligned;
//   path 1, last writer:
//     scatter_owner_kernel        slot_i once per update, and atomicMax(owner[slot_i], i) into an x-entry scratch that
//                                 execute resets to -1 with a memset on the stream (so a captured graph resets it too);
//     scatter_copy_kernel<VEC>    only owner[slot_i] == i copies its slice: coalesced 16-byte or 4-byte runs;
//   path 2, index-ordered fold (ADD / SUB / MUL):
//     scatter_keys_kernel         (slot_i, i) pairs; an update that names no slot gets the key x and is dropped;
//     scatter_hist_kernel, scatter_scan_kernel, scatter_sort_kernel
//                                 a stable LSD radix sort of the pairs by slot, kScatterDigitBits per pass, as many passes
//                                 as x has bits (fixed at resize): per-tile digit histograms, an exclusive scan of each
//                                 digit's row of tiles (one CTA per digit), and a per-tile scatter that keeps the order
//                                 of equal digits;
//     scatter_fold_kernel<OP>     one thread per (segment, slice word) folds its segment's updates into y in update order
//                                 with __fadd_rn / __fsub_rn / __fmul_rn.
// A segment of L updates is L dependent fp32 operations per output word: reassociating them (a tree or an atomic sum) would
// change the bits, so a long segment costs L operations in sequence.  The fold hides the load latency by reading 32 updates
// of the segment ahead of folding them.  All loops are grid-stride with grids sized from the SM count; addresses are 64-bit.
#include <algorithm>
#include <climits>

#include "common.cuh"
#include "scatter_ops.h"

namespace mnnb200 {
namespace {

constexpr unsigned kNoSlot = 0xffffffffu;
constexpr int kFoldAhead = 32;

// slot_i, or kNoSlot.  The destination is summed exactly in 64 bits; it names a slot when every term c_k * stride[k] lies in
// int32 (where the CPU's MUL and SUM are exact too) and the sum lies in [0, total).  Every stride is a multiple of r, so the
// destination is one too.
__device__ __forceinline__ unsigned dest_slot(const ScatterParams& p, long long i) {
    long long dst = 0;
    bool ok = true;
    for (int k = p.d - 1; k >= 0; --k) {
        long long c;
        if (p.mode == 0) {
            c = __ldg(p.idx + i * p.d + k);
        } else {
            const long long rest = i / p.istride[k];
            c = k == p.axis ? (long long)__ldg(p.idx + i) : rest % p.idim[k];
        }
        const long long t = c * p.stride[k];
        ok = ok && t >= INT_MIN && t <= INT_MAX;
        dst += t;
    }
    if (!ok || dst < 0 || dst >= p.total) return kNoSlot;
    return (unsigned)(dst / p.r);
}

template <bool VEC>
__global__ void __launch_bounds__(kScatterThreads) scatter_init_kernel(const void* data, void* y, long long total) {
    using V = typename std::conditional<VEC, uint4, uint32_t>::type;
    const long long nv = total / (VEC ? 4 : 1);
    const V* __restrict__ x = static_cast<const V*>(data);
    V* __restrict__ out = static_cast<V*>(y);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nv; i += (long long)gridDim.x * blockDim.x) {
        V v;
        if (x) v = __ldg(x + i);
        else memset(&v, 0, sizeof(V));
        out[i] = v;
    }
}

__global__ void __launch_bounds__(kScatterThreads) scatter_owner_kernel(const ScatterParams p, unsigned* __restrict__ slot,
                                                                        int* __restrict__ owner) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < p.n; i += (long long)gridDim.x * blockDim.x) {
        const unsigned sl = dest_slot(p, i);
        slot[i] = sl;
        if (sl != kNoSlot) atomicMax(owner + sl, (int)i);
    }
}

// q runs over the n * s / W vectors of the updates (at most 2^31 - 1 words, so 32 bits hold it)
template <bool VEC>
__global__ void __launch_bounds__(kScatterThreads) scatter_copy_kernel(const ScatterParams p, const unsigned* __restrict__ slot,
                                                                       const int* __restrict__ owner) {
    using V = typename std::conditional<VEC, uint4, uint32_t>::type;
    constexpr int W = VEC ? 4 : 1;
    const unsigned sv = (unsigned)(p.s / W), count = (unsigned)(p.n * p.s / W);
    const long long rv = p.r / W;
    const V* __restrict__ u = static_cast<const V*>(p.upd);
    V* __restrict__ y = static_cast<V*>(p.y);
    for (unsigned q = blockIdx.x * blockDim.x + threadIdx.x; q < count; q += gridDim.x * blockDim.x) {
        const unsigned i = q / sv, v = q - i * sv;
        const unsigned sl = __ldg(slot + i);
        if (sl == kNoSlot || __ldg(owner + sl) != (int)i) continue;
        y[sl * rv + v] = __ldg(u + (long long)i * sv + v);
    }
}

__global__ void __launch_bounds__(kScatterThreads) scatter_keys_kernel(const ScatterParams p, unsigned* __restrict__ keys,
                                                                       unsigned* __restrict__ vals) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < p.n; i += (long long)gridDim.x * blockDim.x) {
        const unsigned sl = dest_slot(p, i);
        keys[i] = sl == kNoSlot ? (unsigned)p.x : sl;
        vals[i] = (unsigned)i;
    }
}

// hist[digit * tiles + tile] = the keys of the tile whose digit at `shift` is `digit`
__global__ void __launch_bounds__(kScatterThreads) scatter_hist_kernel(const unsigned* __restrict__ keys, long long n, int shift,
                                                                       unsigned* __restrict__ hist, int tiles) {
    __shared__ unsigned h[kScatterDigits];
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        __syncthreads();
        for (int d = threadIdx.x; d < kScatterDigits; d += kScatterThreads) h[d] = 0;
        __syncthreads();
        const long long e0 = (long long)tile * kScatterTile;
        for (int c = threadIdx.x; c < kScatterTile; c += kScatterThreads)
            if (e0 + c < n) atomicAdd(h + ((__ldg(keys + e0 + c) >> shift) & (kScatterDigits - 1)), 1u);
        __syncthreads();
        for (int d = threadIdx.x; d < kScatterDigits; d += kScatterThreads) hist[(long long)d * tiles + tile] = h[d];
    }
}

// exclusive scan of each digit's row hist[d * tiles .. + tiles) in place, one CTA per digit: the CTA walks its row in
// coalesced blocks of kScatterScanThreads, scans each block and carries the running total; the row's total goes to
// totals[d] (the sort kernel scans the kScatterDigits totals itself)
__global__ void __launch_bounds__(kScatterScanThreads) scatter_scan_kernel(unsigned* __restrict__ hist, int tiles,
                                                                           unsigned* __restrict__ totals) {
    __shared__ unsigned part[kScatterScanThreads];
    unsigned* row = hist + (long long)blockIdx.x * tiles;
    unsigned carry = 0;
    for (int b = 0; b < tiles; b += kScatterScanThreads) {
        const int i = b + threadIdx.x;
        const unsigned v = i < tiles ? row[i] : 0u;
        part[threadIdx.x] = v;
        __syncthreads();
        for (int off = 1; off < kScatterScanThreads; off <<= 1) {
            const unsigned add = threadIdx.x >= (unsigned)off ? part[threadIdx.x - off] : 0u;
            __syncthreads();
            part[threadIdx.x] += add;
            __syncthreads();
        }
        if (i < tiles) row[i] = carry + part[threadIdx.x] - v;
        carry += part[kScatterScanThreads - 1];
        __syncthreads();
    }
    if (threadIdx.x == 0) totals[blockIdx.x] = carry;
}

// one sort pass: each tile's pairs go to their digit's place from the scanned histogram, in tile order.  The tile is read in
// chunks of kScatterThreads consecutive pairs; within a chunk a pair's place among equal digits is its lane rank in its warp
// (match_any) after the counts of the warps before it, so equal digits keep their order.
constexpr int kScatterWarps = kScatterThreads / 32;
__global__ void __launch_bounds__(kScatterThreads) scatter_sort_kernel(const unsigned* __restrict__ kin, const unsigned* __restrict__ vin,
                                                                       unsigned* __restrict__ kout, unsigned* __restrict__ vout,
                                                                       long long n, int shift, const unsigned* __restrict__ hist,
                                                                       int tiles, const unsigned* __restrict__ totals) {
    __shared__ unsigned base[kScatterDigits];
    __shared__ unsigned digit0[kScatterDigits];   // pairs of all smaller digits: the exclusive scan of the row totals
    __shared__ unsigned wcnt[kScatterWarps][kScatterDigits];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    static_assert(kScatterDigits == kScatterThreads, "one thread per digit scans the row totals");
    digit0[threadIdx.x] = __ldg(totals + threadIdx.x);
    __syncthreads();
    for (int off = 1; off < kScatterDigits; off <<= 1) {
        const unsigned add = threadIdx.x >= (unsigned)off ? digit0[threadIdx.x - off] : 0u;
        __syncthreads();
        digit0[threadIdx.x] += add;
        __syncthreads();
    }
    const unsigned mine = digit0[threadIdx.x] - __ldg(totals + threadIdx.x);
    __syncthreads();
    digit0[threadIdx.x] = mine;
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        __syncthreads();
        for (int d = threadIdx.x; d < kScatterDigits; d += kScatterThreads) {
            base[d] = digit0[d] + hist[(long long)d * tiles + tile];
            for (int w = 0; w < kScatterWarps; ++w) wcnt[w][d] = 0;
        }
        __syncthreads();
        for (int c = 0; c < kScatterTileItems; ++c) {
            const long long e = (long long)tile * kScatterTile + c * kScatterThreads + threadIdx.x;
            const bool valid = e < n;
            const unsigned key = valid ? __ldg(kin + e) : 0u, val = valid ? __ldg(vin + e) : 0u;
            const unsigned digit = valid ? (key >> shift) & (kScatterDigits - 1) : (unsigned)kScatterDigits;
            const unsigned peers = __match_any_sync(0xffffffffu, digit);
            const unsigned rank = __popc(peers & ((1u << lane) - 1u));
            if (valid && rank == 0) wcnt[warp][digit] = __popc(peers);
            __syncthreads();
            if (valid) {
                unsigned pos = base[digit] + rank;
                for (int w = 0; w < warp; ++w) pos += wcnt[w][digit];
                kout[pos] = key;
                vout[pos] = val;
            }
            __syncthreads();
            for (int d = threadIdx.x; d < kScatterDigits; d += kScatterThreads) {
                unsigned t = 0;
                for (int w = 0; w < kScatterWarps; ++w) {
                    t += wcnt[w][d];
                    wcnt[w][d] = 0;
                }
                base[d] += t;
            }
            __syncthreads();
        }
    }
}

template <int OP>
__device__ __forceinline__ float fold_op(float a, float b) {
    if (OP == 0) return __fadd_rn(a, b);
    if (OP == 1) return __fsub_rn(a, b);
    return __fmul_rn(a, b);
}

// q runs over the n sorted pairs times the s words of a slice; the thread of a segment's first pair folds the segment
template <int OP>
__global__ void __launch_bounds__(kScatterThreads) scatter_fold_kernel(const ScatterParams p, const unsigned* __restrict__ keys,
                                                                       const unsigned* __restrict__ vals) {
    const float* __restrict__ u = static_cast<const float*>(p.upd);
    float* __restrict__ y = static_cast<float*>(p.y);
    const unsigned s = (unsigned)p.s, count = (unsigned)(p.n * p.s);
    const long long n = p.n;
    for (unsigned q = blockIdx.x * blockDim.x + threadIdx.x; q < count; q += gridDim.x * blockDim.x) {
        const unsigned j = q / s, w = q - j * s;
        const unsigned key = __ldg(keys + j);
        if (key >= (unsigned)p.x || (j > 0 && __ldg(keys + j - 1) == key)) continue;
        float* dst = y + (long long)key * p.r + w;
        float acc = *dst;
        for (long long k = j;; k += kFoldAhead) {
            float v[kFoldAhead];
            int m = 0;
#pragma unroll
            for (int b = 0; b < kFoldAhead; ++b) {
                const bool in = k + b < n && __ldg(keys + k + b) == key;
                v[b] = in ? __ldg(u + (long long)__ldg(vals + k + b) * s + w) : 0.f;
                m += in;
            }
#pragma unroll
            for (int b = 0; b < kFoldAhead; ++b)
                if (b < m) acc = fold_op<OP>(acc, v[b]);
            if (m < kFoldAhead) break;
        }
        *dst = acc;
    }
}

// up to 8 CTAs of kScatterThreads per SM; beyond that the grid-stride loops
int capped_grid(long long work, int sm_count) {
    const long long cap = 8LL * (sm_count > 0 ? sm_count : 1);
    return (int)std::max<long long>(1, std::min(cap, work));
}

long long blocks(long long work) { return (work + kScatterThreads - 1) / kScatterThreads; }

bool aligned16(const void* a) { return ((uintptr_t)a & 15) == 0; }

}  // namespace

int scatter_sort_passes(long long x) {
    int bits = 0;
    while (bits < 62 && (x >> bits) != 0) ++bits;
    return std::max(1, (bits + kScatterDigitBits - 1) / kScatterDigitBits);
}

ScatterLaunch scatter_launch(const ScatterParams& p, int reduction, int passes, int sm_count) {
    ScatterLaunch l{};
    l.init_vec = p.total % 4 == 0 && aligned16(p.data) && aligned16(p.y) ? 16 : 4;
    l.path = p.n == 0 || p.s == 0 ? 0 : (reduction < 0 ? 1 : 2);
    if (l.path == 1) {
        l.vec = p.s % 4 == 0 && p.r % 4 == 0 && aligned16(p.upd) && aligned16(p.y) ? 16 : 4;
        l.grid = capped_grid(blocks(p.n * p.s / (l.vec / 4)), sm_count);
        l.launches = 4;
    } else if (l.path == 2) {
        l.tiles = (int)((p.n + kScatterTile - 1) / kScatterTile);
        l.grid = capped_grid(blocks(p.n * p.s), sm_count);
        l.launches = 3 + 3 * passes;
    } else {
        l.launches = 1;
    }
    return l;
}

cudaError_t launch_scatter(const ScatterParams& p, int reduction, int passes, const ScatterScratch& w, int sm_count,
                           cudaStream_t s) {
    if (p.total <= 0 || p.r <= 0 || p.d < 1 || p.d > kScatterMaxDims || passes < 1 || passes > 4) return cudaErrorInvalidValue;
    const ScatterLaunch l = scatter_launch(p, reduction, passes, sm_count);
    const int ig = capped_grid(blocks(p.total / (l.init_vec / 4)), sm_count);
    if (l.init_vec == 16) scatter_init_kernel<true><<<ig, kScatterThreads, 0, s>>>(p.data, p.y, p.total);
    else scatter_init_kernel<false><<<ig, kScatterThreads, 0, s>>>(p.data, p.y, p.total);
    ++g_launch_count;
    if (l.path == 0) return cudaGetLastError();
    const int ng = capped_grid(blocks(p.n), sm_count);
    if (l.path == 1) {
        cudaError_t e = cudaMemsetAsync(w.owner, 0xff, (size_t)p.x * sizeof(int), s);
        if (e != cudaSuccess) return e;
        scatter_owner_kernel<<<ng, kScatterThreads, 0, s>>>(p, w.keys[0], w.owner);
        if (l.vec == 16) scatter_copy_kernel<true><<<l.grid, kScatterThreads, 0, s>>>(p, w.keys[0], w.owner);
        else scatter_copy_kernel<false><<<l.grid, kScatterThreads, 0, s>>>(p, w.keys[0], w.owner);
        g_launch_count += 2;
        return cudaGetLastError();
    }
    scatter_keys_kernel<<<ng, kScatterThreads, 0, s>>>(p, w.keys[0], w.vals[0]);
    const int tg = capped_grid(l.tiles, sm_count);
    for (int pass = 0; pass < passes; ++pass) {
        const int a = pass & 1, shift = pass * kScatterDigitBits;
        scatter_hist_kernel<<<tg, kScatterThreads, 0, s>>>(w.keys[a], p.n, shift, w.hist, l.tiles);
        unsigned* totals = w.hist + (long long)kScatterDigits * l.tiles;
        scatter_scan_kernel<<<kScatterDigits, kScatterScanThreads, 0, s>>>(w.hist, l.tiles, totals);
        scatter_sort_kernel<<<tg, kScatterThreads, 0, s>>>(w.keys[a], w.vals[a], w.keys[a ^ 1], w.vals[a ^ 1], p.n, shift, w.hist,
                                                           l.tiles, totals);
    }
    const int f = passes & 1;
    if (reduction == 0) scatter_fold_kernel<0><<<l.grid, kScatterThreads, 0, s>>>(p, w.keys[f], w.vals[f]);
    else if (reduction == 1) scatter_fold_kernel<1><<<l.grid, kScatterThreads, 0, s>>>(p, w.keys[f], w.vals[f]);
    else scatter_fold_kernel<2><<<l.grid, kScatterThreads, 0, s>>>(p, w.keys[f], w.vals[f]);
    g_launch_count += 2 + 3 * passes;
    return cudaGetLastError();
}

}  // namespace mnnb200
