// gather.cu -- the gathers of fp32 (and int32) models: Gather / GatherV2 / GatherND as one slice gather, GatherElements as an
// element gather, and the int32 <-> fp32 Cast.  Elements are 4 bytes of any type: nothing here looks at their value.
//
// gather_slices_kernel<VEC>: the op copies slices of `inside` contiguous elements, so it is bound by its loads and stores.  A
// CTA works on tiles: up to kGatherThreads slices whose vectors add up to about kGatherTileVecs, or one chunk of that many
// vectors of one long slice.
//   1. the first threads of the CTA read one slice's index (tuple) each, exactly once, and turn it into a source offset in
//      vectors, or -1 when it lies outside the params (shared memory);
//   2. all threads copy the tile's vectors, consecutive threads taking consecutive vectors of the output, so loads within a
//      slice and all stores are coalesced: 16-byte vectors when inside % 4 == 0 and both bases are 16-byte aligned (VEC), else
//      4-byte elements.  A source offset of -1 writes zeros.
// A grid-stride loop over the tiles holds any number of slices; addresses are 64-bit.
#include <algorithm>

#include "common.cuh"
#include "gather_ops.h"

namespace mnnb200 {
namespace {

template <bool VEC>
__global__ void __launch_bounds__(kGatherThreads) gather_slices_kernel(const GatherParams p, int slices_per_tile, int chunks,
                                                                       long long tiles) {
    using V = typename std::conditional<VEC, uint4, uint32_t>::type;
    constexpr int W = VEC ? 4 : 1;
    __shared__ long long soff[kGatherThreads];
    const long long slices = p.outside * p.n;
    const long long rv = p.inside / W;                        // vectors per slice
    const long long chunk_vecs = chunks > 1 ? kGatherTileVecs : rv;
    const V* __restrict__ x = static_cast<const V*>(p.x);
    V* __restrict__ y = static_cast<V*>(p.y);
    for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const long long group = tile / chunks;
        const long long c0 = (tile - group * chunks) * chunk_vecs;
        const long long s0 = group * slices_per_tile;
        const int ns = (int)std::min<long long>(slices_per_tile, slices - s0);
        __syncthreads();                                      // the previous tile's offsets are no longer read
        if ((int)threadIdx.x < ns) {
            const long long s = s0 + threadIdx.x;
            const long long o = s / p.n, j = s - o * p.n;
            const int* t = p.idx + o * p.idx_outer + j * p.d;
            long long off = o * p.x_outer;
            bool ok = true;
            for (int k = 0; k < p.d; ++k) {
                const int v = __ldg(t + k);
                ok = ok && v >= 0 && v < p.dim[k];
                off += (long long)v * p.stride[k];
            }
            soff[threadIdx.x] = ok ? off / W : -1;
        }
        __syncthreads();
        // vectors of each slice in this tile: at most kGatherTileVecs, and ns * span at most kGatherThreads * kGatherTileVecs
        const unsigned span = (unsigned)std::min<long long>(chunk_vecs, rv - c0);
        const unsigned total = (unsigned)ns * span;
        for (unsigned q = threadIdx.x; q < total; q += kGatherThreads) {
            const unsigned t = q / span;
            const long long v = c0 + (q - t * span);
            const long long off = soff[t];
            V val;
            if (off >= 0) val = __ldg(x + off + v);
            else memset(&val, 0, sizeof(V));
            y[(s0 + t) * rv + v] = val;
        }
    }
}

__global__ void __launch_bounds__(kGatherThreads) gather_elements_kernel(const GatherElementsParams p) {
    const uint32_t* __restrict__ x = static_cast<const uint32_t*>(p.x);
    uint32_t* __restrict__ y = static_cast<uint32_t*>(p.y);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < p.count; i += (long long)gridDim.x * blockDim.x) {
        const int v = __ldg(p.idx + i);
        uint32_t val = 0;
        if (v >= 0 && v < p.axis_len) {
            long long rest = i, off = 0;
            for (int k = p.rank - 1; k >= 0; --k) {
                const long long c = rest % p.odim[k];
                rest /= p.odim[k];
                off += (k == p.axis ? (long long)v : c) * p.xstride[k];
            }
            val = __ldg(x + off);
        }
        y[i] = val;
    }
}

__global__ void __launch_bounds__(kGatherThreads) cast_i32_f32_kernel(const int* __restrict__ x, float* __restrict__ y, long long n) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        y[i] = __int2float_rn(__ldg(x + i));
}

__global__ void __launch_bounds__(kGatherThreads) cast_f32_i32_kernel(const float* __restrict__ x, int* __restrict__ y, long long n) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float f = __ldg(x + i);
        y[i] = (f >= -2147483648.f && f < 2147483648.f) ? __float2int_rz(f) : INT32_MIN;
    }
}

// up to 8 CTAs of kGatherThreads per SM (two waves at full occupancy); beyond that the grid-stride loops
int capped_grid(long long work, int sm_count) {
    const long long cap = 8LL * (sm_count > 0 ? sm_count : 1);
    return (int)std::max<long long>(1, std::min(cap, work));
}

}  // namespace

GatherLaunch gather_launch(const GatherParams& p, int sm_count) {
    GatherLaunch l;
    l.vec = p.inside % 4 == 0 && ((uintptr_t)p.x & 15) == 0 && ((uintptr_t)p.y & 15) == 0;
    const long long rv = l.vec ? p.inside / 4 : p.inside;
    l.slices_per_tile = (int)std::max<long long>(1, std::min<long long>(kGatherThreads, kGatherTileVecs / rv));
    l.chunks = (int)((rv + kGatherTileVecs - 1) / kGatherTileVecs);
    if (l.chunks < 1 || l.slices_per_tile > 1) l.chunks = 1;
    const long long slices = p.outside * p.n;
    l.tiles = (slices + l.slices_per_tile - 1) / l.slices_per_tile * l.chunks;
    l.grid = capped_grid(l.tiles, sm_count);
    return l;
}

cudaError_t launch_gather(const GatherParams& p, int sm_count, cudaStream_t s) {
    const GatherLaunch l = gather_launch(p, sm_count);
    if (l.tiles <= 0 || p.d < 1 || p.d > kGatherMaxDims) return cudaErrorInvalidValue;
    if (l.vec)
        gather_slices_kernel<true><<<l.grid, kGatherThreads, 0, s>>>(p, l.slices_per_tile, l.chunks, l.tiles);
    else
        gather_slices_kernel<false><<<l.grid, kGatherThreads, 0, s>>>(p, l.slices_per_tile, l.chunks, l.tiles);
    ++g_launch_count;
    return cudaGetLastError();
}

int gather_elements_grid(long long count, int sm_count) {
    return capped_grid((count + kGatherThreads - 1) / kGatherThreads, sm_count);
}

cudaError_t launch_gather_elements(const GatherElementsParams& p, int sm_count, cudaStream_t s) {
    if (p.count <= 0 || p.rank < 1 || p.rank > kGatherMaxDims) return cudaErrorInvalidValue;
    gather_elements_kernel<<<gather_elements_grid(p.count, sm_count), kGatherThreads, 0, s>>>(p);
    ++g_launch_count;
    return cudaGetLastError();
}

cudaError_t launch_cast_i32_f32(const int* x, float* y, long long n, int sm_count, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    cast_i32_f32_kernel<<<capped_grid((n + kGatherThreads - 1) / kGatherThreads, sm_count), kGatherThreads, 0, s>>>(x, y, n);
    ++g_launch_count;
    return cudaGetLastError();
}

cudaError_t launch_cast_f32_i32(const float* x, int* y, long long n, int sm_count, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    cast_f32_i32_kernel<<<capped_grid((n + kGatherThreads - 1) / kGatherThreads, sm_count), kGatherThreads, 0, s>>>(x, y, n);
    ++g_launch_count;
    return cudaGetLastError();
}

}  // namespace mnnb200
