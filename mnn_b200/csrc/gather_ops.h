// gather_ops.h -- host-callable launchers of libmnn_b200_gather.so's kernels (gather.cu), enqueue-only on the given stream.
#pragma once
#include <cuda_runtime.h>

namespace mnnb200 {

constexpr int kGatherMaxDims = 8;
constexpr int kGatherThreads = 256;
constexpr int kGatherTileVecs = 4096;   // vectors (16 or 4 bytes) one CTA copies per tile

// Slice gather (Gather / GatherV2 / GatherND): y = [outside][n][inside] of 4-byte elements.  Slice (o, j) reads its index tuple
// t = idx[o * idx_outer + j * d .. + d) once; when every t[k] lies in [0, dim[k]) it copies the `inside` elements at
// x + o * x_outer + sum_k t[k] * stride[k], otherwise it writes zeros.  Gather is d = 1 with x_outer = dim[0] * inside and
// idx_outer = 0; GatherND over batch dims is x_outer = the batch's element count and idx_outer = n * d.
struct GatherParams {
    const void* x;
    const int* idx;
    void* y;
    long long outside, n, inside;
    long long x_outer, idx_outer;
    int d;
    int dim[kGatherMaxDims];
    long long stride[kGatherMaxDims];
};
// the launch: `vec` the 16-byte path (inside % 4 == 0 and x, y 16-byte aligned), *slices_per_tile slices of one tile (1 when a
// slice is longer than a tile: it is then split into *chunks tiles), *grid CTAs of kGatherThreads threads
struct GatherLaunch {
    bool vec;
    int slices_per_tile, chunks, grid;
    long long tiles;
};
GatherLaunch gather_launch(const GatherParams& p, int sm_count);
cudaError_t launch_gather(const GatherParams& p, int sm_count, cudaStream_t s);

// Element gather (GatherElements): y has the shape odim[0..rank) of the indices; y[i] = x[sum_k c[k] * xstride[k]] where c is
// i's coordinate with c[axis] replaced by idx[i]; zero when idx[i] lies outside [0, axis_len).
struct GatherElementsParams {
    const void* x;
    const int* idx;
    void* y;
    long long count;
    int rank, axis, axis_len;
    int odim[kGatherMaxDims];
    long long xstride[kGatherMaxDims];
};
int gather_elements_grid(long long count, int sm_count);
cudaError_t launch_gather_elements(const GatherElementsParams& p, int sm_count, cudaStream_t s);

// Cast (CPUCast's CastDataType): int32 -> fp32 rounds to nearest; fp32 -> int32 truncates, and a NaN or a value outside the
// int32 range gives INT32_MIN, as x86's cvttss2si / cvttps2dq do.
cudaError_t launch_cast_i32_f32(const int* x, float* y, long long n, int sm_count, cudaStream_t s);
cudaError_t launch_cast_f32_i32(const float* x, int* y, long long n, int sm_count, cudaStream_t s);

}  // namespace mnnb200
