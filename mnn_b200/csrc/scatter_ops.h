// scatter_ops.h -- host-callable launchers of libmnn_b200_scatter.so's kernels (scatter.cu), enqueue-only on the given stream.
#pragma once
#include <cuda_runtime.h>

namespace mnnb200 {

constexpr int kScatterMaxDims = 8;
constexpr int kScatterThreads = 256;
constexpr int kScatterDigitBits = 8;                                     // radix of the index-ordered sort
constexpr int kScatterDigits = 1 << kScatterDigitBits;
constexpr int kScatterTileItems = 8;                                     // keys per thread of one sort tile
constexpr int kScatterTile = kScatterThreads * kScatterTileItems;       // keys per sort tile
constexpr int kScatterScanThreads = 1024;

// The scatter of `n` slices of `s` 4-byte words into y of `total` words.  Update i's destination is dst_i = sum_k c_k * stride[k]
// over the `d` components of its index:
//   mode 0 (ScatterNd): c = idx[i * d .. + d);
//   mode 1 (ScatterElements): c = i's coordinate in the indices' shape idim[0..d) (istride: its element strides), with c[axis]
//   replaced by idx[i].
// dst_i lies in slot dst_i / r of the x = total / r slots when every term c_k * stride[k] lies in int32 and 0 <= dst_i < total,
// and names no slot (-1) otherwise.  s <= r, so slices of distinct slots never overlap.  Slice i is upd[i * s .. + s).
struct ScatterParams {
    const void* data;   // y's initial value (total words), or null for zeros
    const int* idx;
    const void* upd;
    void* y;
    long long total, n, s, r, x;
    int mode, d, axis;
    int stride[kScatterMaxDims];
    int idim[kScatterMaxDims];
    long long istride[kScatterMaxDims];
};

// the launch execute makes for a ScatterParams of a given reduction (-1 none, 0 ADD, 1 SUB, 2 MUL) and sort passes
struct ScatterLaunch {
    int path;      // 0 y = data only (n == 0 or s == 0), 1 last writer, 2 index-ordered fold
    int init_vec;  // bytes per access of the initial copy / zero fill: 16 (total % 4 == 0, data and y 16-byte aligned) or 4
    int vec;       // bytes per access of path 1's slice copy: 16 (s % 4 == 0, r % 4 == 0, upd and y aligned) or 4; else 0
    int grid;      // CTAs of the slice copy (path 1) or fold (path 2) kernel, of kScatterThreads each
    int tiles;     // sort tiles of kScatterTile keys (path 2)
    int launches;  // kernels and memsets execute enqueues
};
// x's bits, rounded up to whole digits: 1 - 4 passes
int scatter_sort_passes(long long x);
ScatterLaunch scatter_launch(const ScatterParams& p, int reduction, int passes, int sm_count);

// Scratch of one scatter: owner[x] (path 1), keys / vals [2][n] and hist[kScatterDigits * (tiles + 1)] (path 2: the per-tile
// digit counts, then the kScatterDigits row totals).
struct ScatterScratch {
    int* owner;
    unsigned* keys[2];
    unsigned* vals[2];
    unsigned* hist;
};
cudaError_t launch_scatter(const ScatterParams& p, int reduction, int passes, const ScatterScratch& w, int sm_count,
                           cudaStream_t s);

}  // namespace mnnb200
