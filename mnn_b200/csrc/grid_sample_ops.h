// grid_sample_ops.h -- host-callable launcher of libmnn_b200_grid_sample.so's kernel (grid_sample_f32.cu), enqueue-only on the
// given stream.
#pragma once
#include <cuda_runtime.h>

namespace mnnb200 {

// fp32 GridSample (CPUGridSample) on NCHW-linear tensors: x [n][c][id][ih][iw], grid [n][od][oh][ow][rank - 2] (x, y[, z]),
// y [n][c][od][oh][ow]; a 2-D sample has id = od = 1.  The output pixels of one batch, `pixels` = od * oh * ow, are dealt to
// threads; a thread reads its pixel's grid entry once, computes its taps and weights once and loops over `cper` channels of one
// of `cgroups` channel groups.
struct GridSampleF32Params {
    const float* x;
    const float* grid;
    float* y;
    int n, c, id, ih, iw, pixels;
    int cgroups, cper;
    // the coordinate of one axis: 2-D 0.5 * fma(1 + g, in - a, -b) (a = 1, b = 0 with alignCorners, else a = 0, b = 1); 3-D
    // k * g + k0 with k = 0.5 (in - a) and k0 = 0.5 (in - a - b), both computed at resize in the CPU's float expressions
    float in_a[3], b;         // 2-D: (float)in - a per axis (w, h), and b
    float k[3], k0[3];        // 3-D: per axis (w, h, d)
};
constexpr int kGridSampleThreads = 256;
// the launch: *grid CTAs of kGridSampleThreads threads over n * cgroups * pixels work items
int grid_sample_f32_grid(const GridSampleF32Params& p, int sm_count);
// rank 4 or 5, nearest (else bilinear / trilinear), zeros (else clamp); vec2: read the 2-D grid as float2 (8-byte aligned grid)
cudaError_t launch_grid_sample_f32(const GridSampleF32Params& p, int rank, bool nearest, bool zeros, bool vec2, int sm_count,
                                   cudaStream_t s);

}  // namespace mnnb200
