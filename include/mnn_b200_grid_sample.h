/* mnn_b200_grid_sample.h -- C ABI of libmnn_b200_grid_sample.so: the fp32 GridSample execution (2-D and 3-D nearest, bilinear
 * and trilinear sampling of fp32 models: flow warps, spatial transformers, deformable / BEV sampling, 3D-LUT lookups) on the
 * runtime and execution handles of mnn_b200.h (destroyed by mnnb200_exec_destroy, errors through mnnb200_last_error).  The
 * library links libmnn_b200.so; each library refuses the other's execution types.  A library of its own, as
 * libmnn_b200_interp.so is, so that the other libraries' entry points and kernels stay as they are. */
#ifndef MNN_B200_GRID_SAMPLE_H
#define MNN_B200_GRID_SAMPLE_H
#include "mnn_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- GridSample of fp32 models: CPUGridSample on NCHW-linear device fp32 tensors.  x [n][c][ih][iw] with grid
 *      [n][oh][ow][2] (x, y) and y [n][c][oh][ow] (rank 4), or x [n][c][id][ih][iw] with grid [n][od][oh][ow][3] (x, y, z) and
 *      y [n][c][od][oh][ow] (rank 5).  The output equals the x86 CPU backend's on an AVX-512 host bit for bit: its coordinate
 *      expressions, floor / ceil taps converted as x86 converts (NaN, +-Inf and |c| >= 2^31 give INT_MIN), and its fused and
 *      unfused products and sums.
 *      create      mode 0 bilinear (trilinear for rank 5), 1 nearest (halves round up); padding 0 zeros (an outside tap reads 0),
 *                  1 border (the tap is clamped), 2 reflection, which samples as border, as the CPU's does (unlike PyTorch's
 *                  and ONNX's reflection); align_corners as the op's alignCorners.  NOT_SUPPORT for a mode outside 0-1 or a
 *                  padding outside 0-2 (the backward form is not an execution of this library).
 *      resize      rank (4 or 5), n, c, in_dims = the rank - 2 input dims (D, H, W or H, W), out_dims = the output's (those of
 *                  the grid).  Fixes the coordinate constants and the channel groups: shapes with few output pixels split
 *                  their channels into groups so that the launch fills the device.  NOT_SUPPORT, with the previous plan kept:
 *                  a rank other than 4 and 5, an empty tensor, an index of x, grid or y past 31 bits.  INVALID_VALUE for NULL
 *                  dims.
 *      execute     one launch.  x, grid and y may have any 4-byte alignment; a rank-4 grid is read as float2 when it is
 *                  8-byte aligned, as scalars otherwise.
 *      plan        the first `count` (at most 7) of {rank, taps (1 nearest, 4 bilinear, 8 trilinear), channel groups,
 *                  channels per group, CTAs, threads per CTA, grid-read path of the last execute since resize (1 float2, 0
 *                  scalar, -1 none)} go to fields.  NO_EXECUTION before resize, INVALID_VALUE for any other kind of execution.
 *                  Changes nothing. */
MNNB200_API mnnb200_status mnnb200_grid_sample_f32_create(mnnb200_runtime* rt, int mode, int padding, int align_corners,
                                                          mnnb200_exec** out);
MNNB200_API mnnb200_status mnnb200_grid_sample_f32_resize(mnnb200_exec* e, int rank, int n, int c, const int* in_dims,
                                                          const int* out_dims);
MNNB200_API mnnb200_status mnnb200_grid_sample_f32_execute(mnnb200_exec* e, const float* x, const float* grid, float* y);
MNNB200_API mnnb200_status mnnb200_grid_sample_f32_plan(mnnb200_exec* e, int* fields, int count);

#ifdef __cplusplus
}
#endif
#endif /* MNN_B200_GRID_SAMPLE_H */
