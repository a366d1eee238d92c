// interp_ops.h -- host-callable launcher of libmnn_b200_interp.so's kernels (interp_f32.cu), enqueue-only on the given stream.
#pragma once
#include <cuda_runtime.h>

namespace mnnb200 {

// fp32 Interp (CPUInterp, resize types 1-4) over `planes` NCHW-linear planes: y[p][oy][ox] = V_oy(H(p, row_j, ox)), where H is
// the horizontal interpolation of input row row_j = yi[oy * taps + j] over the columns xi[ox * taps + i] with weights
// xw[ox * taps + i], and V the vertical one over the taps rows with weights yw[oy * taps + j]; taps 1 (nearest, nearest-round: a
// gather, no weights), 2 (bilinear) or 4 (cubic).  The tables are built on the host at resize in the CPU's own expressions.
struct InterpF32Params {
    const float* x;      // [planes][ih][iw]
    float* y;            // [planes][oh][ow]
    const int* xi;       // [ow][taps] input columns, clamped
    const float* xw;     // [ow][taps] column weights (taps > 1)
    const int* yi;       // [oh][taps] input rows, clamped
    const float* yw;     // [oh][taps] row weights (taps > 1)
    int planes, ih, iw, oh, ow, taps;
};
constexpr int kInterpThreads = 256;
// the launch: `vec` the 16-byte store path (ow % 4 == 0 and y 16-byte aligned), *grid CTAs of kInterpThreads threads, *row_groups
// column groups per output row (ow / 4 with vec, else ow)
bool interp_f32_vec(const InterpF32Params& p);
void interp_f32_grid(const InterpF32Params& p, bool vec, int sm_count, int* grid, int* row_groups);
cudaError_t launch_interp_f32(const InterpF32Params& p, int sm_count, cudaStream_t s);

}  // namespace mnnb200
