/* mnn_b200_interp.h -- C ABI of libmnn_b200_interp.so: the fp32 Interp execution (nearest, bilinear and cubic resampling of
 * fp32 models; MNN's Resize op reaches it as a bilinear Interp) on the runtime and execution handles of mnn_b200.h (destroyed by
 * mnnb200_exec_destroy, errors through mnnb200_last_error).  The library links libmnn_b200.so; each library refuses the other's
 * execution types.  A library of its own, as libmnn_b200_llm.so and libmnn_b200_deconv.so are, so that libmnn_b200.so's entry
 * points and kernels stay as they are. */
#ifndef MNN_B200_INTERP_H
#define MNN_B200_INTERP_H
#include "mnn_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- Interp of fp32 models: CPUInterp on NCHW-linear device fp32 tensors of `planes` (batch * channels) planes.
 *      create takes the op's Interp fields as CPUInterpCreator reads them: resize_type (1 nearest, 2 bilinear, 3 cubic, 4
 *                  nearest-round) and the coordinate transform src = dst * scale + offset per axis, as MNN's geometry stage has
 *                  already computed it from the op's ctm / alignCorners / halfPixelCenters / output size.  Nothing is checked
 *                  but the handles: resize refuses what it cannot run.
 *      resize      takes planes, ih, iw, oh, ow, builds every per-column and per-row index and weight on the host in the CPU's
 *                  expressions and uploads them.  NOT_SUPPORT, with the previous plan kept: resize_type outside 1-4, a
 *                  non-finite scale or offset, an empty tensor, an index of x or y past 31 bits.
 *      execute     one launch; the output equals the CPU's bit for bit.  16-byte stores when ow % 4 == 0 and y is 16-byte
 *                  aligned, scalar stores otherwise (x may have any 4-byte alignment).
 *      plan        the first `count` (at most 7) of {taps (1 nearest / nearest-round, 2 bilinear, 4 cubic), path of the last
 *                  execute since resize (1 16-byte stores, 0 scalar, -1 none), CTAs of that launch (0 none), threads per CTA,
 *                  column groups per output row of that launch (0 none), column table entries (ow * taps), row table entries
 *                  (oh * taps)} go to fields.  NO_EXECUTION before resize, INVALID_VALUE for any other kind of execution.
 *                  Changes nothing. */
MNNB200_API mnnb200_status mnnb200_interp_f32_create(mnnb200_runtime* rt, int resize_type, float width_scale, float height_scale,
                                                     float width_offset, float height_offset, mnnb200_exec** out);
MNNB200_API mnnb200_status mnnb200_interp_f32_resize(mnnb200_exec* e, int planes, int ih, int iw, int oh, int ow);
MNNB200_API mnnb200_status mnnb200_interp_f32_execute(mnnb200_exec* e, const float* x_nchw, float* y_nchw);
MNNB200_API mnnb200_status mnnb200_interp_f32_plan(mnnb200_exec* e, int* fields, int count);

#ifdef __cplusplus
}
#endif
#endif /* MNN_B200_INTERP_H */
