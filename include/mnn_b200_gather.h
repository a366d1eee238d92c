/* mnn_b200_gather.h -- C ABI of libmnn_b200_gather.so: the gathers of fp32 models (Gather, GatherV2, GatherND, GatherElements)
 * and the int32 <-> fp32 Cast, on the runtime and execution handles of mnn_b200.h (destroyed by mnnb200_exec_destroy, errors
 * through mnnb200_last_error).  The library links libmnn_b200.so; each library refuses the other's execution types.  A library
 * of its own, as libmnn_b200_interp.so is, so that libmnn_b200.so's entry points and kernels stay as they are. */
#ifndef MNN_B200_GATHER_H
#define MNN_B200_GATHER_H
#include "mnn_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- Gathers on device tensors of 4-byte elements of any type (fp32 or int32), linear in their logical dimension order, with
 *      int32 indices.  The output equals the reference CPU's bit for bit wherever the CPU's result is defined.
 *      create      mode 0: Gather / GatherV2 (out = params[:axis] + indices + params[axis+1:]); 1: GatherND (out =
 *                  indices[:-1] + params[batch_dims + d:], d = the last dimension of indices); 2: GatherElements (out = the
 *                  shape of indices).  Anything else: INVALID_VALUE.
 *      resize      takes both shapes and `axis`: the Gather axis (negative counts from the end), GatherND's batch_dims, or the
 *                  GatherElements axis (negative counts from the end).  Index rules (the CPU's While loop, CPURaster.cpp):
 *                  negative indices are not wrapped; an index (or one component of a GatherND tuple) outside [0, the
 *                  dimension's length) writes zeros in place of its slice or element.  (Where the CPU's source offset still
 *                  falls inside the params, it reads another row there; it zero-fills only offsets outside the params.)
 *                  GatherND reads every tuple, batch dims included, against the params' dims batch_dims .. batch_dims + d
 *                  from the start of params, as the CPU does.  NOT_SUPPORT, with the previous plan kept: an empty tensor, a
 *                  rank past 8, an axis out of range, a GatherND tuple wider than params' rank minus batch_dims, batch_dims
 *                  outside [0, the indices' rank - 1), GatherElements with another rank than params' or a dimension of
 *                  indices past params' outside the axis, or an element count of params, indices or output past 2^31 - 1.
 *      execute     one launch.  Gather / GatherND: 16-byte loads and stores when the slice length is a multiple of 4 and both
 *                  params and output are 16-byte aligned, 4-byte ones otherwise.
 *      plan        the first `count` (at most 8) of {mode, path of the last execute since resize (1 16-byte, 0 4-byte, -1
 *                  none), CTAs of that launch (0 none), threads per CTA, slices per tile (0 GatherElements), outside, slices
 *                  per outside (GatherElements: output elements), slice length in elements (GatherElements: 1)} go to fields.
 *                  NO_EXECUTION before resize, INVALID_VALUE for any other kind of execution.  Changes nothing. */
MNNB200_API mnnb200_status mnnb200_gather_create(mnnb200_runtime* rt, int mode, mnnb200_exec** out);
MNNB200_API mnnb200_status mnnb200_gather_resize(mnnb200_exec* e, const int* params_dims, int params_rank, const int* indices_dims,
                                                 int indices_rank, int axis);
MNNB200_API mnnb200_status mnnb200_gather_execute(mnnb200_exec* e, const void* params, const int* indices, void* out);
MNNB200_API mnnb200_status mnnb200_gather_plan(mnnb200_exec* e, int* fields, int count);

/* ---- Cast of n elements on the runtime's stream (CPUCast's CastDataType): int32 -> fp32 rounds to nearest even; fp32 -> int32
 *      truncates toward zero, and a NaN or a value outside the int32 range gives INT32_MIN, as x86's truncating conversion
 *      does.  n = 0 launches nothing; n < 0 or a NULL tensor with n > 0: INVALID_VALUE. */
MNNB200_API mnnb200_status mnnb200_cast_i32_f32(mnnb200_runtime* rt, const int* x, float* y, long long n);
MNNB200_API mnnb200_status mnnb200_cast_f32_i32(mnnb200_runtime* rt, const float* x, int* y, long long n);

#ifdef __cplusplus
}
#endif
#endif /* MNN_B200_GATHER_H */
