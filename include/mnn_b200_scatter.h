/* mnn_b200_scatter.h -- C ABI of libmnn_b200_scatter.so: ScatterNd and ScatterElements of fp32 models, on the runtime and
 * execution handles of mnn_b200.h (destroyed by mnnb200_exec_destroy, errors through mnnb200_last_error).  The library links
 * libmnn_b200.so; each library refuses the other's execution types.  A library of its own, as libmnn_b200_gather.so is, so
 * that the other libraries' entry points and kernels stay as they are. */
#ifndef MNN_B200_SCATTER_H
#define MNN_B200_SCATTER_H
#include "mnn_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- Scatters on device tensors of 4-byte elements (fp32, or int32 without a reduction), linear in their logical dimension
 *      order, with int32 indices.  The output equals the reference CPU's sequential loop (GeometryScatter.cpp, CPURaster.cpp)
 *      bit for bit wherever the CPU's result is defined: y starts as data (or zeros), then update i, in index order, writes
 *      (no reduction: the last writer wins) or folds (y = y op update, plain fp32) its slice at its destination.  A NaN that
 *      an ADD / SUB / MUL produces or passes on is a NaN on both, but its payload follows the GPU's arithmetic.
 *      create      mode 0: ScatterNd(indices, updates, shape[, data]) (out = the shape input; with_data 0 zero-fills it);
 *                  1: ScatterElements(data, indices, updates[, axis]) (out = data's shape; with_data must be 1).
 *                  reduction: < 0 none, 0 ADD, 1 SUB, 2 MUL (BinaryOpOperation's codes).  Another mode or with_data, or
 *                  ScatterElements without data: INVALID_VALUE; another reduction (MIN, MAX, ...: the CPU drops the updates
 *                  then): NOT_SUPPORT.
 *      resize      takes the output's, the indices' and the updates' shapes, the ScatterElements axis (negative counts from
 *                  the end; ignored by ScatterNd) and whether the tensors are int32.  ScatterNd: N = the product of the
 *                  indices' dims but the last, D = the last, S = the product of the updates' dims from index D on (as the
 *                  CPU computes it: the slice length only when the indices' rank is D + 1), and destination
 *                  sum_d idx[i][d] * (the output's stride of dim d).  ScatterElements: N = the indices' elements, S = 1,
 *                  destination = the element's coordinate in the indices' shape with the axis component replaced by its
 *                  index, against the output's strides; updates are read flat.  R = the output's stride of the last
 *                  index component (1 for ScatterElements).  A destination outside [0, out elements), or with a term
 *                  index * stride outside int32, is skipped.  The CPU skips the first without a reduction and has no bounds
 *                  check with one (its result is undefined there); for the second its MUL / SUM give neither exact nor
 *                  int32-wrapped sums, so the bit-exact claim covers indices whose terms fit in int32.
 *                  NOT_SUPPORT, with the previous plan kept: an empty output, a rank past 8 (or an empty indices rank), D
 *                  outside [1, the output's rank], ScatterElements indices of another rank than the output's or an axis out
 *                  of range, S > R, fewer than N * S updates, int32 tensors with a reduction, or more than 2^31 - 1
 *                  elements in any tensor.  N = 0 or S = 0 leaves y = data.
 *      execute     no host synchronisation, no index read on the host: a captured graph replays with new indices.  Without
 *                  a reduction: an owner pass (atomicMax of the update index per destination) and a copy by each
 *                  destination's last update.  ADD / SUB / MUL: a stable radix sort of the updates by destination and a
 *                  fold of each destination's updates in index order.  data may be NULL only when created without data.
 *      plan        the first `count` (at most 12) of {mode, reduction, N, S, R, X = out elements / R, path of the last
 *                  execute since resize (-1 none, 0 y = data only, 1 last writer, 2 index-ordered fold), sort passes (path
 *                  2: 1-4, from X's bits; else 0), launches of that execute (kernels and memsets), bytes per access of its
 *                  slice copy (16, 4; 0 none), of its initial copy (16, 4), CTAs of its slice copy or fold kernel} go to
 *                  fields.  NO_EXECUTION before resize, INVALID_VALUE for any other kind of execution.  Changes nothing. */
MNNB200_API mnnb200_status mnnb200_scatter_create(mnnb200_runtime* rt, int mode, int reduction, int with_data, mnnb200_exec** out);
MNNB200_API mnnb200_status mnnb200_scatter_resize(mnnb200_exec* e, const int* out_dims, int out_rank, const int* idx_dims,
                                                  int idx_rank, const int* upd_dims, int upd_rank, int axis, int is_int32);
MNNB200_API mnnb200_status mnnb200_scatter_execute(mnnb200_exec* e, const void* data, const int* indices, const void* updates,
                                                   void* out);
MNNB200_API mnnb200_status mnnb200_scatter_plan(mnnb200_exec* e, int* fields, int count);

#ifdef __cplusplus
}
#endif
#endif /* MNN_B200_SCATTER_H */
