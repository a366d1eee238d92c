/* mnn_b200_gru.h -- C ABI of libmnn_b200_gru.so: the fp32 GRU of MNN (OpType_RNNSequenceGRU, which the ONNX converter emits
 * for an ONNX GRU), on the runtime and execution handles of mnn_b200.h (destroyed by mnnb200_exec_destroy, errors through
 * mnnb200_last_error).  The library links libmnn_b200.so; each library refuses the other's execution types.  A library of its
 * own, as libmnn_b200_rnn.so is, so that the other libraries' entry points and kernels stay as they are. */
#ifndef MNN_B200_GRU_H
#define MNN_B200_GRU_H
#include "mnn_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- GRU on device fp32 tensors, contiguous in the op's layouts: X [T][B][I]; per direction gateWeight Wg [I + H][2H] (rows
 *      0 .. I - 1 the x part, then the h part; columns z, then r), gateBias bg [2H], candidateWeight Wc [I + H][H],
 *      candidateBias bc [H], recurrentBias rb [3H] (Rb_z, Rb_r, Rb_h); h0 [D][B][H]; Y [T][D][B][H], Y_h [D][B][H].  Per step
 *      and batch row, the arithmetic is the reference CPU's (CPURNNSequenceGRU.cpp), every line rounded in fp32:
 *        g = [x_t, h] Wg + bg + rb[0:2H], z = sigmoid(g[0:H]), r = sigmoid(g[H:2H]);
 *        linear_before_reset 0: n_pre = [x_t, r * h] Wc + (rb[2H:3H] + bc)  (ONNX's default form);
 *        linear_before_reset 1: n_pre = ((r * (h Wc[I:] + rb[2H:3H])) + x_t Wc[0:I]) + bc  (torch.nn.GRU's form);
 *        n = tanh(n_pre), h' = ((h - n) * z) + n.
 *      Without h0, h starts at zeros.  Direction 1 reads X from t = T - 1 down and writes Y at T - 1 - s.  Y_h is each
 *      direction's last h: Y[T - 1][0] and Y[0][1], ONNX's value (the reference CPU's backward Y_h, with Y and Y_h both
 *      requested, is its zeroed or unset scratch instead).
 *      Error model: the x terms are the split-TF32 MatMul (mnnb200_matmul_create's model); each h . R row is an fp32 FMA sum in
 *      a fixed order (8 partial sums over k mod 8, combined pairwise), whatever the launch; the rest rounds once per operation
 *      in the order above; sigmoid and tanh are UnaryOp's, a few ulp.  The outputs do not depend on T or on the launch plan: a
 *      T-step execute equals T chained one-step executes bit for bit, and a D = 2 execute equals two D = 1 executes.
 *      create      linear_before_reset 0 or 1; another value: INVALID_VALUE.
 *      resize      T, B, I, H, D and whether execute gets h0 (0 or 1, else INVALID_VALUE).  Picks the plan from
 *                  (linear_before_reset, B, H, D) and the device, never from T: batch groups of at most 8 rows, a cluster of
 *                  1, 2, 4, 8 or 16 CTAs per (direction, batch group) each owning a slice of hidden units, R resident in the
 *                  cluster's shared memory when the slice fits (else read from L2 every step), the cluster checked with
 *                  cudaOccupancyMaxActiveClusters (halved until one fits).  Allocates the scratch (the projection
 *                  [T * B][D * 3H] and the repacked weights) and (re)creates the projection MatMul when T * B, I, H or D
 *                  changes; a new MatMul runs once here on zeroed scratch operands so that it allocates its packing scratch
 *                  now.  NOT_SUPPORT, with the previous plan kept: an empty dim, D outside {1, 2}, H past 4096, more than
 *                  2^31 - 1 elements in any tensor or scratch, more than 65535 batch groups, or no cluster that fits.
 *      execute     x required; params: a host array of 5 * D device pointers, each direction's Wg, bg, Wc, bc, rb in the op's
 *                  input order (none NULL); h0 as declared at resize; y or y_h may be NULL, not both.  Three launches: the
 *                  weight repack, the projection MatMul, and the recurrence of all T steps and both directions.  No
 *                  allocation, no host synchronisation and no host read of any tensor: the first execute after a resize can
 *                  be captured, and a captured graph replays with new inputs, weights included.
 *      plan        the first `count` (at most 14) of {linear_before_reset, T, B, I, H, D, cluster size, batch groups, rows
 *                  per group (the last group may have fewer), R resident (1) or streamed (0), dynamic shared memory per CTA
 *                  in bytes, scratch bytes, launches per execute (3), threads per dot product (1, 2, 4, 8)} go to fields.
 *                  NO_EXECUTION before resize, INVALID_VALUE for any other kind of execution.  Changes nothing. */
MNNB200_API mnnb200_status mnnb200_gru_create(mnnb200_runtime* rt, int linear_before_reset, mnnb200_exec** out);
MNNB200_API mnnb200_status mnnb200_gru_resize(mnnb200_exec* e, int T, int B, int I, int H, int D, int has_h0);
MNNB200_API mnnb200_status mnnb200_gru_execute(mnnb200_exec* e, const float* x, const float* const* params, const float* h0,
                                               float* y, float* y_h);
MNNB200_API mnnb200_status mnnb200_gru_plan(mnnb200_exec* e, int* fields, int count);

#ifdef __cplusplus
}
#endif
#endif /* MNN_B200_GRU_H */
