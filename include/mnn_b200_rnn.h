/* mnn_b200_rnn.h -- C ABI of libmnn_b200_rnn.so: the fp32 LSTM and RNN ops of ONNX models (OpType_LSTM / OpType_RNN), on the
 * runtime and execution handles of mnn_b200.h (destroyed by mnnb200_exec_destroy, errors through mnnb200_last_error).  The
 * library links libmnn_b200.so; each library refuses the other's execution types.  A library of its own, as
 * libmnn_b200_scatter.so is, so that the other libraries' entry points and kernels stay as they are. */
#ifndef MNN_B200_RNN_H
#define MNN_B200_RNN_H
#include "mnn_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- LSTM / RNN on device fp32 tensors, contiguous in the ONNX layouts: X [T][B][I], W [D][G*H][I], R [D][G*H][H], bias
 *      [D][G*H] (ONNX's Wb + Rb, summed), h0 / c0 [D][B][H]; Y [T][D][B][H], Y_h / Y_c [D][B][H].  G = 4 gate rows for LSTM in
 *      ONNX order i, o, f, c; G = 1 for RNN.  The arithmetic is the reference CPU's lowering (GeometryLSTM.cpp,
 *      _ComputeLSTMOnnx): Gate = X W^T + bias for all T * B rows, then per step z = Gate_t + h_prev R^T and
 *        LSTM: i = sigmoid(z_i), g = tanh(z_c), f = sigmoid(z_f), o = sigmoid(z_o), c = i * g + f * c_prev, h = tanh(c) * o;
 *        RNN: h = tanh(z).
 *      The activations are always sigmoid / tanh / tanh (the converter drops ONNX's activations, clip and input_forget).
 *      Without h0 the first step has no h_prev R^T term, without c0 no f * c_prev term (c0 absent with h0 given: zeros, as
 *      ONNX defines it).  Direction 1 reads X from t = T - 1 down and writes Y at T - 1 - s; Y_h is the last step's h of each
 *      direction, Y_c its c.
 *      Error model: the projection is the split-TF32 MatMul (mnnb200_matmul_create's model); each gate's h_prev . R row is an
 *      fp32 FMA sum in a fixed order (8 partial sums over k mod 8, combined pairwise), whatever the launch; the cell update
 *      rounds once per operation in the reference's order; sigmoid and tanh are UnaryOp's, a few ulp.  The outputs do not
 *      depend on T or on the launch plan: a T-step execute equals T chained one-step executes bit for bit, and a D = 2
 *      execute equals two D = 1 executes (direction 1 on X reversed).
 *      create      cell 0 LSTM, 1 RNN; another cell: INVALID_VALUE.
 *      resize      T, B, I, H, D and whether execute gets h0 / c0 (has_c0 must be 0 for RNN: INVALID_VALUE).  Picks the plan
 *                  from (cell, B, H, D) and the device, never from T: batch groups of at most 8 rows, a cluster of 1, 2, 4, 8
 *                  or 16 CTAs per (direction, batch group) each owning a slice of hidden units, R resident in the cluster's
 *                  shared memory when the slice fits (else read from L2 every step), the cluster checked with
 *                  cudaOccupancyMaxActiveClusters (halved until one fits).  Allocates the Gate scratch
 *                  ([T * B][D * G * H]) and (re)creates the projection MatMul when T * B, I, H or D changes; a new MatMul
 *                  runs once here on zeroed scratch operands so that it allocates its packing scratch now.
 *                  NOT_SUPPORT, with the previous plan kept: an empty dim, D outside {1, 2}, H past 4096, more than 2^31 - 1
 *                  elements in X, W, R, Y or the Gate scratch, more than 65535 batch groups, or no cluster that fits.
 *      execute     x, w, r and y required; bias may be NULL (zeros); h0 / c0 as declared at resize; y_h and y_c may be
 *                  NULL (y_c ignored for RNN).  Two launches: the projection MatMul, then the recurrence of all T steps and
 *                  both directions in one launch.  No allocation, no host synchronisation and no host read of any input: the
 *                  first execute after a resize can be captured, and a captured graph replays with new inputs, weights
 *                  included.
 *      plan        the first `count` (at most 14) of {cell, T, B, I, H, D, cluster size, batch groups, rows per group
 *                  (the last group may have fewer), R resident (1) or streamed (0), dynamic shared memory per CTA in bytes,
 *                  Gate scratch bytes, recurrence launches per execute (1), threads per dot product (1, 2, 4, 8)} go to
 *                  fields.  NO_EXECUTION before resize, INVALID_VALUE for any other kind of execution.  Changes nothing. */
MNNB200_API mnnb200_status mnnb200_rnn_create(mnnb200_runtime* rt, int cell, mnnb200_exec** out);
MNNB200_API mnnb200_status mnnb200_rnn_resize(mnnb200_exec* e, int T, int B, int I, int H, int D, int has_h0, int has_c0);
MNNB200_API mnnb200_status mnnb200_rnn_execute(mnnb200_exec* e, const float* x, const float* w, const float* r, const float* bias,
                                               const float* h0, const float* c0, float* y, float* y_h, float* y_c);
MNNB200_API mnnb200_status mnnb200_rnn_plan(mnnb200_exec* e, int* fields, int count);

#ifdef __cplusplus
}
#endif
#endif /* MNN_B200_RNN_H */
