/* mnn_b200_deconv.h -- C ABI of libmnn_b200_deconv.so: the float Deconvolution executions (transposed convolutions of fp32 models)
 * on the runtime and execution handles of mnn_b200.h (destroyed by mnnb200_exec_destroy, errors through mnnb200_last_error).
 * The library links libmnn_b200.so; each library refuses the other's execution types.  A library of its own, as
 * libmnn_b200_llm.so is, so that libmnn_b200.so's entry points and kernels stay as they are. */
#ifndef MNN_B200_DECONV_H
#define MNN_B200_DECONV_H
#include "mnn_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- Float Deconvolution (transposed convolution) of fp32 models: CPUDeconvolution and CPUDeconvolutionDepthwise on
 *      NCHW-linear device fp32 tensors.  y[n][oc][oy][ox] = bias[oc] + sum x[n][ic][iy][ix] * w[ic][oc][ky][kx] over every
 *      (ic, ky, kx) with oy + pad_h = iy * stride_h + ky * dilate_h and ox + pad_w = ix * stride_w + kx * dilate_w, then ReLU /
 *      ReLU6 as for conv_f32.  desc->pad_h / pad_w are the begin pads (ConvolutionCommon::convolutionTransposePad).
 *      deconv_f32: group == 1, strides <= 16 (NOT_SUPPORT otherwise).  create takes host weights [ic][oc][kh][kw] and bias [oc]
 *                  (may be NULL) and splits them once per phase into two TF32 halves; execute runs one split-TF32 wgmma launch
 *                  over the stride_h * stride_w phases (output pixels with the same (oy + pad_h) % stride_h and
 *                  (ox + pad_w) % stride_w), each a stride-1 implicit GEMM over the input: error near fp32's, as conv_f32.
 *                  resize takes n, ih, iw and *oh / *ow: > 0 the output size (MNN's shape inference: pads [t, l, b, r], outPads,
 *                  SAME, an output-shape input), else (ih - 1) * stride_h + dilate_h * (kh - 1) + 1 - 2 * pad_h (and the same in
 *                  w), written back.  NOT_SUPPORT, with the previous plan kept: an empty tensor, an output size past
 *                  (ih - 1) * stride_h + dilate_h * (kh - 1) + stride_h - pad_h (rows no stride or out-pad produces), an index past
 *                  32 bits.  set_pad sets the begin pads of a deconv_f32 or dwdeconv_f32 execution, before resize.
 *      dwdeconv_f32: group == ic == oc, weights [c][kh][kw], the same sizes and refusals (no stride limit).
 *      deconv_f32_plan: the first `count` (at most 7) of {bn (tile width 32 / 64 / 128), n_chunks, phases (stride_h * stride_w),
 *                  m_tiles (128-pixel M tiles of the largest phase), num_kb (32-wide K blocks of the deepest phase), stages (K
 *                  blocks the bn-wide kernel's ring holds), taps (of the phase with the most)} go to fields.  NO_EXECUTION before
 *                  resize, INVALID_VALUE for any other kind of execution.  Changes nothing. */
MNNB200_API mnnb200_status mnnb200_deconv_f32_create(mnnb200_runtime* rt, const mnnb200_conv_desc* desc, const float* weight,
                                                     const float* bias, int relu6, mnnb200_exec** out);
MNNB200_API mnnb200_status mnnb200_deconv_f32_set_pad(mnnb200_exec* e, int pad_h, int pad_w);
MNNB200_API mnnb200_status mnnb200_deconv_f32_resize(mnnb200_exec* e, int n, int ih, int iw, int* oh, int* ow);
MNNB200_API mnnb200_status mnnb200_deconv_f32_execute(mnnb200_exec* e, const float* x_nchw, float* y_nchw);
MNNB200_API mnnb200_status mnnb200_deconv_f32_plan(mnnb200_exec* e, int* fields, int count);
MNNB200_API mnnb200_status mnnb200_dwdeconv_f32_create(mnnb200_runtime* rt, const mnnb200_conv_desc* desc, const float* weight,
                                                       const float* bias, int relu6, mnnb200_exec** out);
MNNB200_API mnnb200_status mnnb200_dwdeconv_f32_resize(mnnb200_exec* e, int n, int ih, int iw, int* oh, int* ow);
MNNB200_API mnnb200_status mnnb200_dwdeconv_f32_execute(mnnb200_exec* e, const float* x_nchw, float* y_nchw);

#ifdef __cplusplus
}
#endif
#endif /* MNN_B200_DECONV_H */
