/*
 * mnn_b200.h -- C ABI of the H100-native compute library behind MNN's CUDA backend surface.
 *
 * This is the drop-in boundary for the int8 hot path.  The MNN plugin (mnn_b200/csrc/plugin, a
 * RuntimeCreator/Runtime/Backend/Execution implementation registered under MNN_FORWARD_CUDA) and any
 * other FFI host (ctypes in mnn_b200/_capi.py) call exactly these entry points: plain pointers and
 * sizes, no C++ or torch types.  Each entry point cites the reference interface it replaces
 * (paths relative to the alibaba/MNN tree).
 *
 * Conventions
 *  - Every function returns an mnnb200_status (0 = MNNB200_OK); values mirror MNN::ErrorCode
 *    (include/MNN/ErrorCode.hpp): NO_ERROR=0, OUT_OF_MEMORY=1, NOT_SUPPORT=2, COMPUTE_SIZE_ERROR=3,
 *    NO_EXECUTION=4, INVALID_VALUE=5; 100 = CUDA runtime failure (mnnb200_last_error() has the text).
 *  - Device activation layout (private to the backend, like CUDABackend::realSize,
 *    source/backend/cuda/core/CUDABackend.cpp:245-263): int8 NHWC with C padded to 16
 *    ("NHWC16", INT8_PACK_NUMBER); fp32 tensors at the graph boundary are plain NCHW.
 *  - execute() calls only ENQUEUE work on the runtime's stream (Execution::onExecute contract,
 *    source/core/Execution.hpp:24-135); mnnb200_runtime_sync() is Backend::onSync.
 *  - There is no CPU fallback: without a CUDA device every create() fails with status 100.
 */
#ifndef MNN_B200_H
#define MNN_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MNNB200_API __attribute__((visibility("default")))

typedef int mnnb200_status;
enum { MNNB200_OK = 0, MNNB200_OUT_OF_MEMORY = 1, MNNB200_NOT_SUPPORT = 2, MNNB200_COMPUTE_SIZE_ERROR = 3,
       MNNB200_NO_EXECUTION = 4, MNNB200_INVALID_VALUE = 5, MNNB200_CUDA_ERROR = 100 };

typedef struct mnnb200_runtime mnnb200_runtime; /* CUDARuntime + CUDARuntimeWrapper: device, stream, pools */
typedef struct mnnb200_exec mnnb200_exec;       /* one MNN::Execution (weights resident in HBM)          */

MNNB200_API const char* mnnb200_last_error(void);
MNNB200_API int mnnb200_abi_version(void);

/* ---- Runtime: replaces CUDARuntimeCreator::onCreate + CUDARuntime (source/backend/cuda/Register.cpp:12-38,
 *      core/runtime/CUDARuntime.cpp:29-182).  device_id = MNNDeviceContext::deviceId.
 *      stream == NULL: the runtime creates its own non-blocking stream (one per GPU); otherwise it adopts
 *      the caller's cudaStream_t (e.g. torch's current stream) and does not destroy it. */
MNNB200_API mnnb200_status mnnb200_runtime_create(int device_id, void* stream, mnnb200_runtime** out);
MNNB200_API void mnnb200_runtime_destroy(mnnb200_runtime* rt);
MNNB200_API void* mnnb200_runtime_stream(mnnb200_runtime* rt);
MNNB200_API mnnb200_status mnnb200_runtime_sync(mnnb200_runtime* rt);           /* Backend::onSync */
MNNB200_API mnnb200_status mnnb200_runtime_info(mnnb200_runtime* rt, int* sm_count, int* cc_major, int* cc_minor,
                                                size_t* total_mem);
/* Backend::onAcquire / CUDARuntime::alloc,free,memcpy (core/CUDABackend.cpp:209-243, CUDARuntime.cpp:139-182) */
MNNB200_API mnnb200_status mnnb200_alloc(mnnb200_runtime* rt, size_t bytes, void** dev_ptr);
MNNB200_API mnnb200_status mnnb200_free(mnnb200_runtime* rt, void* dev_ptr);
MNNB200_API mnnb200_status mnnb200_memcpy_h2d(mnnb200_runtime* rt, void* dst_dev, const void* src_host, size_t bytes);
MNNB200_API mnnb200_status mnnb200_memcpy_d2h(mnnb200_runtime* rt, void* dst_host, const void* src_dev, size_t bytes);
MNNB200_API size_t mnnb200_nhwc16_bytes(int n, int c, int h, int w); /* CUDABackend::realSize for int8 */
/* number of kernels this library has launched since load (bench.py's gpu_launches) */
MNNB200_API unsigned long long mnnb200_launch_count(void);

/* ---- Whole-forward CUDA graph: Backend::onExecuteBegin / onExecuteEnd (source/core/Backend.hpp:129-137; the reference CUDA
 *      backend's are empty, core/CUDABackend.cpp:300-310) bracket every Execution::onExecute of one forward.  begin_capture puts
 *      the runtime's stream into capture (thread-local mode): execute() calls between begin and end are RECORDED, not run;
 *      end_capture instantiates the recorded forward; launch enqueues it (one host call per forward instead of one per op).
 *      A graph is only valid while the executions, their shapes and the tensors' device addresses it was captured with are. */
typedef struct mnnb200_graph mnnb200_graph;
MNNB200_API mnnb200_status mnnb200_graph_begin_capture(mnnb200_runtime* rt);
MNNB200_API mnnb200_status mnnb200_graph_end_capture(mnnb200_runtime* rt, mnnb200_graph** out);
MNNB200_API mnnb200_status mnnb200_graph_launch(mnnb200_runtime* rt, mnnb200_graph* g);
MNNB200_API void mnnb200_graph_destroy(mnnb200_graph* g);
/* ---- Host staging for Backend::onCopyBuffer (core/CUDABackend.cpp:431-535 uses synchronous cudaMemcpy from pageable memory):
 *      host_register pins a caller-owned host range in place so cudaMemcpyAsync reads it by DMA at PCIe speed (idempotent per
 *      range; NOT_SUPPORT if the driver refuses); alloc_host / free_host = pinned scratch owned by the backend. */
MNNB200_API mnnb200_status mnnb200_host_register(mnnb200_runtime* rt, void* host_ptr, size_t bytes);
MNNB200_API mnnb200_status mnnb200_host_unregister(mnnb200_runtime* rt, void* host_ptr);
MNNB200_API mnnb200_status mnnb200_alloc_host(mnnb200_runtime* rt, size_t bytes, void** host_ptr);
MNNB200_API mnnb200_status mnnb200_free_host(mnnb200_runtime* rt, void* host_ptr);
/* ---- GPU time of the last forward: Runtime::onGetLastGpuTimeMs (source/core/Backend.hpp:400-402).  mark_begin / mark_end record
 *      CUDA events on the runtime's stream; last_gpu_ms waits for the end event and returns the elapsed device time (-1 if none). */
MNNB200_API mnnb200_status mnnb200_runtime_mark_begin(mnnb200_runtime* rt);
MNNB200_API mnnb200_status mnnb200_runtime_mark_end(mnnb200_runtime* rt);
MNNB200_API float mnnb200_runtime_last_gpu_ms(mnnb200_runtime* rt);

/* ---- Boundary casts: replace FloatToInt8Execution / Int8ToFloatExecution and the quant-aware
 *      CUDABackend::onCopyBuffer (execution/int8/FloatToInt8Execution.cu:19-130, Int8ToFloatExecution.cu:19-70,
 *      core/CUDABackend.cpp:537-589), with the CPU backend's arithmetic (CPUCast.cpp:17-60).
 *      x/y fp32 are NCHW, int8 are NHWC16; scale is the tensor's quant scale. */
MNNB200_API mnnb200_status mnnb200_float_to_int8(mnnb200_runtime* rt, const float* x_nchw, int n, int c, int h, int w,
                                                 float scale, float zero, int min_v, int max_v, int8_t* y_nhwc16);
MNNB200_API mnnb200_status mnnb200_int8_to_float(mnnb200_runtime* rt, const int8_t* x_nhwc16, int n, int c, int h,
                                                 int w, float scale, float zero, float* y_nchw);
/* layout-only copies between logical NCHW int8 and device NHWC16 (CUDABackend::onCopyBuffer int8<->int8) */
MNNB200_API mnnb200_status mnnb200_pack_nchw_int8(mnnb200_runtime* rt, const int8_t* x_nchw, int n, int c, int h, int w,
                                                  int8_t* y_nhwc16);
MNNB200_API mnnb200_status mnnb200_unpack_nchw_int8(mnnb200_runtime* rt, const int8_t* x_nhwc16, int n, int c, int h,
                                                    int w, int8_t* y_nchw);

/* ---- Int8 Conv2D: replaces ConvInt8CutlassExecution {Resource, onResize, onExecute}
 *      (execution/int8/ConvInt8CutlassExecution.cu:146-264, 296-379, 381-445) with the CPU backend's arithmetic
 *      (CPUConvolution.cpp:144-201, compute/ConvInt8TiledExecutor.cpp:2218-2245, GemmInt8_VNNI.cpp:27-39). */
typedef struct mnnb200_conv_desc {
    int32_t ic, oc, kh, kw, stride_h, stride_w, pad_h, pad_w, dilate_h, dilate_w, group, relu;
} mnnb200_conv_desc;

/* create = Resource ctor: weights [oc][ic/group][kh][kw] int8 (the output of ConvolutionCommon::getConvInt8Parameters,
 * source/core/ConvolutionCommon.cpp:881-942) are packed and uploaded once.
 * modern form: wscale = quanParameter.alpha (per-channel weight scale), bias = float bias (may be NULL). */
MNNB200_API mnnb200_status mnnb200_conv_int8_create(mnnb200_runtime* rt, const mnnb200_conv_desc* desc,
                                                    const int8_t* weight, const float* wscale, const float* bias,
                                                    mnnb200_exec** out);
/* legacy form (OpType_ConvInt8 with symmetricQuan{bias:int32, scale}): scale already holds s_in*w/s_out. */
MNNB200_API mnnb200_status mnnb200_conv_int8_create_legacy(mnnb200_runtime* rt, const mnnb200_conv_desc* desc,
                                                           const int8_t* weight, const float* scale,
                                                           const int32_t* bias_i32, mnnb200_exec** out);
/* resize = onResize: fold the tensors' quant info {scale, zero, min, max} (TensorUtils::getQuantInfo) into the
 * epilogue constants and pick launch parameters for this shape.  *oh/*ow: in/out -- a value > 0 on entry is the
 * output size decided by MNN's shape inference (pad_h/pad_w are then the BEGIN pads, e.g. TF-SAME); 0 on entry =
 * compute it from symmetric pads.  Written back on return. */
MNNB200_API mnnb200_status mnnb200_conv_int8_resize(mnnb200_exec* e, int n, int ih, int iw, float in_scale,
                                                    int in_zero, float out_scale, int out_zero, int clamp_min,
                                                    int clamp_max, int* oh, int* ow);
/* begin pads resolved at resize time (ConvolutionCommon::convolutionPad, source/core/ConvolutionCommon.cpp:945-975: SAME /
 * VALID / explicit pads depend on the tensors' shapes); call before *_resize.  Works on conv, dwconv and Winograd executions. */
MNNB200_API mnnb200_status mnnb200_conv_int8_set_pad(mnnb200_exec* e, int pad_h, int pad_w);
/* execute = onExecute: x [n][ih][iw][p16(ic)] -> y [n][oh][ow][p16(oc)], both device NHWC16. */
MNNB200_API mnnb200_status mnnb200_conv_int8_execute(mnnb200_exec* e, const int8_t* x_nhwc16, int8_t* y_nhwc16);
/* force a kernel variant for A/B parity runs (conv or linear execution):
 * 0 = auto (a conv: the dp4a stem kernel for <= 4 input channels unless GEMM-shaped, else the conv-group kernel when it takes
 * the conv (exactly when mnnb200_conv_int8_groupable is 1), else mma.sync), 1 = mma.sync implicit GEMM (conv only), 2 = wgmma:
 * a conv on the conv-group kernel (NOT_SUPPORT at execute when that kernel does not take it), a linear on the GEMM with one CTA
 * per tile, 3 = wgmma CTA-pair GEMM (linear only: 2-CTA cluster, >= 256 tokens), 4 = weight-streaming GEMV (linear only:
 * <= 8 tokens, the decode step; auto picks it there).  A conv takes 0 / 1 / 2, a linear 0 / 2 / 3 / 4; anything else is
 * INVALID_VALUE. */
MNNB200_API mnnb200_status mnnb200_conv_int8_set_variant(mnnb200_exec* e, int variant);
/* algorithmic bytes / MACs of the last resize (input + output + weights once each; SURVEY 8d) */
MNNB200_API mnnb200_status mnnb200_exec_cost(mnnb200_exec* e, double* bytes, double* macs);

/* ---- The remaining ops of an int8 ResNet-50 .mnn (SURVEY F13) --------------------------------------------------------------
 * int8 Scale: replaces CPUScaleInt8 {ctor, onResize, onExecute} (source/backend/cpu/CPUScaleInt8.cpp:19-122; the reference CUDA
 * backend has no int8 Scale) with MNNScaleAndAddBiasInt8's integer arithmetic (compute/Int8FunctionsOpt.cpp:2207-2252).
 * create: per-channel float scale / bias (bias may be NULL); resize: fold the tensors' quant info into 15-bit fixed point. */
MNNB200_API mnnb200_status mnnb200_scale_int8_create(mnnb200_runtime* rt, int channels, const float* scale, const float* bias,
                                                     mnnb200_exec** out);
MNNB200_API mnnb200_status mnnb200_scale_int8_resize(mnnb200_exec* e, float in_scale, int in_zero, float out_scale, int out_zero,
                                                     int clamp_min, int clamp_max);
MNNB200_API mnnb200_status mnnb200_scale_int8_execute(mnnb200_exec* e, const int8_t* x_nhwc16, int n, int h, int w,
                                                      int8_t* y_nhwc16);
/* int8 Pooling between tensors with EQUAL quant attrs: CPUPoolInt8 (source/backend/cpu/CPUPoolInt8.cpp:19-215) with the x86
 * kernels' semantics (x86_x64/FunctionDispatcher.cpp:122-168: uint8 storage; avg = (sum * floor(2^24/count)) >> 24 over the valid
 * window, max = SIGNED compare of the stored bytes).  pad_h/pad_w are the begin pads. */
MNNB200_API mnnb200_status mnnb200_pool_int8(mnnb200_runtime* rt, const int8_t* x_nhwc16, int n, int c, int ih, int iw, int kh,
                                             int kw, int stride_h, int stride_w, int pad_h, int pad_w, int is_avg,
                                             int8_t* y_nhwc16, int oh, int ow);
/* float ReLU (CPURelu.cpp, MNNReluWithSlope): y = x < 0 ? x * slope : x over `count` contiguous floats.
 * x and y must be 16-byte aligned (the kernel moves float4 words): INVALID_VALUE otherwise, before anything is enqueued. */
MNNB200_API mnnb200_status mnnb200_relu_f32(mnnb200_runtime* rt, const float* x, size_t count, float slope, float* y);
/* float Reduction over the middle axis of [outside][axis][inside] (CPUReduction.cpp): op 0 SUM, 1 MEAN, 2 MAX, 3 MIN, 4 PROD */
MNNB200_API mnnb200_status mnnb200_reduce_f32(mnnb200_runtime* rt, const float* x, int outside, int axis, int inside, int op,
                                              float* y);

/* ---- Conv group: ONE persistent launch for a list of int8 convolutions whose inputs are all ready when the group is
 *      enqueued: 1x1 stride-1 unpadded convs as GEMMs, the others (stride_w <= 2) as implicit GEMMs.  Replaces the
 *      per-command Execution::onExecute walk of Pipeline::execute (source/core/Pipeline.cpp:1069-1140) over
 *      ConvInt8CutlassExecution::onExecute
 *      (execution/int8/ConvInt8CutlassExecution.cu:381-445) for such a run of commands: the members' TMA descriptors and
 *      epilogue constants go into a device-side layer table and all (layer, tile) work items into one schedule dealt
 *      round-robin to one CTA per SM.  The members stay owned by the caller and must outlive the group.
 *      create: every member must be a conv execution (mnnb200_conv_int8_create*), count <= 64.
 *      bind:   after every member's resize; xs[i] / ys[i] = member i's NHWC16 input / output (must not alias another
 *              member's output: members are NOT ordered against each other).  NOT_SUPPORT if the conv-group kernel does
 *              not take a member (mnnb200_conv_int8_group_plan says which).
 *      execute: enqueue the one launch on the runtime's stream. */
MNNB200_API mnnb200_status mnnb200_conv_group_create(mnnb200_runtime* rt, mnnb200_exec* const* members, int count,
                                                     mnnb200_exec** out);
MNNB200_API mnnb200_status mnnb200_conv_group_bind(mnnb200_exec* group, const int8_t* const* xs, int8_t* const* ys);
MNNB200_API mnnb200_status mnnb200_conv_group_execute(mnnb200_exec* group);
/* 1 if auto execute runs the (resized) conv on the conv-group kernel; such a conv can be a member of a conv group */
MNNB200_API int mnnb200_conv_int8_groupable(mnnb200_exec* e);
/* read-only view of the resized conv's layer on the conv-group kernel, as resize planned it: the first `count` (at most 10) of
 * {mode (0 = 1x1 GEMM, 1 = implicit GEMM), cb (bytes of K per TMA chunk: 128 / 64 / 16), bn (tile width), n_chunks, m_tiles,
 * num_kb (K blocks per tile), K, R (row boxes per M tile), TWp (pixels per row box), BH (output rows per box)} go to fields.
 * NO_EXECUTION before resize, NOT_SUPPORT if the conv-group kernel does not take the conv.  Changes nothing. */
MNNB200_API mnnb200_status mnnb200_conv_int8_group_plan(mnnb200_exec* e, int* fields, int count);

/* ---- Int8 Winograd Conv2D F(m x m, 3 x 3), m = 2 / 4 / 6: the op carries a winogradAttr (per-position input scales /
 *      zero points and per-(position, oc) weight scales).  Replaces the structure of ConvWinogradExecution {Resource,
 *      onResize, onExecute} + WinoInputTrans / WinoTrans2Output (execution/ConvWinogradExecution.cu:38-520,
 *      WinogradTrans.cuh:7-595, float only in the reference CUDA backend) with the CPU backend's ConvInt8Winograd
 *      arithmetic (compute/ConvInt8Winograd.cpp:25-126 makeWinoResource, :306-356 onExecute, :396-651 WinoExecution), as
 *      built without AVX512 (the AVX512 build of that op is wrong upstream; SURVEY F8).
 *      attr = Convolution2D.symmetricQuan.winogradAttr verbatim (core/WinogradInt8Attr.hpp:45-63), attr_len int32 words.
 *      NOT_SUPPORT for anything but one full-kernel 3x3 unit, stride/dilation/group 1. */
MNNB200_API mnnb200_status mnnb200_conv_int8_wino_create(mnnb200_runtime* rt, const mnnb200_conv_desc* desc,
                                                         const int8_t* weight, const float* wscale, const float* bias,
                                                         const int32_t* attr, int attr_len, mnnb200_exec** out);
/* in/out quant = inputs[0]/outputs[0] quant info when the tensors carry it, else the op's quanParameter.scaleIn/scaleOut and
 * symmetricQuan.{zeroPoint, outputZeroPoint, clampMin, clampMax} (ConvInt8Winograd.cpp:316-330). */
MNNB200_API mnnb200_status mnnb200_conv_int8_wino_resize(mnnb200_exec* e, int n, int ih, int iw, float in_scale,
                                                         int in_zero, float out_scale, int out_zero, int clamp_min,
                                                         int clamp_max, int* oh, int* ow);
MNNB200_API mnnb200_status mnnb200_conv_int8_wino_execute(mnnb200_exec* e, const int8_t* x_nhwc16, int8_t* y_nhwc16);
/* measurement hook: run a subset of the three enqueues (bit 0 input transform, bit 1 position GEMMs, bit 2 output
 * transform); execute() == phases 7.  bench.py times each kernel class alone against its own roofline (SURVEY 8d C3). */
MNNB200_API mnnb200_status mnnb200_conv_int8_wino_execute_phases(mnnb200_exec* e, const int8_t* x_nhwc16,
                                                                 int8_t* y_nhwc16, int phases);
/* resize checks everything before it changes anything: a refusal (COMPUTE_SIZE_ERROR for an empty output or more tiles than
 * 32-bit row coordinates reach, INVALID_VALUE for a zero scale) keeps the previous plan; a failure while building the new one
 * (out of memory) leaves none, and execute returns NO_EXECUTION until a resize succeeds.  execute / execute_phases return
 * INVALID_VALUE unless x and y are 4-byte aligned.
 * Read-only view of the resized execution's launch: the first `count` (at most 13) of {unit, T (Winograd tiles), m_tiles
 * (128-tile rows of the position GEMMs), Cp, OCp (ic / oc rounded up to 16), bn (columns per work item), n_chunks, items
 * (work items), grid (persistent CTAs), one_tile (grid == items), resident_b (the weights stay in shared memory), stages
 * (operand ring), num_kb (128-byte K blocks per item)} go to fields.  F(2,3) reports its fused kernel (bn 8, B streamed);
 * F(4,3) / F(6,3) the batched position GEMM.  NO_EXECUTION before resize, INVALID_VALUE for any other kind of execution. */
MNNB200_API mnnb200_status mnnb200_conv_int8_wino_plan(mnnb200_exec* e, int* fields, int count);

/* ---- Depthwise int8 conv: replaces DepthwiseConvInt8Execution (execution/int8/DepthwiseConvInt8Execution.cu)
 *      with CPUDepthwiseConvInt8 arithmetic (CPUConvolution.cpp:181-192, Int8FunctionsOpt.cpp:1767-1814). */
MNNB200_API mnnb200_status mnnb200_dwconv_int8_create(mnnb200_runtime* rt, const mnnb200_conv_desc* desc,
                                                      const int8_t* weight, const float* wscale, const float* bias,
                                                      mnnb200_exec** out);
MNNB200_API mnnb200_status mnnb200_dwconv_int8_resize(mnnb200_exec* e, int n, int ih, int iw, float in_scale,
                                                      int in_zero, float out_scale, int out_zero, int clamp_min,
                                                      int clamp_max, int* oh, int* ow);
MNNB200_API mnnb200_status mnnb200_dwconv_int8_execute(mnnb200_exec* e, const int8_t* x_nhwc16, int8_t* y_nhwc16);

/* ---- int8 neighbours of the conv path (SURVEY 8f rank 1-2), all on NHWC16 tensors.
 *      binary add: replaces BinaryInt8Execution (execution/int8/BinaryInt8Execution.cu) with MNNBinaryAddInt8's
 *      arithmetic (compute/Int8FunctionsOpt.cpp:1926-1975).
 *      avg pool:   int8 tensors whose quant attrs differ -- the pipeline's Int8ToFloat -> poolingAvg<float> ->
 *      FloatToInt8 chain (CPUPool.hpp:227-394, Pipeline.cpp:367-395) fused into one kernel.
 *      pad_type: 0 CAFFE 1 VALID 2 SAME; count_type: 0 DEFAULT 1 INCLUDE_PADDING 2 EXCLUDE_PADDING (CaffeOp.fbs).
 *      softmax:    CPUSoftmax int8 mode (CPUSoftmax.cpp:85-150) over the channel axis of an [rows][p16(c)] tensor. */
MNNB200_API mnnb200_status mnnb200_binary_add_int8(mnnb200_runtime* rt, const int8_t* x0, float s0, int z0,
                                                   const int8_t* x1, float s1, int z1, int8_t* y, float s_out, int z_out,
                                                   int min_v, int max_v, int n, int c, int h, int w);
MNNB200_API mnnb200_status mnnb200_avgpool_int8(mnnb200_runtime* rt, const int8_t* x, int n, int c, int ih, int iw, int kh,
                                                int kw, int stride_h, int stride_w, int pad_h, int pad_w, int pad_type,
                                                int count_type, float s_in, float z_in, float s_out, float z_out, int min_v,
                                                int max_v, int8_t* y, int oh, int ow);
MNNB200_API mnnb200_status mnnb200_softmax_int8(mnnb200_runtime* rt, const int8_t* x, int rows, int c, float s_in, float z_in,
                                                float s_out, float z_out, int min_v, int max_v, int8_t* y);

/* ---- fp32 neighbours the pipeline leaves between casts (device fp32 tensors are NCHW-linear):
 *      pool_f32:   CPUPool poolingAvg<float> / poolingMax<float> (CPUPool.hpp:227-394) for a Pooling whose input/output quant
 *                  attrs differ (RuntimeCreator::onSetQuantInfo returns false, Pipeline.cpp:361-395 inserts casts around it);
 *      raster_b32: Raster's strided region copies over 4-byte elements (Tensor::InsideDescribe::Region,
 *                  source/core/TensorUtils.hpp:45-52; replaces execution/Raster.cu blit kernels).  Offsets/strides in elements. */
typedef struct mnnb200_region {
    const void* src;
    int32_t src_offset, src_stride[3], dst_offset, dst_stride[3], size[3];
} mnnb200_region;
MNNB200_API mnnb200_status mnnb200_pool_f32(mnnb200_runtime* rt, const float* x_nchw, int n, int c, int ih, int iw, int kh, int kw,
                                            int stride_h, int stride_w, int pad_h, int pad_w, int pad_type, int count_type,
                                            int is_avg, float* y_nchw, int oh, int ow);
MNNB200_API mnnb200_status mnnb200_raster_b32(mnnb200_runtime* rt, const mnnb200_region* regions, int count, void* dst,
                                              size_t dst_bytes, int zero_fill);
/* dst[b][c][r] = src[b][r][c] over 4-byte elements (Raster's transpose regions / the [N][C][tokens] <-> [tokens][C] step either
 * side of the LLM linear layer; replaces execution/Transpose.cu) */
MNNB200_API mnnb200_status mnnb200_transpose_b32(mnnb200_runtime* rt, const void* src, int batch, int rows, int cols, void* dst);
MNNB200_API mnnb200_status mnnb200_memcpy_d2d(mnnb200_runtime* rt, void* dst_dev, const void* src_dev, size_t bytes);

/* ---- LLM linear ("quantized MatMul"): Convolution 1x1 with int8 weights and dynamic per-token activation
 *      quantisation.  Replaces ConvFpAIntBExecution (execution/weight_only_quant/ConvFpAIntBExecution.cu:1401-2010)
 *      with the CPU Memory_Low arithmetic (compute/ConvInt8TiledExecutor.cpp:1990-2096).
 *      wq [oc][ic] int8, alpha [oc], wzero [oc] or NULL (symmetric), bias [oc] or NULL.
 *      x [tokens][ic] fp32 device, y [tokens][oc] fp32 device.
 *      execute picks by token count: >= 256 tokens the CTA-pair wgmma GEMM, <= 8 tokens (the decode step; the reference CUDA backend's
 *      GEMV family, ConvFpAIntBExecution.cu:433-1190) one weight-streaming GEMV kernel with the per-token quantisation fused, otherwise
 *      the single-CTA wgmma GEMM -- all three produce identical bits for the same token count.  ONE token is a different arithmetic
 *      in the reference (inputPlane == 1: asymmetric single-quant with the input zero folded into the bias,
 *      ConvInt8TiledExecutor.cpp:1033-1035, 1432, 2016-2050); only the GEMV kernel implements it, so tokens == 1 with a forced
 *      variant 2 / 3 returns NOT_SUPPORT instead of computing the multi-token form. */
MNNB200_API mnnb200_status mnnb200_linear_w8_create(mnnb200_runtime* rt, int ic, int oc, const int8_t* wq,
                                                    const float* alpha, const float* wzero, const float* bias,
                                                    int relu, int relu6, mnnb200_exec** out);
/* K-blocked weight scales (MNN-LLM's quant_block export; ConvInt8TiledExecutor.cpp mBlockNum): K is split into `blocks` equal runs
 * of bs = ic / blocks channels, alpha and wzero are [oc][blocks] (wzero NULL when symmetric).  Each block's int32 accumulator is
 * finished into an fp32 running sum in block order, the arithmetic of mnn_oracle_linear_w8_dynamic_blocks bit for bit, on the same
 * GEMM and GEMV kernels; resize / execute / set_variant as above.  blocks < 1 or ic % blocks != 0: INVALID_VALUE; bs % 32 != 0
 * (a wgmma k-step is 32 bytes), or bs not a power of two up to 512: NOT_SUPPORT.  blocks == 1 is the per-channel layer.  The
 * CTA-pair variant (3) returns NOT_SUPPORT for blocked layers; auto runs >= 9 tokens on the single-CTA GEMM. */
MNNB200_API mnnb200_status mnnb200_linear_w8_create_blocked(mnnb200_runtime* rt, int ic, int oc, int blocks, const int8_t* wq,
                                                            const float* alpha, const float* wzero, const float* bias,
                                                            int relu, int relu6, mnnb200_exec** out);
MNNB200_API mnnb200_status mnnb200_linear_w8_resize(mnnb200_exec* e, int tokens);
MNNB200_API mnnb200_status mnnb200_linear_w8_execute(mnnb200_exec* e, const float* x, float* y);

/* ---- Float MatMul / BatchMatMul: replaces MatMulExecution {setArguments, onResize, onExecute} and its 18 CUTLASS variants
 *      (execution/MatMulExecution.cu:306-1392) with one wgmma kernel: fp32 operands are read in place as tf32 ( an
 *      operand that is not K-major is transposed first), fp16 operands use f16 wgmma; fp32 accumulate / output.
 *      C[b][e][h] = op(A)[b][e][l] * op(B)[b][l][h] (+ bias[h]); transpose_a: A is stored [l][e]; transpose_b: B is stored
 *      [h][l] (CPUMatMul.cpp / CPUBatchMatMul adjX, adjY).  a/b: device fp32 (inputs_are_f16 = 0) or fp16 (= 1), c: device fp32.
 *      Accuracy: max|C - C_cpu| / max|C_cpu| <= 1e-3 (10-bit operand mantissa; fp32 range for fp32 inputs). */
MNNB200_API mnnb200_status mnnb200_matmul_create(mnnb200_runtime* rt, int batch, int e, int l, int h, int transpose_a,
                                                 int transpose_b, int inputs_are_f16, mnnb200_exec** out);
MNNB200_API mnnb200_status mnnb200_matmul_execute(mnnb200_exec* e, const void* a, const void* b, const float* bias, float* c);

/* ---- Float convolutions of fp32 models and their fp32 neighbours: the CPU backend's float path (CPUConvolution /
 *      ConvolutionTiledExecutor, CPUConvolutionDepthwise, CPUBinary ADD, CPUScale, CPUSoftmax) on NCHW-linear device fp32 tensors.
 *      Activation: desc->relu = ReLU, relu6 = ReLU6 (CPUConvolution.cpp:289-291), applied after the bias.
 *      conv_f32: group == 1 (NOT_SUPPORT otherwise), any kernel / stride / dilation / padding.  create takes host weights
 *                [oc][ic][kh][kw] and bias [oc] (may be NULL) and packs them once on the device as two TF32 halves w = w_hi + w_lo;
 *                execute runs one split-TF32 wgmma implicit GEMM (a_hi*w_hi + a_hi*w_lo + a_lo*w_hi, fp32 accumulate: error near
 *                fp32's).  resize plans the launch for the shape (*oh / *ow as in conv_int8_resize); set_pad sets the begin pads
 *                (ConvolutionCommon::convolutionPad) of a conv_f32 or dwconv_f32 execution, before resize.
 *      dwconv_f32: group == ic == oc, weights [c][kh][kw].
 *      binary_add_f32: y = a + b over count elements (equal shapes, no broadcast).
 *      scale_f32: y[n][c][h][w] = x * scale[c] + bias[c] (bias may be NULL).
 *      softmax_f32: softmax over the middle axis of an [outside][axis][inside] view. */
MNNB200_API mnnb200_status mnnb200_conv_f32_create(mnnb200_runtime* rt, const mnnb200_conv_desc* desc, const float* weight,
                                                   const float* bias, int relu6, mnnb200_exec** out);
MNNB200_API mnnb200_status mnnb200_conv_f32_set_pad(mnnb200_exec* e, int pad_h, int pad_w);
MNNB200_API mnnb200_status mnnb200_conv_f32_resize(mnnb200_exec* e, int n, int ih, int iw, int* oh, int* ow);
MNNB200_API mnnb200_status mnnb200_conv_f32_execute(mnnb200_exec* e, const float* x_nchw, float* y_nchw);
/* read-only view of the resized conv_f32 execution's launch, as resize planned it: the first `count` (at most 7) of
 * {bn (tile width 32 / 64 / 128), n_chunks, m_tiles (128-pixel M tiles), num_kb (32-wide K blocks per tile), stages (K blocks the
 * bn-wide kernel's shared-memory ring holds), cp8 (ic rounded up to 8), taps (kh * kw)} go to fields.  NO_EXECUTION before resize,
 * INVALID_VALUE for any other kind of execution.  Changes nothing. */
MNNB200_API mnnb200_status mnnb200_conv_f32_plan(mnnb200_exec* e, int* fields, int count);
MNNB200_API mnnb200_status mnnb200_dwconv_f32_create(mnnb200_runtime* rt, const mnnb200_conv_desc* desc, const float* weight,
                                                     const float* bias, int relu6, mnnb200_exec** out);
MNNB200_API mnnb200_status mnnb200_dwconv_f32_resize(mnnb200_exec* e, int n, int ih, int iw, int* oh, int* ow);
MNNB200_API mnnb200_status mnnb200_dwconv_f32_execute(mnnb200_exec* e, const float* x_nchw, float* y_nchw);
MNNB200_API mnnb200_status mnnb200_binary_add_f32(mnnb200_runtime* rt, const float* a, const float* b, float* y, size_t count);
MNNB200_API mnnb200_status mnnb200_scale_f32_create(mnnb200_runtime* rt, int channels, const float* scale, const float* bias,
                                                    mnnb200_exec** out);
MNNB200_API mnnb200_status mnnb200_scale_f32_resize(mnnb200_exec* e, int n, int h, int w);
MNNB200_API mnnb200_status mnnb200_scale_f32_execute(mnnb200_exec* e, const float* x_nchw, float* y_nchw);
MNNB200_API mnnb200_status mnnb200_softmax_f32(mnnb200_runtime* rt, const float* x, int outside, int axis, int inside, float* y);

/* ---- Float BinaryOp / UnaryOp / ArgMax of fp32 models (CPUBinary, CPUEltwise, CPUUnary, CPUArgMax) on device fp32 tensors in
 *      any one linear layout; all enqueue-only and capturable into a CUDA graph.
 *      binary_f32: y[i] = a[i] op b[i] over count elements, then ReLU when relu != 0 (BinaryOp.activationType 1).  count_a and
 *                  count_b are count or 1; a one-element side is broadcast and read on the device.  op = BinaryOpOperation:
 *                  ADD 0, SUB 1, MUL 2, REALDIV 7, MINIMUM 8, MAXIMUM 9, SquaredDifference 14 ((a - b) * (a - b)); every op is one
 *                  round-to-nearest fp32 operation, bit-identical to the CPU.  Any other op: NOT_SUPPORT.
 *                  binary_add_f32 above is binary_f32 with ADD, equal counts and no ReLU.
 *      unary_f32:  y[i] = op(x[i]), op = UnaryOpOperation: ABS 0, NEG 1, SQUARE 4, SQRT 5, RSQRT 6, EXP 7, LOG 8,
 *                  RECIPROCAL 15, SIGMOID 29, TANH 30, HARDSWISH 31 ((x * min(max(x + 3, 0), 6)) / 6), GELU 32 (tanh form),
 *                  GELU_STANDARD 33 (erf form), SILU 34.  ABS, NEG, SQUARE, SQRT, RSQRT, RECIPROCAL and HARDSWISH are exact
 *                  round-to-nearest; the others within a few ulp.  Any other op: NOT_SUPPORT.
 *      argmax_f32: y_int32[o][i] = the index along the middle axis of an [outside][axis][inside] view of the first maximum
 *                  (is_min != 0: minimum), CPUArgMax with topK 1 and no max values. */
MNNB200_API mnnb200_status mnnb200_binary_f32(mnnb200_runtime* rt, int op, const float* a, size_t count_a, const float* b,
                                              size_t count_b, float* y, size_t count, int relu);
MNNB200_API mnnb200_status mnnb200_unary_f32(mnnb200_runtime* rt, int op, const float* x, float* y, size_t count);
MNNB200_API mnnb200_status mnnb200_argmax_f32(mnnb200_runtime* rt, const float* x, int outside, int axis, int inside, int is_min,
                                              int32_t* y_int32);

MNNB200_API void mnnb200_exec_destroy(mnnb200_exec* e);

#ifdef __cplusplus
}
#endif
#endif /* MNN_B200_H */
