// kernels.h -- host-callable launchers of the sm_90a kernels (all enqueue-only on the given stream).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

struct alignas(64) CUtensorMap_st_opaque { unsigned long long opaque[16]; };   // same size/alignment as CUtensorMap (cuda.h)

namespace mnnb200 {

struct ConvParams {
    const int8_t* x;      // [N][IH][IW][Cp]           int8 NHWC16
    const int8_t* w;      // [OCw][KH*KW][Cp]          int8, tap-major / channel-minor K, zero padded
    int8_t* y;            // [N][OH][OW][OCp]          int8 NHWC16
    const float* wscale;  // [OCp] first multiplier  (weight scale, or the legacy fused scale)
    const float* bias;    // [OCp] biasFloat (CPUConvolution.cpp:194-197)
    const int32_t* wsum128;  // [OCp] 128 * sum_k w[oc][k]  -- the x86 uint8 storage offset, added in int32
    float scale_x;        // s_in / s_out (1.0 for legacy)
    float minv, maxv;     // clamp (min = z_out when relu)
    int32_t zin_splat;    // input zero point replicated in 4 bytes: value of padded taps
    int N, IH, IW, Cp, OH, OW, OC, OCp, OCw;
    int KH, KW, sh, sw, ph, pw, dh, dw;
    int M;                // N*OH*OW
    int Kc;               // KH*KW*Cp/16: number of 16-byte K chunks
};

// tile configurations of the mma.sync implicit-GEMM kernel
enum ConvTile { TILE_128x64 = 0, TILE_128x32, TILE_128x16, TILE_64x64, TILE_64x32, TILE_128x128, TILE_COUNT };
void conv_tile_shape(int tile, int* bm, int* bn);
cudaError_t launch_conv_int8_igemm(const ConvParams& p, int tile, cudaStream_t stream);

// first-layer convolution (<= 4 input channels): one thread per output pixel, dp4a against a tap-major weight table in smem
bool conv_int8_stem_supported(const ConvParams& p, int ic);
cudaError_t launch_conv_int8_stem(const ConvParams& p, cudaStream_t stream);

// wgmma (s8 x s8 -> s32, register accumulators, TMA operand loads) GEMM with fp32 output for the linear layers and the
// Winograd position GEMMs
struct GemmI8Params {
    const int8_t* a;  // [M][K]  row-major, K % 16 == 0
    const int8_t* b;  // [Nw][K] row-major ("column-major" B), zero padded rows
    int M, N, K;      // N = output columns padded to 16: the n chunks cover N
    int ldy;
    const float* wscale;
    const float* bias;
    const int32_t* wsum128;
    int OC;           // valid output columns
    // dynamic-quant linear: y = acc*alpha*dq[m] + (dq[m]*-128)*wsum[n] + srcsum[m]*wzero[n] + bias[n]
    float* y_f32;     // [M][ldy], required
    const float* dq;      // [M] per-token dequant scale
    const float* srcsum;  // [M] float(sum_k (xq+128)) * dq
    const float* wsumf;   // [N] weightKernelSum
    const float* wzero;   // [N] or nullptr
    int relu, relu6;
    // K-blocked weight scales (bs = 0: per channel, the fields above): K runs in blocks of bs bytes (bs % 32 == 0, bn <= 128),
    // each block's int32 accumulator is finished into an fp32 running sum (mnn_oracle_linear_w8_dynamic_blocks):
    //   f += float(acc_b + bw128[b][n]) * balpha[b][n] * dq[m] + (dq[m] * -128) * bws[b][n] + xsb[m][b] * bwzero[b][n]
    // then + bias[n].  Tables [blocks][N], zero past OC; xsb = float(sum_{k in b} (xq + 128)) * dq.
    int bs, blocks;
    const float *balpha, *bwzero, *bws, *xsb;
    const int32_t* bw128;
    // batched mode (int8 Winograd: one GEMM per transform position a).  A = [batch][a_batch_rows][K],
    // B = [batch][b_batch_rows][K], per-column constants [batch][c_batch_stride], fp32 out [batch][a_batch_rows][ldy]:
    //   y = float(acc + wsum128[a][n]) * wscale[a][n] + bias[a][n]        (wino = 1)
    int batch, a_batch_rows, b_batch_rows, c_batch_stride, wino;
};
cudaError_t launch_gemm_i8_wgmma(const GemmI8Params& p, const void* tmap_a, const void* tmap_b, int bn, cudaStream_t stream,
                                 int sm_count);
// the launch launch_gemm_i8_wgmma makes for (p, bn) on sm_count SMs: work items (batch, m tile, n chunk), persistent grid,
// one_tile (every CTA owns exactly one item), resident_b (the weights stay in shared memory for the whole launch), the
// operand ring's stages, 128-byte K blocks per item and the dynamic shared memory
struct GemmI8Launch {
    int items, grid, one_tile, resident_b, stages, num_kb, smem;
};
GemmI8Launch gemm_i8_wgmma_launch(const GemmI8Params& p, int bn, int sm_count);
// ---- one persistent launch over a LIST of int8 convolutions (conv_group_wgmma.cu); a lone conv runs as a one-layer list.
//      Two layer modes:
//   mode 0  GEMM-shaped (1x1, stride 1, no pad): A = the NHWC16 activation as a 2D matrix, one TMA box per K block
//   mode 1  implicit GEMM (any kernel / stride <= 2 / dilation / padding): an M tile = R whole output rows of TWp pixels each; the
//           A operand of K block (tap, channel chunk) is gathered by R TMA boxes from a 4D {C, W, H, N} view of the input
//           (one view per column parity for stride 2); out-of-image taps are zero-filled by TMA and, for a non-zero input zero
//           point, corrected in the epilogue with a per-(border class, oc) table  z_in * sum_{OOB taps} w
constexpr int kGroupMaxLayers = 64;
constexpr int kGroupMaxBN = 128;     // 64 accumulator registers per consumer thread
constexpr uint32_t kGroupSchedEnd = 0xffffffffu;
// The TMA descriptors of ALL layers travel as ONE __grid_constant__ kernel parameter (24 KB of the 32 KB parameter space): a
// descriptor that lives in global memory is re-fetched by the TMA unit for every cp.async.bulk.tensor (measured: ~1 us per
// instruction, 2.8 us per work item with nothing else left in the kernel), one in the parameter bank is not.
struct GroupMapsParam {
    CUtensorMap_st_opaque a[kGroupMaxLayers];
    CUtensorMap_st_opaque b[kGroupMaxLayers];
    CUtensorMap_st_opaque a1[kGroupMaxLayers];   // odd-column view (stride 2, mode 1)
};
// Inside an n chunk of bn columns the kernel's GEMM columns are permuted so that the wgmma fragment gives each thread
// contiguous output channels: in every 32-column group, GEMM column 32 G + 8 s + 2 q + e computes channel 32 G + 8 q + 2 s + e
// (a 16-wide last group, bn % 32 == 16: 32 G + 4 q + 2 s + e).  The weight rows, the epilogue table and the border-correction
// table are laid out in this order.
inline int group_column_channel(int c, int bn) {
    const int g = c & ~31, s = (c >> 3) & 3, q = (c >> 1) & 3, e = c & 1;
    return bn - g >= 32 ? g + 8 * q + 2 * s + e : g + 4 * q + 2 * s + e;
}
struct GroupLayerParams {            // copied to shared memory by every CTA
    int8_t* y;
    // epilogue table [n_chunks][3][bn], GEMM-column order, zero past OC: wscale, biasFloat (float) and the accumulators' start
    // value preset = 128 sum w (+ 0x4B400000 when K <= 128, for the exact int -> float trick of the small-K requant) (int32)
    const float* ep;
    int M, N, K, bn;                 // mode 0: M rows, K = Cp.  mode 1: M = N*OH*OW, K = taps*Cp
    int n_chunks, m_tiles, num_kb, OC;
    int ldy;
    float scale_x, minv, maxv;
    int mode, cb, TWp, R;            // cb: bytes of K per TMA chunk (128 / 64 / 16); mode 1: R boxes of BH rows x TWp pixels per M tile
};
struct GroupConvGeom {               // mode 1 only; stays in global memory (read once per tile)
    int KH, KW, Cp, NB;
    int sh, sw, ph, pw;
    int dh, dw, OH, OW;
    int SEG, rowboxes, cpt, chunks;  // rowboxes = NB*OHB*SEG boxes; cpt = chunks per tap; chunks = taps*cpt (+1 dummy if odd and cb == 16)
    int BH, OHB, pad0_, pad1_;       // a TMA box covers BH consecutive output rows of one image (stride_h == 1), OHB = OH / BH boxes per image
    const uint8_t* hcls;             // [OH] border class of an output row   (nullptr: z_in == 0, no correction)
    const uint8_t* wcls;             // [OW] border class of an output column
    const int32_t* corr;             // [HC*WC][n_chunks*bn] z_in * sum over the out-of-image taps of sum_c w[oc][tap][c], in
                                     // GEMM-column order (group_column_channel), zero past OC; the interior
                                     // class's row is zeros (the epilogue adds it for pixels next to a border pixel)
    int wc_count, interior_cls;
};
// schedule: grid rows of sched_stride items, each row ends with kGroupSchedEnd.  item = layer << 26 | n chunk << 20 |
// (tiles - 1) << 14 | first m tile; the host puts one M tile in every item (tile count field 0).  A layer whose n chunks or
// M tiles these fields cannot hold is not taken by the conv-group kernel.
constexpr int kGroupItemLayerShift = 26, kGroupItemChunkShift = 20, kGroupItemCountShift = 14;
constexpr uint32_t kGroupItemChunkMask = 0x3fu, kGroupItemCountMask = 0x3fu, kGroupItemTileMask = 0x3fffu;
constexpr int kGroupMaxNChunks = 63, kGroupMaxMTiles = 16383;
cudaError_t launch_conv_group(const GroupMapsParam* maps_host, const GroupLayerParams* params, const GroupConvGeom* geom, int n_layers,
                              const uint32_t* sched, int sched_stride, int grid, cudaStream_t stream);

// CTA-pair variant (2-CTA cluster, 256 x bn per pair, B halves multicast to both CTAs) for the tensor-bound linear layers;
// fp32 dynamic-quant epilogue only.  tmap_b must have a box of bn/2 rows (each CTA of the pair loads half of the B tile);
// bn % 32 == 0.
cudaError_t launch_gemm_i8_2cta(const GemmI8Params& p, const void* tmap_a, const void* tmap_b_half, int bn, cudaStream_t stream,
                                int sm_count);

// float (batched) MatMul on wgmma f16 / tf32 (gemm_f16_wgmma.cu): an operand that is not K-major already is packed first, in its
// own type (fp16 or fp32)
cudaError_t launch_pack_kmajor_f16(const void* src, void* dst, int batch, int rows, int k, int kp, int trans, cudaStream_t s);
cudaError_t launch_pack_kmajor_f32(const float* src, float* dst, int batch, int rows, int k, int kp, int trans, cudaStream_t s);
// k_bytes = bytes of one K-major operand row; tf32 = 1: operands are fp32 consumed as tf32, else fp16
cudaError_t launch_gemm_f16_wgmma(const void* tmap_a, const void* tmap_b, int batch, int M, int N, int k_bytes, int tf32,
                                  int a_batch_rows, int b_batch_rows, int bn, float* c, const float* bias, cudaStream_t stream,
                                  int sm_count);

// fp32 Conv2D (group 1) on split-TF32 wgmma (conv_f32_wgmma.cu): NCHW-linear fp32 in and out.  Weights are packed once into two
// K-major arrays hi / lo [ocp][kp] (k = tap * cp8 + c, cp8 = ic rounded up to 8, kp = taps * cp8 rounded up to 32), w = hi + lo.
struct ConvF32Params {
    const float* x;       // [N][IC][IH][IW]
    float* y;             // [N][OC][OH][OW]
    const float* bias;    // [OC]
    int N, IC, IH, IW, OC, OH, OW;
    int KH, KW, sh, sw, ph, pw, dh, dw;
    int Cp8, taps;        // taps = KH * KW
    int M, num_kb;        // M = N * OH * OW, num_kb = kp / 32
    int m_tiles, n_chunks;
    int act;              // 0 none, 1 ReLU, 2 ReLU6
};
cudaError_t launch_pack_conv_w_f32(const float* w, int oc, int ic, int taps, int cp8, int kp, int ocp, float* hi, float* lo,
                                   cudaStream_t s);
// tmap_hi / tmap_lo: 2D maps over the [ocp][kp * 4 bytes] weight arrays with {128 bytes, bn rows} boxes, 128B swizzle; bn 32 / 64 / 128
cudaError_t launch_conv_f32_wgmma(const ConvF32Params& p, const void* tmap_hi, const void* tmap_lo, int bn, cudaStream_t s,
                                  int sm_count);
// pipeline stages of the bn-wide kernel (how many K blocks its shared-memory ring holds); 0 for a width it does not compile
int conv_f32_stages(int bn);

// fp32 neighbours of the float conv, all NCHW-linear.  dwconv: w [C][KH*KW]; act 0 none, 1 ReLU, 2 ReLU6
struct DwF32Params {
    const float* x;
    const float* w;
    const float* bias;
    float* y;
    int N, C, IH, IW, OH, OW, KH, KW, sh, sw, ph, pw, dh, dw, act;
};
cudaError_t launch_dwconv_f32(const DwF32Params& p, cudaStream_t s);
cudaError_t launch_binary_add_f32(const float* a, const float* b, float* y, size_t n, cudaStream_t s);
// fp32 BinaryOp / UnaryOp codes: the reference's BinaryOpOperation / UnaryOpOperation values (schema TensorflowOp.fbs)
enum {
    kBinaryAdd = 0, kBinarySub = 1, kBinaryMul = 2, kBinaryRealDiv = 7, kBinaryMinimum = 8, kBinaryMaximum = 9,
    kBinarySquaredDifference = 14,
};
enum {
    kUnaryAbs = 0, kUnaryNeg = 1, kUnarySquare = 4, kUnarySqrt = 5, kUnaryRsqrt = 6, kUnaryExp = 7, kUnaryLog = 8,
    kUnaryReciprocal = 15, kUnarySigmoid = 29, kUnaryTanh = 30, kUnaryHardSwish = 31, kUnaryGelu = 32, kUnaryGeluStandard = 33,
    kUnarySilu = 34,
};
// y[i] = a op b (then ReLU when relu != 0); a_one / b_one: that side is one element, broadcast to all n
bool binary_f32_supported(int op);
cudaError_t launch_binary_f32(int op, const float* a, bool a_one, const float* b, bool b_one, float* y, size_t n, int relu,
                              cudaStream_t s);
bool unary_f32_supported(int op);
cudaError_t launch_unary_f32(int op, const float* x, float* y, size_t n, cudaStream_t s);
// index of the first maximum (is_min: minimum) along the middle axis of [outside][axis][inside] -> int32 [outside][inside]
cudaError_t launch_argmax_f32(const float* x, int outside, int axis, int inside, int is_min, int32_t* y, cudaStream_t s);
cudaError_t launch_scale_f32(const float* x, const float* scale, const float* bias, float* y, int n, int c, size_t plane,
                             cudaStream_t s);
cudaError_t launch_softmax_f32(const float* x, float* y, int outside, int axis, int inside, cudaStream_t s);

// elementwise / data movement
cudaError_t launch_float_to_int8(const float* x, int n, int c, int h, int w, float inv_scale, float zero, float minv,
                                 float maxv, int8_t* y, cudaStream_t s);
cudaError_t launch_int8_to_float(const int8_t* x, int n, int c, int h, int w, float scale, float zero, float* y,
                                 cudaStream_t s);
cudaError_t launch_pack_nchw_int8(const int8_t* x, int n, int c, int h, int w, int8_t* y, cudaStream_t s);
cudaError_t launch_unpack_nchw_int8(const int8_t* x, int n, int c, int h, int w, int8_t* y, cudaStream_t s);

struct DwParams {
    const int8_t* x;  // [N][IH][IW][Cp]
    const int8_t* w;  // [KH*KW][Cp]
    int8_t* y;        // [N][OH][OW][Cp]
    const float* scale;       // [Cp]
    const int32_t* bias_i32;  // [Cp] already holds -sum(w)*(z_in+128) etc. (CPUConvolution.cpp:181-192) + 128*sum(w)
    int zin, minv, maxv;
    int N, IH, IW, Cp, C, OH, OW, KH, KW, sh, sw, ph, pw, dh, dw;
};
cudaError_t launch_dwconv_int8(const DwParams& p, cudaStream_t s);

// int8 eltwise add (MNNBinaryAddInt8), avg pooling through fp32 (casts + poolingAvg<float>), int8 softmax
cudaError_t launch_binary_add_int8(const int8_t* x0, float s0, int z0, const int8_t* x1, float s1, int z1, int8_t* y,
                                   float inv_out, int z_out, int minv, int maxv, size_t pixels, int c, int cp, cudaStream_t s);
struct PoolParams {
    const int8_t* x;
    int8_t* y;
    int N, C, Cp, IH, IW, OH, OW, KH, KW, sh, sw, ph, pw, count_type;   // count_type: 1 include padding, 2 exclude
    float s_in, z_in, inv_out, z_out, minv, maxv;
};
cudaError_t launch_avgpool_int8_via_float(const PoolParams& p, cudaStream_t s);
cudaError_t launch_pool_f32(const PoolParams& p, const float* x, float* y, int is_avg, cudaStream_t s);   // NCHW fp32
cudaError_t launch_scale_int8(const int8_t* x, int8_t* y, const int32_t* alpha, const int32_t* bias, int z_in, int z_out, int minv,
                              int maxv, size_t pixels, int c, int cp, cudaStream_t s);
cudaError_t launch_pool_int8_x86(const PoolParams& p, int is_avg, cudaStream_t s);   // int8 pooling, equal quant attrs (x86 semantics)
cudaError_t launch_relu_f32(const float* x, float* y, size_t n, float slope, cudaStream_t s);
cudaError_t launch_reduce_f32(const float* x, float* y, int outside, int axis, int inside, int op, cudaStream_t s);
struct RasterRegion { int32_t src_offset, src_stride[3], dst_offset, dst_stride[3], size[3]; };
cudaError_t launch_raster_b32(const RasterRegion& r, const void* src, void* dst, cudaStream_t s);
cudaError_t launch_transpose_b32(const void* src, void* dst, int batch, int rows, int cols, cudaStream_t s);
cudaError_t launch_softmax_int8(const int8_t* x, int rows, int c, int cp, float s_in, float z_in, float inv_out, float z_out,
                                float minv, float maxv, int8_t* y, cudaStream_t s);

// int8 Winograd F(m x m, 3 x 3) transform kernels (winograd_int8.cu); the alpha^2 position GEMMs run on the batched
// wgmma GEMM above.  Scratch: v = [alpha^2][Mpad][Cp] int8, m = [alpha^2][Mpad][OCp] fp32, Mpad = T rounded up to 128.
struct WinoParams {
    const int8_t* x;   // [N][IH][IW][Cp]
    int8_t* v;
    const float* m;
    int8_t* y;         // [N][OH][OW][OCp]
    const float* fused_bias;   // [OCp] bias/s_out + z_out (ConvInt8Winograd.cpp:215-217)
    int N, IH, IW, Cp, OH, OW, OC, OCp, pad_h, pad_w, unit, hU, wU, Mpad;
    long long T;       // N*hU*wU tiles
    float s_in;
    int z_in;
    float out_inv, minv, maxv;
    float in_inv[64];  // 1 / inputScale[a]
    float in_zero[64]; // inputZeroPoint[a]
};
cudaError_t launch_wino_input(const WinoParams& p, cudaStream_t s);
// F(2,3): the 16 position GEMMs + output transform + requantise fused (all 16 accumulators in registers, no fp32 M tensor);
// tmap_u has boxes of kWinoFusedBN rows; its operand ring has kWinoFusedStages stages
constexpr int kWinoFusedBN = 8, kWinoFusedStages = 6;
struct WinoFusedParams {
    int8_t* y;
    const float *scale, *offset, *fused_bias;   // [16][OCp], [16][OCp], [OCp]
    const int32_t* wsum128;                      // [16][OCp]
    int K, Mpad, OCb, OCp, OC, m_tiles, oc_chunks, OH, OW, hU, wU;
    long long T;
    float out_inv, minv, maxv;
};
cudaError_t launch_wino_f23_fused(const WinoFusedParams& p, const void* tmap_v, const void* tmap_u, cudaStream_t s, int sm_count);
cudaError_t launch_wino_output(const WinoParams& p, cudaStream_t s);

// decode-time linear layer: <= 8 tokens x int8 weights [ocp][icp], HBM-streaming dp4a GEMV with the tensor-core path's exact epilogue
struct GemvW8Params {
    const float* x;          // [tokens][ic] fp32 activations (quantised per token inside the kernel)
    const int8_t* w;         // [ocp][icp]
    float* y;                // [tokens][ldy]
    const float *alpha, *bias, *wsumf, *wzero;   // bias / wzero may be null
    const int32_t* wsum128;
    int tokens, ic, oc, ocp, icp, ldy, relu, relu6;
    // K-blocked weight scales (bs = 0: per channel): blocks of bs bytes, bs a power of two in [32, 512]; balpha / bwzero
    // [ocp][ic / bs] (bwzero zeros when symmetric).  The per-block weight sums are taken from the streamed weights, and
    // alpha / wsumf / wzero / wsum128 are not read.
    int bs;
    const float *balpha, *bwzero;
};
bool linear_w8_gemv_supported(int tokens, int icp, int bs = 0);
cudaError_t launch_linear_w8_gemv(const GemvW8Params& p, cudaStream_t s, int sm_count);

// dynamic per-token quantisation (MNNAbsMax + MNNQuantScale + MNNDynamicQuant fused); bs > 0 also writes
// xsb[token][b] = float(sum_{k in block b} (xq_k + 128)) * dq for the blocks of bs channels (ic % bs == 0, bs % 16 == 0)
cudaError_t launch_dynamic_quant(const float* x, int tokens, int ic, int icp, int8_t* xq, float* dq, float* srcsum,
                                 cudaStream_t s, int bs = 0, float* xsb = nullptr);

}  // namespace mnnb200
