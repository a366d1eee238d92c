// capi.cu -- host side of the H100 backend: runtime (device/stream/memory), the Execution objects
// (create = Resource upload, resize = quant-info fold + launch plan, execute = enqueue) and the C ABI
// declared in include/mnn_b200.h.  Mirrors the roles of CUDARuntime / CUDABackend / ConvInt8CutlassExecution
// in the reference (source/backend/cuda/core/runtime/CUDARuntime.cpp, core/CUDABackend.cpp,
// execution/int8/ConvInt8CutlassExecution.cu) but follows the CPU backend's arithmetic (SURVEY F5).
//
// Host float math here is part of the contract (the epilogue constants must equal the CPU backend's
// bit for bit), so this file is compiled with -Xcompiler -ffp-contract=off.
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/mnn_b200.h"
#include "common.cuh"
#include "kernels.h"

namespace mnnb200 {
std::atomic<unsigned long long> g_launch_count{0};
}
using namespace mnnb200;

static thread_local std::string g_err;
static mnnb200_status fail(mnnb200_status s, const std::string& m) {
    g_err = m;
    return s;
}
#define CK(call)                                                                                   \
    do {                                                                                           \
        cudaError_t _e = (call);                                                                   \
        if (_e != cudaSuccess) {                                                                   \
            cudaGetLastError(); /* do not leave it for an unrelated cudaGetLastError() to report */ \
            return fail(MNNB200_CUDA_ERROR, std::string(#call) + ": " + cudaGetErrorString(_e));   \
        }                                                                                          \
    } while (0)

struct mnnb200_runtime {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    cudaDeviceProp prop;
    cudaEvent_t ev_begin = nullptr, ev_end = nullptr;   // onGetLastGpuTimeMs
    bool ev_valid = false;
};
struct mnnb200_graph {
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
};

struct mnnb200_exec {
    mnnb200_runtime* rt = nullptr;
    int kind = 0;  // 1 conv, 2 depthwise, 3 linear
    int variant = 0;  // mnnb200_conv_int8_set_variant: 0 auto, 1 mma.sync implicit GEMM (conv), 2 wgmma, 3 CTA pair, 4 GEMV (linear)
    double cost_bytes = 0, cost_macs = 0;
    std::vector<void*> dev_bufs;  // everything freed at destroy
    virtual ~mnnb200_exec() {
        for (void* p : dev_bufs)
            if (p) cudaFree(p);
    }
    // grow-only scratch owned by the execution: the previous buffer is released (cudaFree waits for the device, so kernels still
    // reading it have finished) and replaced in dev_bufs -- repeated resizes do not accumulate device memory
    mnnb200_status grow_scratch(void** slot, size_t* cap, size_t bytes) {
        if (bytes <= *cap && *slot) return MNNB200_OK;
        void* q = nullptr;
        CK(cudaMalloc(&q, bytes ? bytes : 16));
        if (*slot) {
            for (auto& b : dev_bufs)
                if (b == *slot) b = nullptr;
            cudaFree(*slot);
        }
        dev_bufs.push_back(q);
        *slot = q;
        *cap = bytes;
        return MNNB200_OK;
    }
    template <class T>
    mnnb200_status upload(const std::vector<T>& h, T** d) {
        size_t bytes = h.size() * sizeof(T);
        CK(cudaMalloc((void**)d, bytes ? bytes : 16));
        dev_bufs.push_back(*d);
        if (bytes) CK(cudaMemcpyAsync(*d, h.data(), bytes, cudaMemcpyHostToDevice, rt->stream));
        CK(cudaStreamSynchronize(rt->stream));  // h may be a temporary
        return MNNB200_OK;
    }
    template <class T>
    mnnb200_status update(const std::vector<T>& h, T* d) {
        CK(cudaMemcpyAsync(d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice, rt->stream));
        CK(cudaStreamSynchronize(rt->stream));
        return MNNB200_OK;
    }
};

// ---- TMA descriptors (driver entry point fetched through the runtime: no link-time libcuda dependency)
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled get_encode() {
    static PFN_encodeTiled fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = (PFN_encodeTiled)f;
    });
    return fn;
}
// row-major int8 matrix [rows][k] -> 2D tensor map with a {128 bytes, box_rows} box, 128B swizzle, zero OOB fill
static mnnb200_status make_tmap_i8(CUtensorMap* m, const void* ptr, int rows, int k, int box_rows) {
    PFN_encodeTiled enc = get_encode();
    if (!enc) return fail(MNNB200_CUDA_ERROR, "cuTensorMapEncodeTiled entry point not available");
    cuuint64_t dims[2] = {(cuuint64_t)k, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)k};
    cuuint32_t box[2] = {128u, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1u, 1u};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(MNNB200_CUDA_ERROR, "cuTensorMapEncodeTiled failed: " + std::to_string((int)r));
    return MNNB200_OK;
}
// generic tiled map over uint8 data: dims/box innermost first, strides (bytes) for dims 1..rank-1; swizzle by the inner box bytes
static mnnb200_status make_tmap_u8(CUtensorMap* m, const void* ptr, int rank, const cuuint64_t* dims, const cuuint64_t* strides,
                                   const cuuint32_t* box) {
    PFN_encodeTiled enc = get_encode();
    if (!enc) return fail(MNNB200_CUDA_ERROR, "cuTensorMapEncodeTiled entry point not available");
    cuuint32_t estr[5] = {1u, 1u, 1u, 1u, 1u};
    const CUtensorMapSwizzle sw = box[0] == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : (box[0] == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_NONE);
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, (cuuint32_t)rank, const_cast<void*>(ptr), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(MNNB200_CUDA_ERROR, "cuTensorMapEncodeTiled (rank " + std::to_string(rank) + ") failed: " + std::to_string((int)r));
    return MNNB200_OK;
}
// columns per wgmma work item: split N into equal chunks of at most 256 columns (multiple of 16)
// When the M tiles alone cannot fill the GPU (the 7x7 / 14x14 feature maps of MobileNet: 13 / 49 tiles), N is split
// further (down to 32 columns) so that m_tiles * n_chunks approaches the SM count: a lone CTA streaming a whole K x (A + B)
// panel through one SM's L2 port is what bounds those layers, not the math.
static int pick_bn(int n_padded, int m_tiles = 1 << 30, int sm_count = 1, int max_bn = 256) {
    int chunks = (n_padded + max_bn - 1) / max_bn;
    if ((long)m_tiles * chunks < sm_count) {
        int want = sm_count / m_tiles, cap = n_padded / 32;
        if (want > cap) want = cap;
        if (want > chunks) chunks = want;
    }
    int bn = ((n_padded + chunks - 1) / chunks + 15) & ~15;
    return bn;
}

static inline int conv_out(int i, int k, int s, int p, int d) { return (i + 2 * p - (d * (k - 1) + 1)) / s + 1; }

// =================================================================================================
// Int8 Conv2D
// =================================================================================================
// How a resized conv runs, decided once at resize (conv_plan): the kernels that take it and, where the conv-group kernel does,
// its layer there -- everything but the x / y pointers, which bind (group_build) adds.
struct ConvPlan {
    bool gemm = false;    // 1x1, stride 1, no pad: mode 0 on the conv-group kernel
    bool stem = false;    // <= 4 input channels: the dp4a stem kernel
    bool group = false;   // the conv-group kernel takes it: q / g / tmap_b hold the layer and the schedule word can address it
    GroupLayerParams q;   // y = nullptr
    GroupConvGeom g;      // mode 1 only; hcls / wcls / corr point into the execution's d_border
    CUtensorMap tmap_b;   // weights, boxes of q.cb bytes x q.bn rows
};
enum class ConvPath { Stem, Group, MmaSync, Refused };
// variant (mnnb200_conv_int8_set_variant): 0 auto, 1 mma.sync, 2 wgmma -- Refused when the conv-group kernel does not take the conv
static ConvPath conv_path(const ConvPlan& c, int variant) {
    if (variant == 1) return ConvPath::MmaSync;
    // first-layer convs (<= 4 input channels, not GEMM-shaped): the dp4a kernel beats the implicit GEMM, whose K would be 13/16
    // padding.  Inside a group they also keep the single-thread TMA producers of every CTA busy and slow the whole group down
    // (measured on MobileNet-v2 B=32: 0.31 ms with the stem inside the group, 0.19 ms with it outside).
    if (variant == 0 && c.stem && !c.gemm) return ConvPath::Stem;
    // wgmma on the conv-group kernel, alone as a one-layer group or as a member of a larger one; mma.sync takes what that
    // kernel does not (stride_w > 2, the largest feature maps)
    if (c.group) return ConvPath::Group;
    return variant == 0 ? ConvPath::MmaSync : ConvPath::Refused;
}

struct ConvInt8Exec : mnnb200_exec {
    mnnb200_conv_desc d;
    bool legacy = false;
    int Cp = 0, OCp = 0, kernel_len = 0;
    std::vector<float> h_wscale, h_bias;   // modern: alpha + float bias; legacy: fused scale
    std::vector<int32_t> h_bias_i32;       // legacy
    std::vector<int32_t> h_isum;           // sum_k w[oc][k]
    std::vector<int32_t> h_tapsum;         // [OCp][taps] sum_c w[oc][tap][c]: padding correction of the implicit-GEMM kernel
    ConvPlan plan;
    int32_t* d_border = nullptr;           // border-class tables of plan.g, grow-only
    size_t border_cap = 0;
    struct GroupState* solo = nullptr;     // this layer alone on the conv-group kernel
    const void* solo_x = nullptr;
    const void* solo_y = nullptr;
    ~ConvInt8Exec() override;
    int8_t* d_w = nullptr;
    int8_t* d_wg = nullptr;                // the conv-group kernel's copy: [n_chunks * bn][taps * Cp], rows permuted per chunk
    float* d_ep = nullptr;                 // its epilogue table (GroupLayerParams::ep), grow-only
    size_t ep_cap = 0;
    float *d_wscale = nullptr, *d_bias = nullptr;
    int32_t* d_wsum128 = nullptr;
    ConvParams p;
    int tile = TILE_128x64;
    bool resized = false;
};

// the conv-group kernel's tile width for OCp output channels: equal n chunks of at most kGroupMaxBN columns
static int group_bn(int OCp) {
    const int chunks = (OCp + kGroupMaxBN - 1) / kGroupMaxBN;
    return ((OCp + chunks - 1) / chunks + 15) & ~15;
}

static mnnb200_status conv_create_common(mnnb200_runtime* rt, const mnnb200_conv_desc* desc, const int8_t* weight,
                                         ConvInt8Exec* e) {
    e->rt = rt;
    e->kind = 1;
    e->d = *desc;
    const auto& d = e->d;
    if (d.group != 1) return fail(MNNB200_NOT_SUPPORT, "conv_int8: group != 1 (use dwconv for depthwise)");
    if (d.ic <= 0 || d.oc <= 0 || d.kh <= 0 || d.kw <= 0 || d.stride_h <= 0 || d.stride_w <= 0 || d.dilate_h <= 0 ||
        d.dilate_w <= 0)
        return fail(MNNB200_INVALID_VALUE, "conv_int8: bad descriptor");
    e->Cp = up16(d.ic);
    e->OCp = up16(d.oc);
    e->kernel_len = d.ic * d.kh * d.kw;
    const int taps = d.kh * d.kw;
    // pack [oc][ic][kh][kw] -> [OCp][tap][Cp]  (WeightInt8PackFill's job, ConvInt8CutlassExecution.cu:70-105)
    std::vector<int8_t> wp((size_t)e->OCp * taps * e->Cp, 0);
    e->h_isum.assign(e->OCp, 0);
    e->h_tapsum.assign((size_t)e->OCp * taps, 0);
    for (int o = 0; o < d.oc; ++o) {
        int32_t s = 0;
        for (int c = 0; c < d.ic; ++c)
            for (int t = 0; t < taps; ++t) {
                int8_t v = weight[((size_t)o * d.ic + c) * taps + t];
                wp[((size_t)o * taps + t) * e->Cp + c] = v;
                s += v;
                e->h_tapsum[(size_t)o * taps + t] += v;
            }
        e->h_isum[o] = s;
    }
    mnnb200_status st = e->upload(wp, &e->d_w);
    if (st) return st;
    {   // the conv-group kernel's weights: GEMM column c of chunk nc is channel nc * bn + group_column_channel(c, bn)
        const int bn = group_bn(e->OCp), n_chunks = (e->OCp + bn - 1) / bn;
        const size_t row = (size_t)taps * e->Cp;
        std::vector<int8_t> wg((size_t)n_chunks * bn * row, 0);
        for (int nc = 0; nc < n_chunks; ++nc)
            for (int c = 0; c < bn; ++c) {
                const int o = nc * bn + group_column_channel(c, bn);
                if (o < e->OCp) memcpy(&wg[((size_t)nc * bn + c) * row], &wp[(size_t)o * row], row);
            }
        if ((st = e->upload(wg, &e->d_wg))) return st;
    }
    std::vector<float> z(e->OCp, 0.f);
    std::vector<int32_t> zi(e->OCp, 0);
    if ((st = e->upload(z, &e->d_wscale))) return st;
    if ((st = e->upload(z, &e->d_bias))) return st;
    if ((st = e->upload(zi, &e->d_wsum128))) return st;
    return MNNB200_OK;
}

// ---- conv group: one persistent launch over a list of convolutions (conv_group_wgmma.cu) ----------------------------
struct GroupState {
    mnnb200_runtime* rt = nullptr;
    GroupMapsParam* h_maps = nullptr;       // host: passed by value as the kernel's __grid_constant__ parameter
    GroupLayerParams* d_params = nullptr;
    GroupConvGeom* d_geom = nullptr;
    uint32_t* d_sched = nullptr;
    size_t sched_cap = 0;
    int n_layers = 0, sched_stride = 0, grid = 0;
    ~GroupState() {
        delete h_maps;
        if (d_params) cudaFree(d_params);
        if (d_geom) cudaFree(d_geom);
        if (d_sched) cudaFree(d_sched);
    }
};
ConvInt8Exec::~ConvInt8Exec() { delete solo; }

// Builds the conv's plan: which kernels take it and, for the conv-group kernel, its layer without the x / y pointers.  Every
// limit of that kernel and of its schedule word is checked here; a layer outside them is not taken (plan.group = false).
static mnnb200_status conv_plan(ConvInt8Exec* e, int zin, const std::vector<float>& ws, const std::vector<float>& bf,
                                const std::vector<int32_t>& k128) {
    const ConvParams& p = e->p;
    const auto& d = e->d;
    ConvPlan& plan = e->plan;
    plan.gemm = d.kh == 1 && d.kw == 1 && d.stride_h == 1 && d.stride_w == 1 && d.pad_h == 0 && d.pad_w == 0;
    plan.stem = conv_int8_stem_supported(p, d.ic);
    plan.group = false;
    if (!plan.gemm && (p.sw > 2 || p.KH > 32 || p.KW > 32 || (p.sw == 2 && p.IW < 2))) return MNNB200_OK;
    GroupLayerParams& q = plan.q;
    GroupConvGeom& g = plan.g;
    memset(&q, 0, sizeof(q));
    memset(&g, 0, sizeof(g));
    q.bn = group_bn(e->OCp);
    q.n_chunks = (e->OCp + q.bn - 1) / q.bn;
    // GEMM column c of chunk nc -> output channel (group_column_channel), and whether it is one of the layer's OC
    auto channel = [&](int nc, int c) { return nc * q.bn + group_column_channel(c, q.bn); };
    const int ncol = q.n_chunks * q.bn;
    q.M = p.M; q.N = e->OCp; q.OC = d.oc;
    q.ldy = e->OCp; q.scale_x = p.scale_x; q.minv = p.minv; q.maxv = p.maxv;
    q.mode = plan.gemm ? 0 : 1;
    const int taps = p.KH * p.KW;
    if (plan.gemm) {
        q.K = e->Cp; q.cb = 128; q.TWp = 128; q.R = 1;
        q.m_tiles = (p.M + 127) / 128; q.num_kb = (e->Cp + 127) / 128;
    } else {
        g.KH = p.KH; g.KW = p.KW; g.Cp = e->Cp; g.NB = p.N;
        g.sh = p.sh; g.sw = p.sw; g.ph = p.ph; g.pw = p.pw; g.dh = p.dh; g.dw = p.dw; g.OH = p.OH; g.OW = p.OW;
        g.SEG = (p.OW + 127) / 128;
        q.TWp = (((p.OW + g.SEG - 1) / g.SEG) + 7) & ~7;
        // a TMA box = BH consecutive output rows of one image when stride_h == 1 (their input rows are consecutive too): BH = the
        // largest divisor of OH with BH * TWp <= 128; R = boxes per M tile.  One box per row needed up to 16 TMA issues per K block
        // and made the single-thread producer the limiter on small feature maps (ResNet 7x7 / 14x14).
        g.BH = 1;
        if (p.sh == 1) for (int bh = 1; bh <= p.OH && bh * q.TWp <= 128; ++bh) if (p.OH % bh == 0) g.BH = bh;
        g.OHB = p.OH / g.BH;
        q.R = std::max(1, std::min(16, 128 / (g.BH * q.TWp)));
        g.rowboxes = p.N * g.OHB * g.SEG;
        q.m_tiles = (g.rowboxes + q.R - 1) / q.R;
        q.cb = (e->Cp % 128 == 0) ? 128 : ((e->Cp % 64 == 0) ? 64 : 16);
        g.cpt = e->Cp / q.cb;
        g.chunks = taps * g.cpt;
        if (q.cb == 16 && (g.chunks & 1)) ++g.chunks;            // one all-zero chunk: an MMA eats 2 x 16 bytes of K
        q.num_kb = q.cb >= 64 ? g.chunks : (g.chunks + 7) / 8;
        q.K = q.cb == 16 ? 16 * g.chunks : taps * e->Cp;
    }
    if (q.n_chunks > kGroupMaxNChunks || q.m_tiles > kGroupMaxMTiles) return MNNB200_OK;
    mnnb200_status st;
    {   // B: the permuted copy [n_chunks * bn][taps * Cp], chunk-wide boxes of bn rows
        cuuint64_t dims[2] = {(cuuint64_t)taps * e->Cp, (cuuint64_t)ncol};
        cuuint64_t strides[1] = {(cuuint64_t)taps * e->Cp};
        cuuint32_t box[2] = {(cuuint32_t)q.cb, (cuuint32_t)q.bn};
        if ((st = make_tmap_u8(&plan.tmap_b, e->d_wg, 2, dims, strides, box))) return st;
    }
    {   // epilogue table [n_chunks][3][bn]: wscale, biasFloat, preset = 128 sum w (+ 0x4B400000 for requant_fast_small)
        const int32_t magic = q.K <= 128 ? 0x4B400000 : 0;
        std::vector<float> ep((size_t)3 * ncol, 0.f);
        for (int nc = 0; nc < q.n_chunks; ++nc)
            for (int c = 0; c < q.bn; ++c) {
                const int o = channel(nc, c);
                if (o >= d.oc) continue;
                float* row = &ep[(size_t)nc * 3 * q.bn];
                row[c] = ws[o];
                row[q.bn + c] = bf[o];
                const int32_t pre = (int32_t)((uint32_t)k128[o] + (uint32_t)magic);
                memcpy(&row[2 * q.bn + c], &pre, 4);
            }
        if ((st = e->grow_scratch((void**)&e->d_ep, &e->ep_cap, ep.size() * 4))) return st;
        if ((st = e->update(ep, e->d_ep))) return st;
        q.ep = e->d_ep;
    }
    // padding correction (input zero point != 0): the reference fills padded taps with z_in (ConvInt8TiledExecutor.cpp:2269-2271),
    // the TMA unit fills zeros -> add z_in * sum_{out-of-image taps} sum_c w[oc][tap][c] per border class
    if (!plan.gemm && zin != 0) {
        std::vector<uint32_t> hu, wu;
        auto cls_of = [](std::vector<uint32_t>& uniq, uint32_t m) {
            for (size_t i = 0; i < uniq.size(); ++i) if (uniq[i] == m) return (int)i;
            uniq.push_back(m);
            return (int)uniq.size() - 1;
        };
        std::vector<uint8_t> hc(p.OH), wc(p.OW);
        bool ok = true;
        for (int oh = 0; oh < p.OH && ok; ++oh) {
            uint32_t m = 0;
            for (int kh = 0; kh < p.KH; ++kh) { int ih = oh * p.sh - p.ph + kh * p.dh; if (ih >= 0 && ih < p.IH) m |= 1u << kh; }
            int c = cls_of(hu, m); ok = c < 255; hc[oh] = (uint8_t)c;
        }
        for (int ow = 0; ow < p.OW && ok; ++ow) {
            uint32_t m = 0;
            for (int kw = 0; kw < p.KW; ++kw) { int iw = ow * p.sw - p.pw + kw * p.dw; if (iw >= 0 && iw < p.IW) m |= 1u << kw; }
            int c = cls_of(wu, m); ok = c < 255; wc[ow] = (uint8_t)c;
        }
        if (!ok) return MNNB200_OK;   // too many border classes for the byte-wide class tables
        const uint32_t fullh = p.KH >= 32 ? 0xffffffffu : ((1u << p.KH) - 1), fullw = p.KW >= 32 ? 0xffffffffu : ((1u << p.KW) - 1);
        bool any_border = false;
        for (uint32_t m : hu) any_border |= m != fullh;
        for (uint32_t m : wu) any_border |= m != fullw;
        if (any_border) {
            // one buffer: corr [HC * WC][n_chunks * bn] in GEMM-column order, then hcls [OH] and wcls [OW] bytes
            const int HC = (int)hu.size(), WC = (int)wu.size();
            const size_t ncorr = (size_t)HC * WC * ncol;
            std::vector<int32_t> tab(ncorr + (p.OH + p.OW + 3) / 4, 0);
            g.interior_cls = -1;
            for (int a = 0; a < HC; ++a)
                for (int b = 0; b < WC; ++b) {
                    if (hu[a] == fullh && wu[b] == fullw) { g.interior_cls = a * WC + b; continue; }
                    for (int col = 0; col < ncol; ++col) {
                        const int o = channel(col / q.bn, col % q.bn);
                        if (o >= d.oc) continue;
                        int32_t sum = 0;
                        for (int kh = 0; kh < p.KH; ++kh)
                            for (int kw = 0; kw < p.KW; ++kw)
                                if (!((hu[a] >> kh) & 1u) || !((wu[b] >> kw) & 1u)) sum += e->h_tapsum[(size_t)o * taps + kh * p.KW + kw];
                        tab[((size_t)a * WC + b) * ncol + col] = zin * sum;
                    }
                }
            memcpy(tab.data() + ncorr, hc.data(), p.OH);
            memcpy((uint8_t*)(tab.data() + ncorr) + p.OH, wc.data(), p.OW);
            if ((st = e->grow_scratch((void**)&e->d_border, &e->border_cap, tab.size() * 4))) return st;
            if ((st = e->update(tab, e->d_border))) return st;
            g.corr = e->d_border;
            g.hcls = (const uint8_t*)(e->d_border + ncorr);
            g.wcls = g.hcls + p.OH;
            g.wc_count = WC;
        }
    }
    plan.group = true;
    return MNNB200_OK;
}

// Binds planned convs to their activations: the A tensor maps, the y pointers and the schedule.
static mnnb200_status group_build(GroupState& gs, const std::vector<ConvInt8Exec*>& members, const int8_t* const* xs,
                                  int8_t* const* ys, double* cost_bytes, double* cost_macs) {
    mnnb200_runtime* rt = gs.rt;
    const int L = (int)members.size();
    CK(cudaSetDevice(rt->device));
    if (!gs.h_maps) { gs.h_maps = new GroupMapsParam; memset(gs.h_maps, 0, sizeof(GroupMapsParam)); }
    if (!gs.d_params) CK(cudaMalloc((void**)&gs.d_params, sizeof(GroupLayerParams) * kGroupMaxLayers));
    if (!gs.d_geom) CK(cudaMalloc((void**)&gs.d_geom, sizeof(GroupConvGeom) * kGroupMaxLayers));
    static_assert(sizeof(CUtensorMap) == sizeof(CUtensorMap_st_opaque), "tensor map size");
    std::vector<GroupLayerParams> prm(L);
    std::vector<GroupConvGeom> geo(L);
    std::vector<uint32_t> items;
    if (cost_bytes) *cost_bytes = 0;
    if (cost_macs) *cost_macs = 0;
    mnnb200_status st;
    for (int l = 0; l < L; ++l) {
        const ConvInt8Exec* e = members[l];
        if (!e->resized || !e->plan.group) return fail(MNNB200_NOT_SUPPORT, "conv group: a member is not a resized conv the wgmma group kernel takes");
        const ConvParams& p = e->p;
        const GroupLayerParams& q = e->plan.q;
        if ((uintptr_t)ys[l] % 8) return fail(MNNB200_INVALID_VALUE, "conv group: an output is not 8-byte aligned");
        prm[l] = q;
        prm[l].y = ys[l];
        geo[l] = e->plan.g;
        CUtensorMap* ta = reinterpret_cast<CUtensorMap*>(&gs.h_maps->a[l]);
        CUtensorMap* ta1 = reinterpret_cast<CUtensorMap*>(&gs.h_maps->a1[l]);
        memcpy(&gs.h_maps->b[l], &e->plan.tmap_b, sizeof(CUtensorMap));
        if (q.mode == 0) {
            if ((st = make_tmap_i8(ta, xs[l], p.M, e->Cp, 128))) return st;
        } else {
            // A: one 4D {C, W', H, N} view of the NHWC16 input per column parity (W' = every sw-th column)
            for (int par = 0; par < p.sw; ++par) {
                cuuint64_t dims[4] = {(cuuint64_t)e->Cp, (cuuint64_t)((p.IW - par + p.sw - 1) / p.sw), (cuuint64_t)p.IH, (cuuint64_t)p.N};
                cuuint64_t strides[3] = {(cuuint64_t)p.sw * e->Cp, (cuuint64_t)p.IW * e->Cp, (cuuint64_t)p.IH * p.IW * e->Cp};
                cuuint32_t box[4] = {(cuuint32_t)q.cb, (cuuint32_t)q.TWp, (cuuint32_t)e->plan.g.BH, 1u};
                if ((st = make_tmap_u8(par ? ta1 : ta, xs[l] + (size_t)par * e->Cp, 4, dims, strides, box))) return st;
            }
        }
        if (p.sw == 1) *ta1 = *ta;
        if (cost_bytes) *cost_bytes += e->cost_bytes;
        if (cost_macs) *cost_macs += e->cost_macs;
        // an item = ONE M tile of one n chunk: measured on MobileNet-v2 B=32, 1 tile per item is best (0.184 ms; 2: 0.186, 8: 0.192)
        for (int mt = 0; mt < q.m_tiles; ++mt)
            for (int nc = 0; nc < q.n_chunks; ++nc)
                items.push_back(((uint32_t)l << kGroupItemLayerShift) | ((uint32_t)nc << kGroupItemChunkShift) | (uint32_t)mt);
    }
    // round-robin, item i -> CTA i mod grid: every CTA gets the same mix of layers, so the balance needs no cost model
    // (measured on MobileNet-v2 B=32: 0.28 ms against 0.81 ms for a contiguous cost-balanced partition).
    // Every role of a CTA walks its whole row up to the first terminator.  The row keeps a second one so that a walk over
    // alternate items (i = g, g + 2, ..., one per consumer warpgroup) would also meet an end marker inside the row.
    const int grid = (int)std::min<size_t>(items.size(), (size_t)rt->prop.multiProcessorCount);
    const size_t stride = (items.size() + grid - 1) / grid + 2;
    std::vector<uint32_t> sched(stride * grid, kGroupSchedEnd);
    for (size_t i = 0; i < items.size(); ++i) sched[(i % grid) * stride + i / grid] = items[i];
    if (sched.size() > gs.sched_cap) {
        if (gs.d_sched) cudaFree(gs.d_sched);
        gs.d_sched = nullptr;
        CK(cudaMalloc((void**)&gs.d_sched, sched.size() * 4));
        gs.sched_cap = sched.size();
    }
    CK(cudaMemcpy(gs.d_params, prm.data(), sizeof(GroupLayerParams) * L, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(gs.d_geom, geo.data(), sizeof(GroupConvGeom) * L, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(gs.d_sched, sched.data(), sched.size() * 4, cudaMemcpyHostToDevice));
    gs.sched_stride = (int)stride;
    gs.grid = grid;
    gs.n_layers = L;
    return MNNB200_OK;
}
static mnnb200_status group_launch(const GroupState& gs) {
    CK(launch_conv_group(gs.h_maps, gs.d_params, gs.d_geom, gs.n_layers, gs.d_sched, gs.sched_stride, gs.grid, gs.rt->stream));
    return MNNB200_OK;
}

static int pick_tile(int M, int OCp, int sm_count) {
    int bn = OCp <= 16 ? 16 : (OCp <= 32 ? 32 : 64);
    if (OCp >= 256 && M >= 128 * sm_count) bn = 128;
    int bm = 128;
    long ctas = (long)((M + 127) / 128) * ((OCp + bn - 1) / bn);
    if (bn >= 32 && bn <= 64 && ctas < 2L * sm_count) bm = 64;
    if (bm == 128) return bn == 16 ? TILE_128x16 : bn == 32 ? TILE_128x32 : bn == 64 ? TILE_128x64 : TILE_128x128;
    return bn == 32 ? TILE_64x32 : TILE_64x64;
}

extern "C" {

const char* mnnb200_last_error(void) { return g_err.c_str(); }
int mnnb200_abi_version(void) { return 2; }
unsigned long long mnnb200_launch_count(void) { return g_launch_count.load(); }
size_t mnnb200_nhwc16_bytes(int n, int c, int h, int w) { return (size_t)n * h * w * up16(c); }

mnnb200_status mnnb200_runtime_create(int device_id, void* stream, mnnb200_runtime** out) {
    if (!out) return fail(MNNB200_INVALID_VALUE, "runtime_create: out == NULL");
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0)
        return fail(MNNB200_CUDA_ERROR, std::string("no CUDA device (there is no CPU fallback): ") + cudaGetErrorString(e));
    if (device_id < 0 || device_id >= count) return fail(MNNB200_INVALID_VALUE, "runtime_create: bad device id");
    CK(cudaSetDevice(device_id));
    auto* rt = new mnnb200_runtime;
    rt->device = device_id;
    CK(cudaGetDeviceProperties(&rt->prop, device_id));
    if (rt->prop.major != 9) {
        delete rt;
        return fail(MNNB200_NOT_SUPPORT, "mnn_b200 is built for sm_90a (H100) only");
    }
    if (stream) {
        rt->stream = (cudaStream_t)stream;
    } else {
        CK(cudaStreamCreateWithFlags(&rt->stream, cudaStreamNonBlocking));
        rt->own_stream = true;
    }
    *out = rt;
    return MNNB200_OK;
}
void mnnb200_runtime_destroy(mnnb200_runtime* rt) {
    if (!rt) return;
    if (rt->ev_begin) cudaEventDestroy(rt->ev_begin);
    if (rt->ev_end) cudaEventDestroy(rt->ev_end);
    if (rt->own_stream) cudaStreamDestroy(rt->stream);
    delete rt;
}
void* mnnb200_runtime_stream(mnnb200_runtime* rt) { return rt ? (void*)rt->stream : nullptr; }
mnnb200_status mnnb200_runtime_sync(mnnb200_runtime* rt) {
    CK(cudaStreamSynchronize(rt->stream));
    return MNNB200_OK;
}
mnnb200_status mnnb200_runtime_info(mnnb200_runtime* rt, int* sm_count, int* cc_major, int* cc_minor, size_t* total_mem) {
    if (sm_count) *sm_count = rt->prop.multiProcessorCount;
    if (cc_major) *cc_major = rt->prop.major;
    if (cc_minor) *cc_minor = rt->prop.minor;
    if (total_mem) *total_mem = rt->prop.totalGlobalMem;
    return MNNB200_OK;
}
mnnb200_status mnnb200_alloc(mnnb200_runtime* rt, size_t bytes, void** dev_ptr) {
    CK(cudaSetDevice(rt->device));
    CK(cudaMalloc(dev_ptr, bytes ? bytes : 16));
    return MNNB200_OK;
}
mnnb200_status mnnb200_free(mnnb200_runtime* rt, void* dev_ptr) {
    (void)rt;
    CK(cudaFree(dev_ptr));
    return MNNB200_OK;
}
mnnb200_status mnnb200_memcpy_h2d(mnnb200_runtime* rt, void* dst, const void* src, size_t bytes) {
    CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, rt->stream));
    return MNNB200_OK;
}
mnnb200_status mnnb200_memcpy_d2h(mnnb200_runtime* rt, void* dst, const void* src, size_t bytes) {
    CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, rt->stream));
    return MNNB200_OK;
}

// ---- whole-forward graph, pinned host staging, GPU timing -----------------------------------------------------------
mnnb200_status mnnb200_graph_begin_capture(mnnb200_runtime* rt) {
    if (!rt) return fail(MNNB200_INVALID_VALUE, "graph_begin_capture: NULL runtime");
    CK(cudaSetDevice(rt->device));
    CK(cudaStreamBeginCapture(rt->stream, cudaStreamCaptureModeThreadLocal));
    return MNNB200_OK;
}
mnnb200_status mnnb200_graph_end_capture(mnnb200_runtime* rt, mnnb200_graph** out) {
    if (!rt || !out) return fail(MNNB200_INVALID_VALUE, "graph_end_capture: NULL argument");
    cudaGraph_t g = nullptr;
    cudaError_t e = cudaStreamEndCapture(rt->stream, &g);
    if (e != cudaSuccess || !g) {
        cudaGetLastError();
        return fail(MNNB200_CUDA_ERROR, std::string("cudaStreamEndCapture: ") + cudaGetErrorString(e));
    }
    cudaGraphExec_t x = nullptr;
    e = cudaGraphInstantiate(&x, g, 0);
    if (e != cudaSuccess) {
        cudaGraphDestroy(g);
        return fail(MNNB200_CUDA_ERROR, std::string("cudaGraphInstantiate: ") + cudaGetErrorString(e));
    }
    auto* h = new mnnb200_graph;
    h->graph = g; h->exec = x;
    *out = h;
    return MNNB200_OK;
}
mnnb200_status mnnb200_graph_launch(mnnb200_runtime* rt, mnnb200_graph* g) {
    if (!rt || !g || !g->exec) return fail(MNNB200_INVALID_VALUE, "graph_launch: NULL argument");
    CK(cudaGraphLaunch(g->exec, rt->stream));
    return MNNB200_OK;
}
void mnnb200_graph_destroy(mnnb200_graph* g) {
    if (!g) return;
    if (g->exec) cudaGraphExecDestroy(g->exec);
    if (g->graph) cudaGraphDestroy(g->graph);
    delete g;
}
mnnb200_status mnnb200_host_register(mnnb200_runtime* rt, void* p, size_t bytes) {
    if (!rt || !p || !bytes) return fail(MNNB200_INVALID_VALUE, "host_register: bad argument");
    cudaError_t e = cudaHostRegister(p, bytes, cudaHostRegisterDefault);
    if (e == cudaErrorHostMemoryAlreadyRegistered) { cudaGetLastError(); return MNNB200_OK; }
    if (e != cudaSuccess) { cudaGetLastError(); return fail(MNNB200_NOT_SUPPORT, std::string("cudaHostRegister: ") + cudaGetErrorString(e)); }
    return MNNB200_OK;
}
mnnb200_status mnnb200_host_unregister(mnnb200_runtime* rt, void* p) {
    (void)rt;
    cudaError_t e = cudaHostUnregister(p);
    if (e != cudaSuccess) { cudaGetLastError(); return fail(MNNB200_INVALID_VALUE, std::string("cudaHostUnregister: ") + cudaGetErrorString(e)); }
    return MNNB200_OK;
}
mnnb200_status mnnb200_alloc_host(mnnb200_runtime* rt, size_t bytes, void** p) {
    if (!rt || !p) return fail(MNNB200_INVALID_VALUE, "alloc_host: NULL argument");
    CK(cudaSetDevice(rt->device));
    CK(cudaHostAlloc(p, bytes ? bytes : 16, cudaHostAllocDefault));
    return MNNB200_OK;
}
mnnb200_status mnnb200_free_host(mnnb200_runtime* rt, void* p) {
    (void)rt;
    CK(cudaFreeHost(p));
    return MNNB200_OK;
}
mnnb200_status mnnb200_runtime_mark_begin(mnnb200_runtime* rt) {
    if (!rt) return fail(MNNB200_INVALID_VALUE, "mark_begin: NULL runtime");
    if (!rt->ev_begin) { CK(cudaEventCreate(&rt->ev_begin)); CK(cudaEventCreate(&rt->ev_end)); }
    rt->ev_valid = false;
    CK(cudaEventRecord(rt->ev_begin, rt->stream));
    return MNNB200_OK;
}
mnnb200_status mnnb200_runtime_mark_end(mnnb200_runtime* rt) {
    if (!rt || !rt->ev_begin) return fail(MNNB200_INVALID_VALUE, "mark_end without mark_begin");
    CK(cudaEventRecord(rt->ev_end, rt->stream));
    rt->ev_valid = true;
    return MNNB200_OK;
}
float mnnb200_runtime_last_gpu_ms(mnnb200_runtime* rt) {
    if (!rt || !rt->ev_valid) return -1.0f;
    float ms = -1.0f;
    if (cudaEventSynchronize(rt->ev_end) != cudaSuccess || cudaEventElapsedTime(&ms, rt->ev_begin, rt->ev_end) != cudaSuccess) {
        cudaGetLastError();
        return -1.0f;
    }
    return ms;
}

// ---- casts ---------------------------------------------------------------------------------------
mnnb200_status mnnb200_float_to_int8(mnnb200_runtime* rt, const float* x, int n, int c, int h, int w, float scale,
                                     float zero, int min_v, int max_v, int8_t* y) {
    float inv = scale == 0.f ? 0.f : 1.f / scale;  // CPUCast.cpp:24
    CK(launch_float_to_int8(x, n, c, h, w, inv, zero, (float)min_v, (float)max_v, y, rt->stream));
    return MNNB200_OK;
}
mnnb200_status mnnb200_int8_to_float(mnnb200_runtime* rt, const int8_t* x, int n, int c, int h, int w, float scale,
                                     float zero, float* y) {
    CK(launch_int8_to_float(x, n, c, h, w, scale, zero, y, rt->stream));
    return MNNB200_OK;
}
mnnb200_status mnnb200_pack_nchw_int8(mnnb200_runtime* rt, const int8_t* x, int n, int c, int h, int w, int8_t* y) {
    CK(launch_pack_nchw_int8(x, n, c, h, w, y, rt->stream));
    return MNNB200_OK;
}
mnnb200_status mnnb200_unpack_nchw_int8(mnnb200_runtime* rt, const int8_t* x, int n, int c, int h, int w, int8_t* y) {
    CK(launch_unpack_nchw_int8(x, n, c, h, w, y, rt->stream));
    return MNNB200_OK;
}

// ---- int8 neighbours -------------------------------------------------------------------------------
mnnb200_status mnnb200_binary_add_int8(mnnb200_runtime* rt, const int8_t* x0, float s0, int z0, const int8_t* x1, float s1,
                                       int z1, int8_t* y, float s_out, int z_out, int min_v, int max_v, int n, int c, int h,
                                       int w) {
    float inv = s_out != 0 ? 1 / s_out : 0;   // CPUBinaryInt8.cpp:37-41
    CK(launch_binary_add_int8(x0, s0, z0, x1, s1, z1, y, inv, z_out, min_v, max_v, (size_t)n * h * w, c, up16(c), rt->stream));
    return MNNB200_OK;
}
mnnb200_status mnnb200_avgpool_int8(mnnb200_runtime* rt, const int8_t* x, int n, int c, int ih, int iw, int kh, int kw,
                                    int stride_h, int stride_w, int pad_h, int pad_w, int pad_type, int count_type, float s_in,
                                    float z_in, float s_out, float z_out, int min_v, int max_v, int8_t* y, int oh, int ow) {
    PoolParams p;
    p.x = x; p.y = y; p.N = n; p.C = c; p.Cp = up16(c); p.IH = ih; p.IW = iw; p.OH = oh; p.OW = ow; p.KH = kh; p.KW = kw;
    p.sh = stride_h; p.sw = stride_w; p.ph = pad_h; p.pw = pad_w;
    p.count_type = count_type == 0 ? (pad_type == 0 ? 1 : 2) : count_type;   // CPUPool.hpp:239-245
    p.s_in = s_in; p.z_in = z_in; p.inv_out = s_out == 0.f ? 0.f : 1.f / s_out; p.z_out = z_out;
    p.minv = (float)min_v; p.maxv = (float)max_v;
    CK(launch_avgpool_int8_via_float(p, rt->stream));
    return MNNB200_OK;
}
mnnb200_status mnnb200_pool_f32(mnnb200_runtime* rt, const float* x, int n, int c, int ih, int iw, int kh, int kw, int stride_h,
                                int stride_w, int pad_h, int pad_w, int pad_type, int count_type, int is_avg, float* y, int oh,
                                int ow) {
    PoolParams p;
    memset(&p, 0, sizeof(p));
    p.N = n; p.C = c; p.Cp = c; p.IH = ih; p.IW = iw; p.OH = oh; p.OW = ow; p.KH = kh; p.KW = kw;
    p.sh = stride_h; p.sw = stride_w; p.ph = pad_h; p.pw = pad_w;
    p.count_type = count_type == 0 ? (pad_type == 0 ? 1 : 2) : count_type;   // CPUPool.hpp:239-245
    CK(launch_pool_f32(p, x, y, is_avg, rt->stream));
    return MNNB200_OK;
}
mnnb200_status mnnb200_raster_b32(mnnb200_runtime* rt, const mnnb200_region* regions, int count, void* dst, size_t dst_bytes,
                                  int zero_fill) {
    if (!rt || (!regions && count) || !dst) return fail(MNNB200_INVALID_VALUE, "raster_b32: NULL argument");
    if (zero_fill) CK(cudaMemsetAsync(dst, 0, dst_bytes, rt->stream));
    for (int i = 0; i < count; ++i) {
        RasterRegion r;
        r.src_offset = regions[i].src_offset; r.dst_offset = regions[i].dst_offset;
        for (int k = 0; k < 3; ++k) { r.src_stride[k] = regions[i].src_stride[k]; r.dst_stride[k] = regions[i].dst_stride[k]; r.size[k] = regions[i].size[k]; }
        CK(launch_raster_b32(r, regions[i].src, dst, rt->stream));
    }
    return MNNB200_OK;
}
mnnb200_status mnnb200_transpose_b32(mnnb200_runtime* rt, const void* src, int batch, int rows, int cols, void* dst) {
    if (!rt || !src || !dst || batch <= 0 || rows <= 0 || cols <= 0) return fail(MNNB200_INVALID_VALUE, "transpose_b32: bad argument");
    CK(launch_transpose_b32(src, dst, batch, rows, cols, rt->stream));
    return MNNB200_OK;
}
mnnb200_status mnnb200_memcpy_d2d(mnnb200_runtime* rt, void* dst, const void* src, size_t bytes) {
    CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, rt->stream));
    return MNNB200_OK;
}
// ---- ResNet-50 neighbours: int8 Scale, int8 pooling (equal attrs), float ReLU / Reduction ----------------------------------
struct ScaleInt8Exec : mnnb200_exec {
    int c = 0, cp = 0;
    std::vector<float> h_scale, h_bias;
    int32_t *d_alpha = nullptr, *d_bias = nullptr;
    int zin = 0, zout = 0, minv = -127, maxv = 127;
    bool resized = false;
};
mnnb200_status mnnb200_scale_int8_create(mnnb200_runtime* rt, int channels, const float* scale, const float* bias, mnnb200_exec** out) {
    if (!rt || !scale || !out || channels <= 0) return fail(MNNB200_INVALID_VALUE, "scale_int8_create: bad argument");
    auto* e = new ScaleInt8Exec;
    e->rt = rt; e->kind = 7; e->c = channels; e->cp = up16(channels);
    e->h_scale.assign(scale, scale + channels);
    e->h_bias.assign(channels, 0.f);
    if (bias) e->h_bias.assign(bias, bias + channels);
    std::vector<int32_t> z(e->cp, 0);
    mnnb200_status st;
    if ((st = e->upload(z, &e->d_alpha)) || (st = e->upload(z, &e->d_bias))) { delete e; return st; }
    *out = e;
    return MNNB200_OK;
}
mnnb200_status mnnb200_scale_int8_resize(mnnb200_exec* ex, float in_scale, int in_zero, float out_scale, int out_zero, int clamp_min,
                                         int clamp_max) {
    if (!ex || ex->kind != 7) return fail(MNNB200_INVALID_VALUE, "scale_int8_resize: not a Scale execution");
    auto* e = static_cast<ScaleInt8Exec*>(ex);
    // CPUScaleInt8::onResize (CPUScaleInt8.cpp:60-90): 15-bit fixed point, float products left to right, roundf
    const float inv_out = out_scale == 0.f ? 0.f : 1.f / out_scale;
    std::vector<int32_t> al(e->cp, 0), bi(e->cp, 0);
    for (int i = 0; i < e->c; ++i) {
        float t = e->h_scale[i] * in_scale;
        t = t * inv_out;
        t = t * (float)(1 << 15);
        al[i] = (int32_t)roundf(t);
        float b = e->h_bias[i] * inv_out;
        b = b * (float)(1 << 15);
        bi[i] = (int32_t)roundf(b);
    }
    mnnb200_status st;
    if ((st = e->update(al, e->d_alpha)) || (st = e->update(bi, e->d_bias))) return st;
    e->zin = (int)(int8_t)in_zero; e->zout = (int)(int8_t)out_zero; e->minv = clamp_min; e->maxv = clamp_max;
    e->resized = true;
    return MNNB200_OK;
}
mnnb200_status mnnb200_scale_int8_execute(mnnb200_exec* ex, const int8_t* x, int n, int h, int w, int8_t* y) {
    if (!ex || ex->kind != 7) return fail(MNNB200_INVALID_VALUE, "scale_int8_execute: not a Scale execution");
    auto* e = static_cast<ScaleInt8Exec*>(ex);
    if (!e->resized) return fail(MNNB200_NO_EXECUTION, "scale_int8_execute before resize");
    CK(launch_scale_int8(x, y, e->d_alpha, e->d_bias, e->zin, e->zout, e->minv, e->maxv, (size_t)n * h * w, e->c, e->cp, e->rt->stream));
    return MNNB200_OK;
}
mnnb200_status mnnb200_pool_int8(mnnb200_runtime* rt, const int8_t* x, int n, int c, int ih, int iw, int kh, int kw, int stride_h,
                                 int stride_w, int pad_h, int pad_w, int is_avg, int8_t* y, int oh, int ow) {
    if (!rt || !x || !y || n <= 0 || c <= 0 || oh <= 0 || ow <= 0) return fail(MNNB200_INVALID_VALUE, "pool_int8: bad argument");
    PoolParams p;
    memset(&p, 0, sizeof(p));
    p.x = x; p.y = y; p.N = n; p.C = c; p.Cp = up16(c); p.IH = ih; p.IW = iw; p.OH = oh; p.OW = ow; p.KH = kh; p.KW = kw;
    p.sh = stride_h; p.sw = stride_w; p.ph = pad_h; p.pw = pad_w;
    CK(launch_pool_int8_x86(p, is_avg, rt->stream));
    return MNNB200_OK;
}
mnnb200_status mnnb200_relu_f32(mnnb200_runtime* rt, const float* x, size_t count, float slope, float* y) {
    if (!rt || !x || !y) return fail(MNNB200_INVALID_VALUE, "relu_f32: NULL argument");
    // the kernel moves float4 words: both buffers must be 16-byte aligned (every device allocation is)
    if (((uintptr_t)x & 15) || ((uintptr_t)y & 15)) return fail(MNNB200_INVALID_VALUE, "relu_f32: x / y not 16-byte aligned");
    if (count == 0) return MNNB200_OK;
    CK(launch_relu_f32(x, y, count, slope, rt->stream));
    return MNNB200_OK;
}
mnnb200_status mnnb200_reduce_f32(mnnb200_runtime* rt, const float* x, int outside, int axis, int inside, int op, float* y) {
    if (!rt || !x || !y || outside <= 0 || axis <= 0 || inside <= 0 || op < 0 || op > 4) return fail(MNNB200_INVALID_VALUE, "reduce_f32: bad argument");
    CK(launch_reduce_f32(x, y, outside, axis, inside, op, rt->stream));
    return MNNB200_OK;
}
mnnb200_status mnnb200_softmax_int8(mnnb200_runtime* rt, const int8_t* x, int rows, int c, float s_in, float z_in, float s_out,
                                    float z_out, int min_v, int max_v, int8_t* y) {
    CK(launch_softmax_int8(x, rows, c, up16(c), s_in, z_in, s_out == 0.f ? 0.f : 1.f / s_out, z_out, (float)min_v, (float)max_v,
                           y, rt->stream));
    return MNNB200_OK;
}

// ---- conv ----------------------------------------------------------------------------------------
mnnb200_status mnnb200_conv_int8_create(mnnb200_runtime* rt, const mnnb200_conv_desc* desc, const int8_t* weight,
                                        const float* wscale, const float* bias, mnnb200_exec** out) {
    if (!rt || !desc || !weight || !wscale || !out) return fail(MNNB200_INVALID_VALUE, "conv_int8_create: NULL argument");
    auto* e = new ConvInt8Exec;
    mnnb200_status st = conv_create_common(rt, desc, weight, e);
    if (st) { delete e; return st; }
    e->legacy = false;
    e->h_wscale.assign(wscale, wscale + desc->oc);
    e->h_bias.assign(desc->oc, 0.f);
    if (bias) e->h_bias.assign(bias, bias + desc->oc);
    *out = e;
    return MNNB200_OK;
}
mnnb200_status mnnb200_conv_int8_create_legacy(mnnb200_runtime* rt, const mnnb200_conv_desc* desc, const int8_t* weight,
                                               const float* scale, const int32_t* bias_i32, mnnb200_exec** out) {
    if (!rt || !desc || !weight || !scale || !out) return fail(MNNB200_INVALID_VALUE, "conv_int8_create_legacy: NULL argument");
    auto* e = new ConvInt8Exec;
    mnnb200_status st = conv_create_common(rt, desc, weight, e);
    if (st) { delete e; return st; }
    e->legacy = true;
    e->h_wscale.assign(scale, scale + desc->oc);
    e->h_bias_i32.assign(desc->oc, 0);
    if (bias_i32) e->h_bias_i32.assign(bias_i32, bias_i32 + desc->oc);
    *out = e;
    return MNNB200_OK;
}

mnnb200_status mnnb200_conv_int8_resize(mnnb200_exec* ex, int n, int ih, int iw, float in_scale, int in_zero,
                                        float out_scale, int out_zero, int clamp_min, int clamp_max, int* oh, int* ow) {
    if (!ex || ex->kind != 1) return fail(MNNB200_INVALID_VALUE, "conv_int8_resize: not a conv execution");
    auto* e = static_cast<ConvInt8Exec*>(ex);
    const auto& d = e->d;
    // MNN's shape inference owns the output size (SAME padding pads more at the end than at the beginning);
    // a caller that knows it passes it in through *oh/*ow (> 0), pad_h/pad_w being the BEGIN pads.
    int OH = (oh && *oh > 0) ? *oh : conv_out(ih, d.kh, d.stride_h, d.pad_h, d.dilate_h);
    int OW = (ow && *ow > 0) ? *ow : conv_out(iw, d.kw, d.stride_w, d.pad_w, d.dilate_w);
    if (n <= 0 || OH <= 0 || OW <= 0) return fail(MNNB200_COMPUTE_SIZE_ERROR, "conv_int8_resize: empty output");
    // ---- fold (CPU backend arithmetic; see file header)
    std::vector<float> ws(e->OCp, 0.f), bf(e->OCp, 0.f);
    std::vector<int32_t> k128(e->OCp, 0);
    float scale_x = 1.0f;
    if (!e->legacy) {
        if (in_scale == 0.f || out_scale == 0.f) return fail(MNNB200_INVALID_VALUE, "conv_int8_resize: zero quant scale");
        // MutableResourceInt8::updateInputOutputScale, CPUConvolution.cpp:144-201
        const float zoff = (float)in_zero + 128.f;
        for (int o = 0; o < d.oc; ++o) {
            float wsum = (float)e->h_isum[o] * e->h_wscale[o];  // _computeReorderQuantInfo, ConvInt8TiledExecutor.cpp:243-267
            float t = wsum * zoff;
            t = t * in_scale;
            bf[o] = (e->h_bias[o] - t) / out_scale + (float)out_zero;
            ws[o] = e->h_wscale[o];
        }
        scale_x = in_scale / out_scale;  // ConvInt8TiledExecutor.cpp:1967-1976
    } else {
        // old models: ConvInt8TiledExecutor.cpp:796-805 and CPUConvolution.cpp:126-132
        for (int o = 0; o < d.oc; ++o) {
            float ksum = (float)e->h_isum[o];
            float tmp = (float)e->h_bias_i32[o] - 128.f * ksum;
            int32_t b = (int32_t)tmp;
            bf[o] = (float)b * e->h_wscale[o];
            ws[o] = e->h_wscale[o];
        }
    }
    for (int o = 0; o < d.oc; ++o) k128[o] = 128 * e->h_isum[o];
    mnnb200_status st;
    e->resized = false;   // until the new plan is complete
    if ((st = e->update(ws, e->d_wscale))) return st;
    if ((st = e->update(bf, e->d_bias))) return st;
    if ((st = e->update(k128, e->d_wsum128))) return st;

    ConvParams& p = e->p;
    memset(&p, 0, sizeof(p));
    p.w = e->d_w; p.wscale = e->d_wscale; p.bias = e->d_bias; p.wsum128 = e->d_wsum128;
    p.scale_x = scale_x;
    p.minv = (float)(d.relu ? out_zero : clamp_min);  // ConvInt8TiledExecutor.cpp:2231-2236
    p.maxv = (float)clamp_max;
    uint32_t zb = (uint32_t)(uint8_t)(int8_t)in_zero;
    p.zin_splat = (int32_t)(zb | (zb << 8) | (zb << 16) | (zb << 24));
    p.N = n; p.IH = ih; p.IW = iw; p.Cp = e->Cp; p.OH = OH; p.OW = OW; p.OC = d.oc; p.OCp = e->OCp; p.OCw = e->OCp;
    p.KH = d.kh; p.KW = d.kw; p.sh = d.stride_h; p.sw = d.stride_w; p.ph = d.pad_h; p.pw = d.pad_w;
    p.dh = d.dilate_h; p.dw = d.dilate_w;
    p.M = n * OH * OW;
    p.Kc = d.kh * d.kw * (e->Cp / 16);
    e->tile = pick_tile(p.M, p.OCp, e->rt->prop.multiProcessorCount);
    // algorithmic bytes: logical (unpadded) int8 input + output + weights, once each (SURVEY 8d)
    e->cost_bytes = (double)n * ih * iw * d.ic + (double)p.M * d.oc + (double)d.oc * d.ic * d.kh * d.kw;
    e->cost_macs = (double)p.M * d.oc * d.ic * d.kh * d.kw;
    if ((st = conv_plan(e, in_zero, ws, bf, k128))) return st;
    e->solo_x = e->solo_y = nullptr;
    e->resized = true;
    if (oh) *oh = OH;
    if (ow) *ow = OW;
    return MNNB200_OK;
}

mnnb200_status mnnb200_conv_int8_execute(mnnb200_exec* ex, const int8_t* x, int8_t* y) {
    if (!ex || ex->kind != 1) return fail(MNNB200_INVALID_VALUE, "conv_int8_execute: not a conv execution");
    auto* e = static_cast<ConvInt8Exec*>(ex);
    if (!e->resized) return fail(MNNB200_NO_EXECUTION, "conv_int8_execute before resize");
    ConvParams p = e->p;
    p.x = x;
    p.y = y;
    switch (conv_path(e->plan, e->variant)) {
    case ConvPath::Refused:
        return fail(MNNB200_NOT_SUPPORT, "wgmma variant: this conv shape is not taken by the conv-group kernel (stride_w > 2?)");
    case ConvPath::Stem:
        CK(launch_conv_int8_stem(p, e->rt->stream));
        return MNNB200_OK;
    case ConvPath::Group:
        if (!e->solo || e->solo_x != (const void*)x || e->solo_y != (const void*)y) {
            if (!e->solo) { e->solo = new GroupState; e->solo->rt = e->rt; }
            else CK(cudaStreamSynchronize(e->rt->stream));
            std::vector<ConvInt8Exec*> one{e};
            const int8_t* xs[1] = {x};
            int8_t* ys[1] = {y};
            mnnb200_status st = group_build(*e->solo, one, xs, ys, nullptr, nullptr);
            if (st) return st;
            e->solo_x = x; e->solo_y = y;
        }
        return group_launch(*e->solo);
    case ConvPath::MmaSync:
        break;
    }
    CK(launch_conv_int8_igemm(p, e->tile, e->rt->stream));
    return MNNB200_OK;
}
// ---- conv group C ABI (GroupState / group_build are defined above, before the conv entry points)
struct ConvGroupExec : mnnb200_exec {
    std::vector<ConvInt8Exec*> members;
    GroupState gs;
    bool bound = false;
};

int mnnb200_conv_int8_groupable(mnnb200_exec* ex) {
    if (!ex || ex->kind != 1) return 0;
    auto* e = static_cast<ConvInt8Exec*>(ex);
    return e->resized && conv_path(e->plan, 0) == ConvPath::Group;
}
mnnb200_status mnnb200_conv_int8_group_plan(mnnb200_exec* ex, int* fields, int count) {
    if (!ex || ex->kind != 1 || !fields || count < 0) return fail(MNNB200_INVALID_VALUE, "conv_int8_group_plan: bad argument");
    auto* e = static_cast<ConvInt8Exec*>(ex);
    if (!e->resized) return fail(MNNB200_NO_EXECUTION, "conv_int8_group_plan before resize");
    if (!e->plan.group) return fail(MNNB200_NOT_SUPPORT, "conv_int8_group_plan: the conv-group kernel does not take this conv");
    const GroupLayerParams& q = e->plan.q;
    const int v[] = {q.mode, q.cb, q.bn, q.n_chunks, q.m_tiles, q.num_kb, q.K, q.R, q.TWp, e->plan.g.BH};
    for (int i = 0; i < count && i < (int)(sizeof(v) / sizeof(v[0])); ++i) fields[i] = v[i];
    return MNNB200_OK;
}
mnnb200_status mnnb200_conv_group_create(mnnb200_runtime* rt, mnnb200_exec* const* members, int count, mnnb200_exec** out) {
    if (!rt || !members || !out || count <= 0) return fail(MNNB200_INVALID_VALUE, "conv_group_create: bad argument");
    if (count > kGroupMaxLayers) return fail(MNNB200_NOT_SUPPORT, "conv_group_create: more than 64 members");
    auto* g = new ConvGroupExec;
    g->rt = rt;
    g->kind = 6;
    g->gs.rt = rt;
    for (int i = 0; i < count; ++i) {
        if (!members[i] || members[i]->kind != 1 || members[i]->rt != rt) {
            delete g;
            return fail(MNNB200_INVALID_VALUE, "conv_group_create: member is not a conv execution of this runtime");
        }
        g->members.push_back(static_cast<ConvInt8Exec*>(members[i]));
    }
    *out = g;
    return MNNB200_OK;
}
mnnb200_status mnnb200_conv_group_bind(mnnb200_exec* ex, const int8_t* const* xs, int8_t* const* ys) {
    if (!ex || ex->kind != 6 || !xs || !ys) return fail(MNNB200_INVALID_VALUE, "conv_group_bind: bad argument");
    auto* g = static_cast<ConvGroupExec*>(ex);
    CK(cudaStreamSynchronize(g->rt->stream));       // a previous launch may still read the layer table and schedule being replaced
    mnnb200_status st = group_build(g->gs, g->members, xs, ys, &g->cost_bytes, &g->cost_macs);
    g->bound = st == MNNB200_OK;
    return st;
}
mnnb200_status mnnb200_conv_group_execute(mnnb200_exec* ex) {
    if (!ex || ex->kind != 6) return fail(MNNB200_INVALID_VALUE, "conv_group_execute: not a conv group");
    auto* g = static_cast<ConvGroupExec*>(ex);
    if (!g->bound) return fail(MNNB200_NO_EXECUTION, "conv_group_execute before bind");
    return group_launch(g->gs);
}

mnnb200_status mnnb200_conv_int8_set_variant(mnnb200_exec* ex, int variant) {
    if (!ex || (ex->kind != 1 && ex->kind != 3)) return fail(MNNB200_INVALID_VALUE, "set_variant: not a conv/linear execution");
    const bool ok = ex->kind == 1 ? (variant >= 0 && variant <= 2) : (variant == 0 || (variant >= 2 && variant <= 4));
    if (!ok) return fail(MNNB200_INVALID_VALUE, "set_variant: a conv takes variant 0, 1 or 2, a linear 0, 2, 3 or 4");
    ex->variant = variant;
    return MNNB200_OK;
}
mnnb200_status mnnb200_exec_cost(mnnb200_exec* e, double* bytes, double* macs) {
    if (!e) return fail(MNNB200_INVALID_VALUE, "exec_cost: NULL");
    if (bytes) *bytes = e->cost_bytes;
    if (macs) *macs = e->cost_macs;
    return MNNB200_OK;
}
void mnnb200_exec_destroy(mnnb200_exec* e) { delete e; }

}  // extern "C"

// =================================================================================================
// Depthwise int8 conv
// =================================================================================================
struct DwConvInt8Exec : mnnb200_exec {
    mnnb200_conv_desc d;
    int Cp = 0;
    std::vector<float> h_wscale, h_bias;
    std::vector<int32_t> h_isum;
    int8_t* d_w = nullptr;
    float* d_scale = nullptr;
    int32_t* d_bias = nullptr;
    DwParams p;
    bool resized = false;
};

extern "C" {
mnnb200_status mnnb200_dwconv_int8_create(mnnb200_runtime* rt, const mnnb200_conv_desc* desc, const int8_t* weight,
                                          const float* wscale, const float* bias, mnnb200_exec** out) {
    if (!rt || !desc || !weight || !wscale || !out) return fail(MNNB200_INVALID_VALUE, "dwconv_int8_create: NULL argument");
    if (desc->group != desc->ic || desc->ic != desc->oc) return fail(MNNB200_NOT_SUPPORT, "dwconv: group == ic == oc required");
    auto* e = new DwConvInt8Exec;
    e->rt = rt; e->kind = 2; e->d = *desc;
    const int C = desc->oc, taps = desc->kh * desc->kw;
    e->Cp = up16(C);
    std::vector<int8_t> wp((size_t)taps * e->Cp, 0);
    e->h_isum.assign(e->Cp, 0);
    for (int c = 0; c < C; ++c) {
        int32_t s = 0;
        for (int t = 0; t < taps; ++t) { int8_t v = weight[(size_t)c * taps + t]; wp[(size_t)t * e->Cp + c] = v; s += v; }
        e->h_isum[c] = s;
    }
    e->h_wscale.assign(wscale, wscale + C);
    e->h_bias.assign(C, 0.f);
    if (bias) e->h_bias.assign(bias, bias + C);
    mnnb200_status st;
    std::vector<float> z(e->Cp, 0.f);
    std::vector<int32_t> zi(e->Cp, 0);
    if ((st = e->upload(wp, &e->d_w)) || (st = e->upload(z, &e->d_scale)) || (st = e->upload(zi, &e->d_bias))) { delete e; return st; }
    *out = e;
    return MNNB200_OK;
}

mnnb200_status mnnb200_dwconv_int8_resize(mnnb200_exec* ex, int n, int ih, int iw, float in_scale, int in_zero,
                                          float out_scale, int out_zero, int clamp_min, int clamp_max, int* oh, int* ow) {
    if (!ex || ex->kind != 2) return fail(MNNB200_INVALID_VALUE, "dwconv_int8_resize: not a depthwise execution");
    auto* e = static_cast<DwConvInt8Exec*>(ex);
    const auto& d = e->d;
    // MNN's shape inference owns the output size (SAME padding pads more at the end than at the beginning);
    // a caller that knows it passes it in through *oh/*ow (> 0), pad_h/pad_w being the BEGIN pads.
    int OH = (oh && *oh > 0) ? *oh : conv_out(ih, d.kh, d.stride_h, d.pad_h, d.dilate_h);
    int OW = (ow && *ow > 0) ? *ow : conv_out(iw, d.kw, d.stride_w, d.pad_w, d.dilate_w);
    if (n <= 0 || OH <= 0 || OW <= 0) return fail(MNNB200_COMPUTE_SIZE_ERROR, "dwconv_int8_resize: empty output");
    if (in_scale == 0.f || out_scale == 0.f) return fail(MNNB200_INVALID_VALUE, "dwconv_int8_resize: zero quant scale");
    // depthwise branch of updateInputOutputScale, CPUConvolution.cpp:181-192
    std::vector<float> sc(e->Cp, 0.f);
    std::vector<int32_t> bi(e->Cp, 0);
    const float scale_div = in_scale / out_scale;
    for (int c = 0; c < d.oc; ++c) {
        float ws = e->h_wscale[c];
        if (fabs(ws) < 1e-6) ws = 1e-6;
        sc[c] = ws * scale_div;
        int32_t zfused = (int32_t)((float)out_zero / sc[c]);
        float v = (float)(int32_t)(e->h_bias[c] / (in_scale * ws)) - (float)e->h_isum[c] * ((float)in_zero + 128.f) + (float)zfused;
        int32_t b = (int32_t)v;
        bi[c] = b + 128 * e->h_isum[c];  // device activations are plain int8: fold the x86 +128 storage offset here
    }
    mnnb200_status st;
    if ((st = e->update(sc, e->d_scale)) || (st = e->update(bi, e->d_bias))) return st;
    DwParams& p = e->p;
    memset(&p, 0, sizeof(p));
    p.w = e->d_w; p.scale = e->d_scale; p.bias_i32 = e->d_bias;
    p.zin = in_zero;
    p.minv = d.relu ? out_zero : clamp_min;  // CPUDepthwiseConvInt8.cpp:55-61
    p.maxv = clamp_max;
    p.N = n; p.IH = ih; p.IW = iw; p.Cp = e->Cp; p.C = d.oc; p.OH = OH; p.OW = OW; p.KH = d.kh; p.KW = d.kw;
    p.sh = d.stride_h; p.sw = d.stride_w; p.ph = d.pad_h; p.pw = d.pad_w; p.dh = d.dilate_h; p.dw = d.dilate_w;
    e->cost_bytes = (double)n * ih * iw * e->Cp + (double)n * OH * OW * e->Cp + (double)d.kh * d.kw * e->Cp;
    e->cost_macs = (double)n * OH * OW * d.oc * d.kh * d.kw;
    e->resized = true;
    if (oh) *oh = OH;
    if (ow) *ow = OW;
    return MNNB200_OK;
}

mnnb200_status mnnb200_dwconv_int8_execute(mnnb200_exec* ex, const int8_t* x, int8_t* y) {
    if (!ex || ex->kind != 2) return fail(MNNB200_INVALID_VALUE, "dwconv_int8_execute: not a depthwise execution");
    auto* e = static_cast<DwConvInt8Exec*>(ex);
    if (!e->resized) return fail(MNNB200_NO_EXECUTION, "dwconv_int8_execute before resize");
    DwParams p = e->p;
    p.x = x; p.y = y;
    CK(launch_dwconv_int8(p, e->rt->stream));
    return MNNB200_OK;
}
}  // extern "C"

// =================================================================================================
// LLM linear: W8 weights, dynamic per-token A8
// =================================================================================================
struct LinearW8Exec : mnnb200_exec {
    int ic = 0, oc = 0, icp = 0, ocp = 0, relu = 0, relu6 = 0, tokens = 0;
    bool has_zero = false, has_bias = false;
    int8_t* d_w = nullptr;
    float *d_alpha = nullptr, *d_wzero = nullptr, *d_bias = nullptr, *d_wsumf = nullptr;
    int32_t* d_wsum128 = nullptr;
    int8_t* d_xq = nullptr;
    float *d_dq = nullptr, *d_srcsum = nullptr;
    size_t xq_cap = 0, dq_cap = 0, ss_cap = 0;
    int bn = 0, bn2 = 0;            // bn2 != 0: the CTA-pair kernel is usable for this shape
    CUtensorMap tmap_a, tmap_b, tmap_b_half;
    // K-blocked weight scales (mnnb200_linear_w8_create_blocked): blocks of bs input channels, bs = 0 per channel
    int bs = 0, blocks = 1;
    float *d_balpha = nullptr, *d_bwzero = nullptr;                     // [ocp][blocks]: the GEMV's layout
    float *d_talpha = nullptr, *d_twzero = nullptr, *d_tws = nullptr;   // [blocks][ocp]: the GEMM's layout, ws_b precomputed
    int32_t* d_tw128 = nullptr;                                         // [blocks][ocp] 128 * sum_b w
    float* d_xsb = nullptr;                                             // [tokens][blocks] xsum_b * dq (GEMM path)
    size_t xsb_cap = 0;
};

extern "C" {
mnnb200_status mnnb200_linear_w8_create(mnnb200_runtime* rt, int ic, int oc, const int8_t* wq, const float* alpha,
                                        const float* wzero, const float* bias, int relu, int relu6, mnnb200_exec** out) {
    if (!rt || !wq || !alpha || !out || ic <= 0 || oc <= 0) return fail(MNNB200_INVALID_VALUE, "linear_w8_create: bad argument");
    auto* e = new LinearW8Exec;
    e->rt = rt; e->kind = 3; e->ic = ic; e->oc = oc; e->icp = up16(ic); e->ocp = up16(oc); e->relu = relu; e->relu6 = relu6;
    e->has_zero = wzero != nullptr; e->has_bias = bias != nullptr;
    std::vector<int8_t> wp((size_t)e->ocp * e->icp, 0);
    std::vector<float> al(e->ocp, 0.f), wz(e->ocp, 0.f), bs(e->ocp, 0.f), wsf(e->ocp, 0.f);
    std::vector<int32_t> k128(e->ocp, 0);
    for (int o = 0; o < oc; ++o) {
        int32_t s = 0;
        for (int k = 0; k < ic; ++k) { int8_t v = wq[(size_t)o * ic + k]; wp[(size_t)o * e->icp + k] = v; s += v; }
        al[o] = alpha[o];
        float zb = wzero ? wzero[o] : 0.0f * alpha[o];
        if (wzero) wz[o] = wzero[o];
        if (bias) bs[o] = bias[o];
        wsf[o] = (float)s * alpha[o] + (float)ic * zb;  // _computeReorderQuantInfo, ConvInt8TiledExecutor.cpp:226-267
        k128[o] = 128 * s;
    }
    mnnb200_status st;
    if ((st = e->upload(wp, &e->d_w)) || (st = e->upload(al, &e->d_alpha)) || (st = e->upload(wz, &e->d_wzero)) ||
        (st = e->upload(bs, &e->d_bias)) || (st = e->upload(wsf, &e->d_wsumf)) || (st = e->upload(k128, &e->d_wsum128))) {
        delete e;
        return st;
    }
    *out = e;
    return MNNB200_OK;
}

mnnb200_status mnnb200_linear_w8_create_blocked(mnnb200_runtime* rt, int ic, int oc, int blocks, const int8_t* wq,
                                                const float* alpha, const float* wzero, const float* bias, int relu, int relu6,
                                                mnnb200_exec** out) {
    if (!rt || !wq || !alpha || !out || ic <= 0 || oc <= 0 || blocks < 1 || ic % blocks)
        return fail(MNNB200_INVALID_VALUE, "linear_w8_create_blocked: bad argument (blocks must divide ic)");
    if (blocks == 1) return mnnb200_linear_w8_create(rt, ic, oc, wq, alpha, wzero, bias, relu, relu6, out);
    const int bs = ic / blocks;
    if (bs % 32) return fail(MNNB200_NOT_SUPPORT, "linear_w8_create_blocked: a block must be a multiple of 32 channels (one wgmma k-step)");
    if (bs > 512 || (bs & (bs - 1)))
        return fail(MNNB200_NOT_SUPPORT, "linear_w8_create_blocked: the GEMV takes power-of-two blocks of at most 512 channels");
    auto* e = new LinearW8Exec;
    e->rt = rt; e->kind = 3; e->ic = ic; e->oc = oc; e->icp = up16(ic); e->ocp = up16(oc); e->relu = relu; e->relu6 = relu6;
    e->has_zero = wzero != nullptr; e->has_bias = bias != nullptr; e->bs = bs; e->blocks = blocks;
    const size_t nt = (size_t)e->ocp * blocks;
    std::vector<int8_t> wp((size_t)e->ocp * e->icp, 0);
    std::vector<float> bsv(e->ocp, 0.f), ba(nt, 0.f), bz(nt, 0.f), ta(nt, 0.f), tz(nt, 0.f), tws(nt, 0.f);
    std::vector<int32_t> tw128(nt, 0);
    for (int o = 0; o < oc; ++o) {
        for (int k = 0; k < ic; ++k) wp[(size_t)o * e->icp + k] = wq[(size_t)o * ic + k];
        if (bias) bsv[o] = bias[o];
        for (int b = 0; b < blocks; ++b) {
            int32_t isum = 0;
            for (int k = b * bs; k < (b + 1) * bs; ++k) isum += wq[(size_t)o * ic + k];
            const size_t ob = (size_t)o * blocks + b, bo = (size_t)b * e->ocp + o;
            const float a = alpha[ob], z = wzero ? wzero[ob] : 0.0f;
            ba[ob] = a; bz[ob] = z;
            ta[bo] = a; tz[bo] = z;
            tws[bo] = (float)isum * a + (float)bs * z;   // the block's weightKernelSum
            tw128[bo] = 128 * isum;
        }
    }
    mnnb200_status st;
    if ((st = e->upload(wp, &e->d_w)) || (st = e->upload(bsv, &e->d_bias)) || (st = e->upload(ba, &e->d_balpha)) ||
        (st = e->upload(bz, &e->d_bwzero)) || (st = e->upload(ta, &e->d_talpha)) || (st = e->upload(tz, &e->d_twzero)) ||
        (st = e->upload(tws, &e->d_tws)) || (st = e->upload(tw128, &e->d_tw128))) {
        delete e;
        return st;
    }
    *out = e;
    return MNNB200_OK;
}

mnnb200_status mnnb200_linear_w8_resize(mnnb200_exec* ex, int tokens) {
    if (!ex || ex->kind != 3) return fail(MNNB200_INVALID_VALUE, "linear_w8_resize: not a linear execution");
    auto* e = static_cast<LinearW8Exec*>(ex);
    if (tokens <= 0) return fail(MNNB200_COMPUTE_SIZE_ERROR, "linear_w8_resize: tokens <= 0");
    {
        mnnb200_status st;
        if ((st = e->grow_scratch((void**)&e->d_xq, &e->xq_cap, (size_t)tokens * e->icp)) ||
            (st = e->grow_scratch((void**)&e->d_dq, &e->dq_cap, (size_t)tokens * sizeof(float))) ||
            (st = e->grow_scratch((void**)&e->d_srcsum, &e->ss_cap, (size_t)tokens * sizeof(float))))
            return st;
        if (e->bs && (st = e->grow_scratch((void**)&e->d_xsb, &e->xsb_cap, (size_t)tokens * e->blocks * sizeof(float)))) return st;
    }
    e->tokens = tokens;
    // blocked: at most 128 columns per tile, the other half of the accumulator registers holds the fp32 block sums
    e->bn = pick_bn(e->ocp, (tokens + 127) / 128, e->rt->prop.multiProcessorCount, e->bs ? 128 : 256);
    mnnb200_status st;
    if ((st = make_tmap_i8(&e->tmap_a, e->d_xq, tokens, e->icp, 128))) return st;
    if ((st = make_tmap_i8(&e->tmap_b, e->d_w, e->ocp, e->icp, e->bn))) return st;
    // tensor-bound shapes run on CTA pairs (2-CTA cluster, 256 rows): needs >= 256 rows and a B tile that splits into two halves
    e->bn2 = 0;
    if (tokens >= 256 && e->ocp >= 64 && !e->bs) {
        int chunks = (e->ocp + 255) / 256;
        e->bn2 = (((e->ocp + chunks - 1) / chunks) + 31) & ~31;
        if ((st = make_tmap_i8(&e->tmap_b_half, e->d_w, e->ocp, e->icp, e->bn2 / 2))) return st;
    }
    e->cost_bytes = (double)tokens * e->ic * 4 + (double)tokens * e->oc * 4 + (double)e->oc * e->ic +
                    (e->bs ? (double)e->oc * e->blocks * 8 : 0.0);
    e->cost_macs = (double)tokens * e->oc * e->ic;
    return MNNB200_OK;
}

mnnb200_status mnnb200_linear_w8_execute(mnnb200_exec* ex, const float* x, float* y) {
    if (!ex || ex->kind != 3) return fail(MNNB200_INVALID_VALUE, "linear_w8_execute: not a linear execution");
    auto* e = static_cast<LinearW8Exec*>(ex);
    if (e->tokens <= 0) return fail(MNNB200_NO_EXECUTION, "linear_w8_execute before resize");
    if (e->bs && e->variant == 3) return fail(MNNB200_NOT_SUPPORT, "the CTA-pair variant takes per-channel weight scales only");
    // decode (<= 8 tokens): weight-streaming GEMV, bit-identical to the tensor-core kernels (variant 4 forces it)
    if (e->variant == 4 && !linear_w8_gemv_supported(e->tokens, e->icp, e->bs)) return fail(MNNB200_NOT_SUPPORT, "the GEMV variant takes 1..8 tokens");
    // ONE token is a different ARITHMETIC in the reference (asymmetric single-quant, input zero folded into the bias: see
    // linear_w8_gemv.cu), which only the GEMV kernel implements: the tensor-core kernels would silently compute the multi-token form
    if (e->tokens == 1 && (e->variant == 2 || e->variant == 3 || !linear_w8_gemv_supported(1, e->icp, e->bs)))
        return fail(MNNB200_NOT_SUPPORT, "a single token runs the reference's decode arithmetic: GEMV kernel only (variant 0 or 4, ic <= 25600)");
    if (e->variant == 4 || e->tokens == 1 || (e->variant == 0 && linear_w8_gemv_supported(e->tokens, e->icp, e->bs))) {
        GemvW8Params g;
        g.x = x; g.w = e->d_w; g.y = y; g.alpha = e->d_alpha; g.bias = e->has_bias ? e->d_bias : nullptr; g.wsumf = e->d_wsumf;
        g.wzero = e->has_zero ? e->d_wzero : nullptr; g.wsum128 = e->d_wsum128;
        g.tokens = e->tokens; g.ic = e->ic; g.oc = e->oc; g.ocp = e->ocp; g.icp = e->icp; g.ldy = e->oc; g.relu = e->relu; g.relu6 = e->relu6;
        g.bs = e->bs; g.balpha = e->d_balpha; g.bwzero = e->d_bwzero;
        CK(launch_linear_w8_gemv(g, e->rt->stream, e->rt->prop.multiProcessorCount));
        return MNNB200_OK;
    }
    CK(launch_dynamic_quant(x, e->tokens, e->ic, e->icp, e->d_xq, e->d_dq, e->d_srcsum, e->rt->stream, e->bs, e->d_xsb));
    if (e->variant == 3 && !e->bn2) return fail(MNNB200_NOT_SUPPORT, "the CTA-pair variant needs >= 256 tokens and >= 64 output channels");
    GemmI8Params g;
    memset(&g, 0, sizeof(g));
    g.a = e->d_xq; g.b = e->d_w; g.M = e->tokens; g.N = e->ocp; g.K = e->icp;
    g.y_f32 = y; g.ldy = e->oc; g.wscale = e->d_alpha; g.bias = e->has_bias ? e->d_bias : nullptr; g.wsum128 = e->d_wsum128;
    g.OC = e->oc; g.dq = e->d_dq; g.srcsum = e->d_srcsum; g.wsumf = e->d_wsumf; g.wzero = e->has_zero ? e->d_wzero : nullptr;
    g.relu = e->relu; g.relu6 = e->relu6;
    g.bs = e->bs; g.blocks = e->blocks; g.balpha = e->d_talpha; g.bwzero = e->d_twzero; g.bws = e->d_tws; g.bw128 = e->d_tw128;
    g.xsb = e->d_xsb;
    if (e->variant == 3 || (e->variant == 0 && e->bn2)) {
        CK(launch_gemm_i8_2cta(g, &e->tmap_a, &e->tmap_b_half, e->bn2, e->rt->stream, e->rt->prop.multiProcessorCount));
        return MNNB200_OK;
    }
    CK(launch_gemm_i8_wgmma(g, &e->tmap_a, &e->tmap_b, e->bn, e->rt->stream, e->rt->prop.multiProcessorCount));
    return MNNB200_OK;
}
}  // extern "C"

// =================================================================================================
// Int8 Winograd conv (SURVEY a5/a6): host side = ConvInt8Winograd::makeWinoResource + onResize
// (source/backend/cpu/compute/ConvInt8Winograd.cpp:25-126, 183-241) -- float weight transform G (w_q * wscale) G^T,
// per-(position, oc) requantisation, scale/offset tables -- then three enqueues per execute:
// input transform -> alpha^2 batched wgmma int8 GEMMs -> output transform + requantise.
// =================================================================================================
struct WinoConvInt8Exec : mnnb200_exec {
    mnnb200_conv_desc d;
    int unit = 0, alpha = 0, alpha2 = 0, Cp = 0, OCp = 0, OCb = 0, bn = 0;
    std::vector<float> h_bias, h_in_scale;
    std::vector<int32_t> h_in_zero;
    int8_t* d_u = nullptr;                 // [alpha2][OCb][Cp]
    float *d_scale = nullptr, *d_offset = nullptr, *d_fused = nullptr;   // [alpha2][OCp], [alpha2][OCp], [OCp]
    int32_t* d_wsum128 = nullptr;          // [alpha2][OCp]
    int8_t* d_v = nullptr;
    float* d_m = nullptr;
    size_t v_bytes = 0, m_bytes = 0;
    WinoParams p;
    CUtensorMap tmap_a, tmap_b, tmap_u_fused;   // tmap_u_fused: kWinoFusedBN-row boxes of U for the fused F(2,3) kernel
    bool resized = false;
};

// Math::WinogradGenerater(unit, kernel, interp = 1, dividedInG = true), G only: source/math/WingoradGenerater.cpp:96-135,
// 139-222.  g[alpha][r]
static void wino_generate_g(int unit, int r, std::vector<float>& g) {
    const int alpha = unit + r - 1;
    std::vector<float> a(alpha, 0.f), fdiag(alpha, 1.f);
    int sign = 1;
    for (int i = 0; i < alpha - 1; ++i) {
        a[i + 1] = (float)(sign * (1 + i / 2)) * 1.0f;
        sign = -sign;
    }
    for (int x = 0; x < alpha - 1; ++x) {
        float prod = 1.0f;
        for (int i = 0; i < alpha - 1; ++i)
            if (i != x) prod *= (a[x] - a[i]);
        fdiag[x] = prod;
    }
    if (fdiag[0] < 0) fdiag[0] = -fdiag[0];
    g.assign((size_t)alpha * r, 0.f);
    for (int x = 0; x < alpha; ++x)
        for (int y = 0; y < r; ++y) {
            float v = x < alpha - 1 ? ((x == 0 && y == 0) ? 1.0f : ::powf(a[x], (float)y)) : (y == r - 1 ? 1.0f : 0.0f);
            g[(size_t)x * r + y] = v / fdiag[x];
        }
}

extern "C" {
mnnb200_status mnnb200_conv_int8_wino_create(mnnb200_runtime* rt, const mnnb200_conv_desc* desc, const int8_t* weight,
                                             const float* wscale, const float* bias, const int32_t* attr, int attr_len,
                                             mnnb200_exec** out) {
    if (!rt || !desc || !weight || !wscale || !attr || !out) return fail(MNNB200_INVALID_VALUE, "conv_int8_wino_create: NULL argument");
    const auto& d = *desc;
    if (d.group != 1 || d.stride_h != 1 || d.stride_w != 1 || d.dilate_h != 1 || d.dilate_w != 1)
        return fail(MNNB200_NOT_SUPPORT, "conv_int8_wino: stride/dilate/group must be 1");
    // winogradAttr blob (source/core/WinogradInt8Attr.hpp:45-63): version, unitNum, {unitSize, kyStart, kxStart, kySize,
    // kxSize, unitY, unitX, inputScales[a2], inputZeroPoints[a2], weightScales[a2*oc]}*
    if (attr_len < 9 || attr[0] != 0) return fail(MNNB200_INVALID_VALUE, "conv_int8_wino: bad winogradAttr (version must be 0)");
    if (attr[1] != 1) return fail(MNNB200_NOT_SUPPORT, "conv_int8_wino: exactly one Winograd unit is supported");
    const int unit_size = attr[2];
    const int32_t* u = attr + 3;
    const int ky0 = u[0], kx0 = u[1], kys = u[2], kxs = u[3], unit_y = u[4], unit_x = u[5];
    if (ky0 != 0 || kx0 != 0 || kys != d.kh || kxs != d.kw || d.kh != 3 || d.kw != 3 || unit_y != unit_x ||
        (unit_y != 2 && unit_y != 4 && unit_y != 6))
        return fail(MNNB200_NOT_SUPPORT, "conv_int8_wino: only one full-kernel 3x3 unit with F(2/4/6, 3) is supported");
    auto* e = new WinoConvInt8Exec;
    e->rt = rt; e->kind = 4; e->d = d;
    e->unit = unit_y; e->alpha = unit_y + 2; e->alpha2 = e->alpha * e->alpha;
    const int a2 = e->alpha2, alpha = e->alpha, oc = d.oc, ic = d.ic, r = 3;
    if (unit_size != 6 + 2 * a2 + a2 * oc || attr_len < 3 + unit_size) {
        delete e;
        return fail(MNNB200_INVALID_VALUE, "conv_int8_wino: winogradAttr size does not match alpha^2 and oc");
    }
    const float* in_scales = reinterpret_cast<const float*>(u + 6);
    const int32_t* in_zeros = u + 6 + a2;
    const float* w_scales = reinterpret_cast<const float*>(u + 6 + 2 * a2);
    e->h_in_scale.assign(in_scales, in_scales + a2);
    e->h_in_zero.assign(in_zeros, in_zeros + a2);
    e->h_bias.assign(oc, 0.f);
    if (bias) e->h_bias.assign(bias, bias + oc);
    e->Cp = up16(ic); e->OCp = up16(oc);
    e->bn = pick_bn(e->OCp);
    e->OCb = ((e->OCp + e->bn - 1) / e->bn) * e->bn;

    // ---- makeWinoResource: transform the dequantised weights in float, requantise per (position, oc)
    std::vector<float> g;
    wino_generate_g(e->unit, r, g);
    std::vector<float> wt((size_t)a2 * oc * ic);
    for (int o = 0; o < oc; ++o)
        for (int c = 0; c < ic; ++c) {
            float k[9], m[8 * 3], kt[64];
            for (int i = 0; i < 9; ++i) k[i] = (float)weight[((size_t)o * ic + c) * 9 + i] * wscale[o];
            for (int y = 0; y < alpha; ++y)          // M = G * K            (Matrix::multi, source/math/Matrix.cpp:41-78)
                for (int x = 0; x < r; ++x) {
                    float sum = 0.0f;
                    for (int i = 0; i < r; ++i) sum += g[y * r + i] * k[i * r + x];
                    m[y * r + x] = sum;
                }
            for (int y = 0; y < alpha; ++y)          // K' = M * G^T
                for (int x = 0; x < alpha; ++x) {
                    float sum = 0.0f;
                    for (int i = 0; i < r; ++i) sum += m[y * r + i] * g[x * r + i];
                    kt[y * alpha + x] = sum;
                }
            for (int i = 0; i < a2; ++i) wt[((size_t)i * oc + o) * ic + c] = kt[i];
        }
    std::vector<int8_t> uq((size_t)a2 * e->OCb * e->Cp, 0);
    std::vector<float> sc((size_t)a2 * e->OCp, 0.f), of((size_t)a2 * e->OCp, 0.f);
    std::vector<int32_t> k128((size_t)a2 * e->OCp, 0);
    for (int a = 0; a < a2; ++a)
        for (int o = 0; o < oc; ++o) {
            float offset = 0.f;
            const float scale = w_scales[a * oc + o];
            int32_t isum = 0;
            for (int c = 0; c < ic; ++c) {
                const float src = wt[((size_t)a * oc + o) * ic + c];
                const float eps = (float)(((src / scale) > 0 ? 1 : -1) * 1e-6);
                float rv = ::roundf(src / scale + eps);
                rv = rv > -127.f ? rv : -127.f;
                rv = rv < 127.f ? rv : 127.f;
                const int8_t q = (int8_t)rv;
                uq[((size_t)a * e->OCb + o) * e->Cp + c] = q;
                isum += q;
                offset += (float)((int)q * (-in_zeros[a]));
                offset += (float)((int)q * (-128));   // x86 uint8 activation storage (MNN_USE_SSE)
            }
            of[(size_t)a * e->OCp + o] = offset * scale * in_scales[a];
            sc[(size_t)a * e->OCp + o] = scale * in_scales[a];
            k128[(size_t)a * e->OCp + o] = 128 * isum;
        }
    std::vector<float> zf(e->OCp, 0.f);
    mnnb200_status st;
    if ((st = e->upload(uq, &e->d_u)) || (st = e->upload(sc, &e->d_scale)) || (st = e->upload(of, &e->d_offset)) ||
        (st = e->upload(k128, &e->d_wsum128)) || (st = e->upload(zf, &e->d_fused))) {
        delete e;
        return st;
    }
    *out = e;
    return MNNB200_OK;
}

mnnb200_status mnnb200_conv_int8_wino_resize(mnnb200_exec* ex, int n, int ih, int iw, float in_scale, int in_zero,
                                             float out_scale, int out_zero, int clamp_min, int clamp_max, int* oh, int* ow) {
    if (!ex || ex->kind != 4) return fail(MNNB200_INVALID_VALUE, "conv_int8_wino_resize: not a Winograd execution");
    auto* e = static_cast<WinoConvInt8Exec*>(ex);
    const auto& d = e->d;
    // every check first, on locals: a refused resize leaves the previous plan, fused bias and tensor maps as they were
    const int OH = (oh && *oh > 0) ? *oh : conv_out(ih, 3, 1, d.pad_h, 1);
    const int OW = (ow && *ow > 0) ? *ow : conv_out(iw, 3, 1, d.pad_w, 1);
    if (n <= 0 || OH <= 0 || OW <= 0) return fail(MNNB200_COMPUTE_SIZE_ERROR, "conv_int8_wino_resize: empty output");
    if (in_scale == 0.f || out_scale == 0.f) return fail(MNNB200_INVALID_VALUE, "conv_int8_wino_resize: zero quant scale");
    const int hU = (OH + e->unit - 1) / e->unit, wU = (OW + e->unit - 1) / e->unit;
    // the V / U tensor maps' row counts and the position GEMMs' row coordinates (a * Mpad + m, a * OCb + n) are 32-bit:
    // Mpad * alpha2 and OCb * alpha2 <= INT32_MAX (hU * wU is bounded first, so that n * hU * wU cannot overflow)
    const long long lim = 0x7fffffffLL / e->alpha2, tiles = (long long)hU * wU;
    if (tiles > lim || (n * tiles + 127) / 128 * 128 > lim || e->OCb > lim)
        return fail(MNNB200_COMPUTE_SIZE_ERROR, "conv_int8_wino_resize: too many tiles");
    const long long T = n * tiles, Mpad = (T + 127) / 128 * 128;
    // commit; a failure from here on (out of memory, tensor-map encode) leaves no plan, so execute returns NO_EXECUTION
    e->resized = false;
    std::vector<float> fused(e->OCp, 0.f);
    for (int o = 0; o < d.oc; ++o) fused[o] = e->h_bias[o] / out_scale + (float)out_zero;   // mFusedBias, :215-217
    mnnb200_status st;
    if ((st = e->update(fused, e->d_fused))) return st;
    WinoParams& p = e->p;
    memset(&p, 0, sizeof(p));
    p.N = n; p.IH = ih; p.IW = iw; p.Cp = e->Cp; p.OH = OH; p.OW = OW; p.OC = d.oc; p.OCp = e->OCp;
    p.pad_h = d.pad_h; p.pad_w = d.pad_w; p.unit = e->unit;
    p.hU = hU; p.wU = wU;
    p.T = T;
    p.Mpad = (int)Mpad;
    p.s_in = in_scale; p.z_in = in_zero;
    p.out_inv = (float)(1.0 / (double)out_scale);                 // float outputdequantScale = 1.0 / mOutputScale, :340
    p.minv = (float)(d.relu ? out_zero : clamp_min);              // :347-351
    p.maxv = (float)clamp_max;
    for (int a = 0; a < e->alpha2; ++a) {
        p.in_inv[a] = 1.0f / e->h_in_scale[a];                    // makeWinoResource :66-71
        p.in_zero[a] = (float)e->h_in_zero[a];
    }
    p.fused_bias = e->d_fused;
    const size_t vb = (size_t)e->alpha2 * p.Mpad * e->Cp, mb = (size_t)e->alpha2 * p.Mpad * e->OCp * sizeof(float);
    if ((st = e->grow_scratch((void**)&e->d_v, &e->v_bytes, vb)) || (st = e->grow_scratch((void**)&e->d_m, &e->m_bytes, mb))) return st;
    p.v = e->d_v; p.m = e->d_m;
    if ((st = make_tmap_i8(&e->tmap_a, e->d_v, e->alpha2 * p.Mpad, e->Cp, 128))) return st;
    if ((st = make_tmap_i8(&e->tmap_b, e->d_u, e->alpha2 * e->OCb, e->Cp, e->bn))) return st;
    if (e->unit == 2 && (st = make_tmap_i8(&e->tmap_u_fused, e->d_u, e->alpha2 * e->OCb, e->Cp, kWinoFusedBN))) return st;
    // algorithmic bytes / MACs in direct-conv terms (SURVEY 8d C3): int8 in + out + weights once; MACs of the direct form
    e->cost_bytes = (double)n * ih * iw * d.ic + (double)n * OH * OW * d.oc + (double)d.oc * d.ic * 9;
    e->cost_macs = (double)n * OH * OW * d.oc * d.ic * 9;
    e->resized = true;
    if (oh) *oh = OH;
    if (ow) *ow = OW;
    return MNNB200_OK;
}

mnnb200_status mnnb200_conv_int8_set_pad(mnnb200_exec* ex, int pad_h, int pad_w) {
    if (!ex) return fail(MNNB200_INVALID_VALUE, "set_pad: NULL");
    if (ex->kind == 1) { auto* e = static_cast<ConvInt8Exec*>(ex); e->d.pad_h = pad_h; e->d.pad_w = pad_w; }
    else if (ex->kind == 2) { auto* e = static_cast<DwConvInt8Exec*>(ex); e->d.pad_h = pad_h; e->d.pad_w = pad_w; }
    else if (ex->kind == 4) { auto* e = static_cast<WinoConvInt8Exec*>(ex); e->d.pad_h = pad_h; e->d.pad_w = pad_w; }
    else return fail(MNNB200_INVALID_VALUE, "set_pad: not a convolution execution");
    return MNNB200_OK;
}
}  // extern "C"

// the alpha^2 batched position GEMMs of a resized F(4,3) / F(6,3) execution (and of F(2,3)'s three-kernel form)
static GemmI8Params wino_gemm_params(const WinoConvInt8Exec* e) {
    const WinoParams& p = e->p;
    GemmI8Params g;
    memset(&g, 0, sizeof(g));
    g.a = e->d_v; g.b = e->d_u; g.M = (int)p.T; g.N = e->OCp; g.K = e->Cp;
    g.y_f32 = e->d_m; g.ldy = e->OCp; g.wscale = e->d_scale; g.bias = e->d_offset; g.wsum128 = e->d_wsum128; g.OC = e->d.oc;
    g.batch = e->alpha2; g.a_batch_rows = p.Mpad; g.b_batch_rows = e->OCb; g.c_batch_stride = e->OCp; g.wino = 1;
    return g;
}

extern "C" {
mnnb200_status mnnb200_conv_int8_wino_execute(mnnb200_exec* ex, const int8_t* x, int8_t* y) {
    return mnnb200_conv_int8_wino_execute_phases(ex, x, y, 7);
}
mnnb200_status mnnb200_conv_int8_wino_execute_phases(mnnb200_exec* ex, const int8_t* x, int8_t* y, int phases) {
    if (!ex || ex->kind != 4) return fail(MNNB200_INVALID_VALUE, "conv_int8_wino_execute: not a Winograd execution");
    auto* e = static_cast<WinoConvInt8Exec*>(ex);
    if (!e->resized) return fail(MNNB200_NO_EXECUTION, "conv_int8_wino_execute before resize");
    // the transforms move 4 input channels and up to 4 output channels per access
    if (!x || !y || ((uintptr_t)x & 3) || ((uintptr_t)y & 3))
        return fail(MNNB200_INVALID_VALUE, "conv_int8_wino_execute: x and y must be 4-byte aligned");
    WinoParams p = e->p;
    p.x = x; p.y = y;
    if (phases & 1) CK(launch_wino_input(p, e->rt->stream));
    // F(2,3): position GEMMs + output transform fused (16 accumulators resident in registers, no fp32 M round trip); the three-
    // kernel form stays reachable through a single phase bit (per-kernel timing)
    if (e->unit == 2 && (phases & 6) == 6) {
        WinoFusedParams f;
        f.y = y; f.scale = e->d_scale; f.offset = e->d_offset; f.fused_bias = e->d_fused; f.wsum128 = e->d_wsum128;
        f.K = e->Cp; f.Mpad = p.Mpad; f.OCb = e->OCb; f.OCp = e->OCp; f.OC = e->d.oc;
        f.m_tiles = p.Mpad / 128; f.oc_chunks = (e->OCp + kWinoFusedBN - 1) / kWinoFusedBN; f.OH = p.OH; f.OW = p.OW; f.hU = p.hU; f.wU = p.wU; f.T = p.T;
        f.out_inv = p.out_inv; f.minv = p.minv; f.maxv = p.maxv;
        CK(launch_wino_f23_fused(f, &e->tmap_a, &e->tmap_u_fused, e->rt->stream, e->rt->prop.multiProcessorCount));
        return MNNB200_OK;
    }
    if (!(phases & 2)) {
        if (phases & 4) CK(launch_wino_output(p, e->rt->stream));
        return MNNB200_OK;
    }
    CK(launch_gemm_i8_wgmma(wino_gemm_params(e), &e->tmap_a, &e->tmap_b, e->bn, e->rt->stream, e->rt->prop.multiProcessorCount));
    if (phases & 4) CK(launch_wino_output(p, e->rt->stream));
    return MNNB200_OK;
}

mnnb200_status mnnb200_conv_int8_wino_plan(mnnb200_exec* ex, int* fields, int count) {
    if (!ex || ex->kind != 4 || !fields || count < 0) return fail(MNNB200_INVALID_VALUE, "conv_int8_wino_plan: bad argument");
    auto* e = static_cast<WinoConvInt8Exec*>(ex);
    if (!e->resized) return fail(MNNB200_NO_EXECUTION, "conv_int8_wino_plan before resize");
    const WinoParams& p = e->p;
    const int sm = e->rt->prop.multiProcessorCount, m_tiles = p.Mpad / 128, num_kb = (e->Cp + 127) / 128;
    int bn, n_chunks, items, grid, one_tile, resident_b, stages;
    if (e->unit == 2) {            // the fused kernel: (m tile, 8-channel chunk) items over a persistent grid, B streamed
        bn = kWinoFusedBN; n_chunks = e->OCp / kWinoFusedBN; items = m_tiles * n_chunks;
        grid = std::min(items, sm); one_tile = grid == items; resident_b = 0; stages = kWinoFusedStages;
    } else {
        const GemmI8Launch l = gemm_i8_wgmma_launch(wino_gemm_params(e), e->bn, sm);
        bn = e->bn; n_chunks = e->OCb / e->bn; items = l.items;
        grid = l.grid; one_tile = l.one_tile; resident_b = l.resident_b; stages = l.stages;
    }
    const int v[] = {e->unit, (int)p.T, m_tiles, e->Cp, e->OCp, bn, n_chunks, items, grid, one_tile, resident_b, stages, num_kb};
    for (int i = 0; i < count && i < (int)(sizeof(v) / sizeof(v[0])); ++i) fields[i] = v[i];
    return MNNB200_OK;
}
}  // extern "C"

// =================================================================================================
// Float (batched) MatMul (SURVEY a9): C[b][e][h] = A x B (+ bias), MatMul / BatchMatMul semantics of
// source/backend/cpu/CPUMatMul.cpp (transposeA / transposeB) and CPUBatchMatMul (adjX / adjY).
// =================================================================================================
struct MatMulExec : mnnb200_exec {
    int batch = 0, e = 0, l = 0, h = 0, lp = 0, ta = 0, tb = 0, bn = 0;
    int tf32 = 0, esize = 2;               // tf32: fp32 operands consumed as tf32 (no conversion pass); else fp16 operands
    void *d_a = nullptr, *d_b = nullptr;   // K-major scratch operands [batch][e][lp], [batch][h][lp] (only when a pack is needed)
    CUtensorMap tmap_a, tmap_b;
    const void *tmap_a_ptr = nullptr, *tmap_b_ptr = nullptr;
};

extern "C" {
mnnb200_status mnnb200_matmul_create(mnnb200_runtime* rt, int batch, int e, int l, int h, int transpose_a, int transpose_b,
                                     int inputs_are_f16, mnnb200_exec** out) {
    if (!rt || !out || batch <= 0 || e <= 0 || l <= 0 || h <= 0) return fail(MNNB200_INVALID_VALUE, "matmul_create: bad argument");
    auto* m = new MatMulExec;
    m->rt = rt; m->kind = 5; m->batch = batch; m->e = e; m->l = l; m->h = h; m->ta = transpose_a; m->tb = transpose_b;
    // fp32 operands: tf32 wgmma reads them in place (K-major operands need no pass at all)
    m->tf32 = inputs_are_f16 ? 0 : 1;
    m->esize = m->tf32 ? 4 : 2;
    const int kalign = 16 / m->esize;
    m->lp = (l + kalign - 1) / kalign * kalign;
    m->bn = pick_bn(up16(h), batch * ((e + 127) / 128), rt->prop.multiProcessorCount);
    m->cost_bytes = (double)batch * ((double)e * l + (double)l * h + (double)e * h) * 4;
    m->cost_macs = (double)batch * e * l * h;
    *out = m;
    return MNNB200_OK;
}
mnnb200_status mnnb200_matmul_execute(mnnb200_exec* ex, const void* a, const void* b, const float* bias, float* c) {
    if (!ex || ex->kind != 5) return fail(MNNB200_INVALID_VALUE, "matmul_execute: not a matmul execution");
    auto* m = static_cast<MatMulExec*>(ex);
    // A logical [e][l]: memory [e][l] (ta = 0) or [l][e] (ta = 1).  B logical [l][h]; the kernel wants B^T = [h][l]:
    // memory [l][h] (tb = 0) is the transposed form, memory [h][l] (tb = 1) is already K-major.
    const bool aligned = m->lp == m->l;
    const bool a_direct = m->tf32 && !m->ta && aligned && ((uintptr_t)a & 15) == 0;
    const bool b_direct = m->tf32 && m->tb && aligned && ((uintptr_t)b & 15) == 0;
    const size_t row_bytes = (size_t)m->lp * m->esize;
    auto scratch = [&](void** p, size_t rows) -> mnnb200_status {
        if (*p) return MNNB200_OK;
        // one extra tile of rows: the last tile of the last batch reads past the operand
        CK(cudaMalloc(p, (rows + 256) * row_bytes));
        CK(cudaMemsetAsync(*p, 0, (rows + 256) * row_bytes, m->rt->stream));
        m->dev_bufs.push_back(*p);
        return MNNB200_OK;
    };
    mnnb200_status st;
    const void *pa = a, *pb = b;
    if (!a_direct) {
        if ((st = scratch(&m->d_a, (size_t)m->batch * m->e))) return st;
        if (m->tf32) CK(launch_pack_kmajor_f32((const float*)a, (float*)m->d_a, m->batch, m->e, m->l, m->lp, m->ta ? 1 : 0, m->rt->stream));
        else CK(launch_pack_kmajor_f16(a, m->d_a, m->batch, m->e, m->l, m->lp, m->ta ? 1 : 0, m->rt->stream));
        pa = m->d_a;
    }
    if (!b_direct) {
        if ((st = scratch(&m->d_b, (size_t)m->batch * m->h))) return st;
        if (m->tf32) CK(launch_pack_kmajor_f32((const float*)b, (float*)m->d_b, m->batch, m->h, m->l, m->lp, m->tb ? 0 : 1, m->rt->stream));
        else CK(launch_pack_kmajor_f16(b, m->d_b, m->batch, m->h, m->l, m->lp, m->tb ? 0 : 1, m->rt->stream));
        pb = m->d_b;
    }
    if (m->tmap_a_ptr != pa) {
        // direct operands are exactly batch*e rows (TMA zero-fills rows past the end); scratch has a padded tail
        if ((st = make_tmap_i8(&m->tmap_a, pa, m->batch * m->e + (a_direct ? 0 : 128), (int)row_bytes, 128))) return st;
        m->tmap_a_ptr = pa;
    }
    if (m->tmap_b_ptr != pb) {
        if ((st = make_tmap_i8(&m->tmap_b, pb, m->batch * m->h + (b_direct ? 0 : 256), (int)row_bytes, m->bn))) return st;
        m->tmap_b_ptr = pb;
    }
    CK(launch_gemm_f16_wgmma(&m->tmap_a, &m->tmap_b, m->batch, m->e, m->h, (int)row_bytes, m->tf32, m->e, m->h, m->bn, c, bias,
                               m->rt->stream, m->rt->prop.multiProcessorCount));
    return MNNB200_OK;
}
}  // extern "C"

// =================================================================================================
// Float convolutions and their fp32 neighbours (device fp32 tensors are NCHW-linear): the CPU backend's float path
// (CPUConvolution / ConvolutionTiledExecutor, CPUConvolutionDepthwise, CPUBinary ADD, CPUScale, CPUSoftmax) on the GPU.
// =================================================================================================
static int float_act(const mnnb200_conv_desc* d, int relu6) { return relu6 ? 2 : (d->relu ? 1 : 0); }

struct ConvF32Exec : mnnb200_exec {
    mnnb200_conv_desc d;
    int act = 0, cp8 = 0, taps = 0, kp = 0, ocp = 0, bn = 0;
    float *d_hi = nullptr, *d_lo = nullptr, *d_bias = nullptr;
    CUtensorMap tmap_hi, tmap_lo;
    ConvF32Params p;
    bool resized = false;
};
struct DwConvF32Exec : mnnb200_exec {
    mnnb200_conv_desc d;
    int act = 0;
    float *d_w = nullptr, *d_bias = nullptr;
    DwF32Params p;
    bool resized = false;
};
struct ScaleF32Exec : mnnb200_exec {
    int c = 0, n = 0;
    size_t plane = 0;
    float *d_scale = nullptr, *d_bias = nullptr;
    bool resized = false;
};

static bool conv_desc_valid(const mnnb200_conv_desc* d) {
    return d->ic > 0 && d->oc > 0 && d->kh > 0 && d->kw > 0 && d->stride_h > 0 && d->stride_w > 0 && d->dilate_h > 0 &&
           d->dilate_w > 0 && d->pad_h >= 0 && d->pad_w >= 0;
}

extern "C" {
mnnb200_status mnnb200_conv_f32_create(mnnb200_runtime* rt, const mnnb200_conv_desc* desc, const float* weight, const float* bias,
                                       int relu6, mnnb200_exec** out) {
    if (!rt || !desc || !weight || !out) return fail(MNNB200_INVALID_VALUE, "conv_f32_create: NULL argument");
    if (!conv_desc_valid(desc)) return fail(MNNB200_INVALID_VALUE, "conv_f32_create: bad descriptor");
    if (desc->group != 1) return fail(MNNB200_NOT_SUPPORT, "conv_f32: group > 1 (depthwise has its own execution)");
    auto* e = new ConvF32Exec;
    e->rt = rt; e->kind = 8; e->d = *desc; e->act = float_act(desc, relu6);
    e->taps = desc->kh * desc->kw;
    e->cp8 = (desc->ic + 7) & ~7;
    e->kp = (e->taps * e->cp8 + 31) & ~31;
    e->ocp = (desc->oc + 127) & ~127;          // a whole number of tiles of every width: no weight tile reads past the array
    const size_t wn = (size_t)desc->oc * desc->ic * e->taps, packed = (size_t)e->ocp * e->kp;
    std::vector<float> hw(weight, weight + wn), hb(desc->oc, 0.f);
    if (bias) hb.assign(bias, bias + desc->oc);
    float* d_raw = nullptr;
    mnnb200_status st;
    if ((st = e->upload(hw, &d_raw)) || (st = e->upload(hb, &e->d_bias))) { delete e; return st; }
    auto packed_buf = [&](float** p) -> mnnb200_status {
        CK(cudaMalloc((void**)p, packed * sizeof(float)));
        e->dev_bufs.push_back(*p);
        return MNNB200_OK;
    };
    if ((st = packed_buf(&e->d_hi)) || (st = packed_buf(&e->d_lo))) { delete e; return st; }
    cudaError_t ce = launch_pack_conv_w_f32(d_raw, desc->oc, desc->ic, e->taps, e->cp8, e->kp, e->ocp, e->d_hi, e->d_lo, rt->stream);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(rt->stream);
    for (auto& b : e->dev_bufs)                  // the unpacked weights are not needed after the split
        if (b == d_raw) b = nullptr;
    cudaFree(d_raw);
    if (ce != cudaSuccess) { delete e; return fail(MNNB200_CUDA_ERROR, std::string("conv_f32_create: ") + cudaGetErrorString(ce)); }
    *out = e;
    return MNNB200_OK;
}

mnnb200_status mnnb200_conv_f32_set_pad(mnnb200_exec* ex, int pad_h, int pad_w) {
    if (!ex || pad_h < 0 || pad_w < 0) return fail(MNNB200_INVALID_VALUE, "conv_f32_set_pad: bad argument");
    if (ex->kind == 8) { auto* e = static_cast<ConvF32Exec*>(ex); e->d.pad_h = pad_h; e->d.pad_w = pad_w; }
    else if (ex->kind == 9) { auto* e = static_cast<DwConvF32Exec*>(ex); e->d.pad_h = pad_h; e->d.pad_w = pad_w; }
    else return fail(MNNB200_INVALID_VALUE, "conv_f32_set_pad: not a float convolution execution");
    return MNNB200_OK;
}

mnnb200_status mnnb200_conv_f32_resize(mnnb200_exec* ex, int n, int ih, int iw, int* oh, int* ow) {
    if (!ex || ex->kind != 8) return fail(MNNB200_INVALID_VALUE, "conv_f32_resize: not a float conv execution");
    auto* e = static_cast<ConvF32Exec*>(ex);
    const auto& d = e->d;
    const int OH = (oh && *oh > 0) ? *oh : conv_out(ih, d.kh, d.stride_h, d.pad_h, d.dilate_h);
    const int OW = (ow && *ow > 0) ? *ow : conv_out(iw, d.kw, d.stride_w, d.pad_w, d.dilate_w);
    if (n <= 0 || ih <= 0 || iw <= 0 || OH <= 0 || OW <= 0) return fail(MNNB200_COMPUTE_SIZE_ERROR, "conv_f32_resize: empty output");
    const long long M = (long long)n * OH * OW;
    if (M > 0x7fffffffLL - 128 || (long long)n * d.ic * ih * iw > 0x7fffffffLL || (long long)n * d.oc * OH * OW > 0x7fffffffLL)
        return fail(MNNB200_NOT_SUPPORT, "conv_f32_resize: tensor too large for 32-bit indexing");
    // the plan, once per shape: tile width from the layer's shape (fill the SMs before widening the tile), then the weight maps
    const int sm = e->rt->prop.multiProcessorCount;
    const int m_tiles = (int)((M + 127) / 128);
    int bn = d.oc <= 32 ? 32 : (d.oc <= 64 ? 64 : 128);
    while (bn > 32 && (long long)m_tiles * ((d.oc + bn - 1) / bn) < sm) bn >>= 1;
    mnnb200_status st;
    if (bn != e->bn) {
        if ((st = make_tmap_i8(&e->tmap_hi, e->d_hi, e->ocp, e->kp * 4, bn)) ||
            (st = make_tmap_i8(&e->tmap_lo, e->d_lo, e->ocp, e->kp * 4, bn)))
            return st;
        e->bn = bn;
    }
    ConvF32Params& p = e->p;
    memset(&p, 0, sizeof(p));
    p.bias = e->d_bias;
    p.N = n; p.IC = d.ic; p.IH = ih; p.IW = iw; p.OC = d.oc; p.OH = OH; p.OW = OW;
    p.KH = d.kh; p.KW = d.kw; p.sh = d.stride_h; p.sw = d.stride_w; p.ph = d.pad_h; p.pw = d.pad_w; p.dh = d.dilate_h; p.dw = d.dilate_w;
    p.Cp8 = e->cp8; p.taps = e->taps; p.M = (int)M; p.num_kb = e->kp / 32; p.m_tiles = m_tiles; p.n_chunks = (d.oc + bn - 1) / bn;
    p.act = e->act;
    e->cost_bytes = 4.0 * ((double)n * d.ic * ih * iw + (double)M * d.oc + (double)d.oc * d.ic * e->taps);
    e->cost_macs = (double)M * d.oc * d.ic * e->taps;
    e->resized = true;
    if (oh) *oh = OH;
    if (ow) *ow = OW;
    return MNNB200_OK;
}

mnnb200_status mnnb200_conv_f32_execute(mnnb200_exec* ex, const float* x, float* y) {
    if (!ex || ex->kind != 8) return fail(MNNB200_INVALID_VALUE, "conv_f32_execute: not a float conv execution");
    auto* e = static_cast<ConvF32Exec*>(ex);
    if (!e->resized) return fail(MNNB200_NO_EXECUTION, "conv_f32_execute before resize");
    if (!x || !y) return fail(MNNB200_INVALID_VALUE, "conv_f32_execute: NULL tensor");
    ConvF32Params p = e->p;
    p.x = x; p.y = y;
    CK(launch_conv_f32_wgmma(p, &e->tmap_hi, &e->tmap_lo, e->bn, e->rt->stream, e->rt->prop.multiProcessorCount));
    return MNNB200_OK;
}

mnnb200_status mnnb200_conv_f32_plan(mnnb200_exec* ex, int* fields, int count) {
    if (!ex || ex->kind != 8 || !fields || count < 0) return fail(MNNB200_INVALID_VALUE, "conv_f32_plan: bad argument");
    auto* e = static_cast<ConvF32Exec*>(ex);
    if (!e->resized) return fail(MNNB200_NO_EXECUTION, "conv_f32_plan before resize");
    const ConvF32Params& p = e->p;
    const int v[] = {e->bn, p.n_chunks, p.m_tiles, p.num_kb, conv_f32_stages(e->bn), p.Cp8, p.taps};
    for (int i = 0; i < count && i < (int)(sizeof(v) / sizeof(v[0])); ++i) fields[i] = v[i];
    return MNNB200_OK;
}

mnnb200_status mnnb200_dwconv_f32_create(mnnb200_runtime* rt, const mnnb200_conv_desc* desc, const float* weight, const float* bias,
                                         int relu6, mnnb200_exec** out) {
    if (!rt || !desc || !weight || !out) return fail(MNNB200_INVALID_VALUE, "dwconv_f32_create: NULL argument");
    if (!conv_desc_valid(desc)) return fail(MNNB200_INVALID_VALUE, "dwconv_f32_create: bad descriptor");
    if (desc->group != desc->ic || desc->ic != desc->oc) return fail(MNNB200_NOT_SUPPORT, "dwconv_f32: group == ic == oc required");
    auto* e = new DwConvF32Exec;
    e->rt = rt; e->kind = 9; e->d = *desc; e->act = float_act(desc, relu6);
    std::vector<float> hw(weight, weight + (size_t)desc->oc * desc->kh * desc->kw), hb(desc->oc, 0.f);
    if (bias) hb.assign(bias, bias + desc->oc);
    mnnb200_status st;
    if ((st = e->upload(hw, &e->d_w)) || (st = e->upload(hb, &e->d_bias))) { delete e; return st; }
    *out = e;
    return MNNB200_OK;
}

mnnb200_status mnnb200_dwconv_f32_resize(mnnb200_exec* ex, int n, int ih, int iw, int* oh, int* ow) {
    if (!ex || ex->kind != 9) return fail(MNNB200_INVALID_VALUE, "dwconv_f32_resize: not a float depthwise execution");
    auto* e = static_cast<DwConvF32Exec*>(ex);
    const auto& d = e->d;
    const int OH = (oh && *oh > 0) ? *oh : conv_out(ih, d.kh, d.stride_h, d.pad_h, d.dilate_h);
    const int OW = (ow && *ow > 0) ? *ow : conv_out(iw, d.kw, d.stride_w, d.pad_w, d.dilate_w);
    if (n <= 0 || ih <= 0 || iw <= 0 || OH <= 0 || OW <= 0) return fail(MNNB200_COMPUTE_SIZE_ERROR, "dwconv_f32_resize: empty output");
    DwF32Params& p = e->p;
    memset(&p, 0, sizeof(p));
    p.w = e->d_w; p.bias = e->d_bias;
    p.N = n; p.C = d.oc; p.IH = ih; p.IW = iw; p.OH = OH; p.OW = OW; p.KH = d.kh; p.KW = d.kw;
    p.sh = d.stride_h; p.sw = d.stride_w; p.ph = d.pad_h; p.pw = d.pad_w; p.dh = d.dilate_h; p.dw = d.dilate_w; p.act = e->act;
    e->cost_bytes = 4.0 * ((double)n * d.oc * ih * iw + (double)n * d.oc * OH * OW + (double)d.oc * d.kh * d.kw);
    e->cost_macs = (double)n * OH * OW * d.oc * d.kh * d.kw;
    e->resized = true;
    if (oh) *oh = OH;
    if (ow) *ow = OW;
    return MNNB200_OK;
}

mnnb200_status mnnb200_dwconv_f32_execute(mnnb200_exec* ex, const float* x, float* y) {
    if (!ex || ex->kind != 9) return fail(MNNB200_INVALID_VALUE, "dwconv_f32_execute: not a float depthwise execution");
    auto* e = static_cast<DwConvF32Exec*>(ex);
    if (!e->resized) return fail(MNNB200_NO_EXECUTION, "dwconv_f32_execute before resize");
    if (!x || !y) return fail(MNNB200_INVALID_VALUE, "dwconv_f32_execute: NULL tensor");
    DwF32Params p = e->p;
    p.x = x; p.y = y;
    CK(launch_dwconv_f32(p, e->rt->stream));
    return MNNB200_OK;
}

mnnb200_status mnnb200_binary_add_f32(mnnb200_runtime* rt, const float* a, const float* b, float* y, size_t count) {
    if (!rt || !a || !b || !y) return fail(MNNB200_INVALID_VALUE, "binary_add_f32: NULL argument");
    return mnnb200_binary_f32(rt, kBinaryAdd, a, count, b, count, y, count, 0);
}

mnnb200_status mnnb200_binary_f32(mnnb200_runtime* rt, int op, const float* a, size_t count_a, const float* b, size_t count_b,
                                  float* y, size_t count, int relu) {
    if (!rt || !a || !b || !y) return fail(MNNB200_INVALID_VALUE, "binary_f32: NULL argument");
    if (!binary_f32_supported(op)) return fail(MNNB200_NOT_SUPPORT, "binary_f32: op " + std::to_string(op) + " is not supported");
    if (count == 0) return MNNB200_OK;
    if ((count_a != count && count_a != 1) || (count_b != count && count_b != 1))
        return fail(MNNB200_INVALID_VALUE, "binary_f32: each input must have count elements or one");
    CK(launch_binary_f32(op, a, count_a != count, b, count_b != count, y, count, relu ? 1 : 0, rt->stream));
    return MNNB200_OK;
}

mnnb200_status mnnb200_unary_f32(mnnb200_runtime* rt, int op, const float* x, float* y, size_t count) {
    if (!rt || !x || !y) return fail(MNNB200_INVALID_VALUE, "unary_f32: NULL argument");
    if (!unary_f32_supported(op)) return fail(MNNB200_NOT_SUPPORT, "unary_f32: op " + std::to_string(op) + " is not supported");
    if (count == 0) return MNNB200_OK;
    CK(launch_unary_f32(op, x, y, count, rt->stream));
    return MNNB200_OK;
}

mnnb200_status mnnb200_argmax_f32(mnnb200_runtime* rt, const float* x, int outside, int axis, int inside, int is_min, int32_t* y) {
    if (!rt || !x || !y || outside <= 0 || axis <= 0 || inside <= 0) return fail(MNNB200_INVALID_VALUE, "argmax_f32: bad argument");
    CK(launch_argmax_f32(x, outside, axis, inside, is_min ? 1 : 0, y, rt->stream));
    return MNNB200_OK;
}

mnnb200_status mnnb200_scale_f32_create(mnnb200_runtime* rt, int channels, const float* scale, const float* bias, mnnb200_exec** out) {
    if (!rt || !scale || !out || channels <= 0) return fail(MNNB200_INVALID_VALUE, "scale_f32_create: bad argument");
    auto* e = new ScaleF32Exec;
    e->rt = rt; e->kind = 10; e->c = channels;
    std::vector<float> hs(scale, scale + channels), hb(channels, 0.f);
    if (bias) hb.assign(bias, bias + channels);
    mnnb200_status st;
    if ((st = e->upload(hs, &e->d_scale)) || (st = e->upload(hb, &e->d_bias))) { delete e; return st; }
    *out = e;
    return MNNB200_OK;
}

mnnb200_status mnnb200_scale_f32_resize(mnnb200_exec* ex, int n, int h, int w) {
    if (!ex || ex->kind != 10) return fail(MNNB200_INVALID_VALUE, "scale_f32_resize: not a float Scale execution");
    auto* e = static_cast<ScaleF32Exec*>(ex);
    if (n <= 0 || h <= 0 || w <= 0) return fail(MNNB200_COMPUTE_SIZE_ERROR, "scale_f32_resize: empty tensor");
    e->n = n; e->plane = (size_t)h * w;
    e->cost_bytes = 8.0 * n * e->c * (double)e->plane;
    e->cost_macs = (double)n * e->c * (double)e->plane;
    e->resized = true;
    return MNNB200_OK;
}

mnnb200_status mnnb200_scale_f32_execute(mnnb200_exec* ex, const float* x, float* y) {
    if (!ex || ex->kind != 10) return fail(MNNB200_INVALID_VALUE, "scale_f32_execute: not a float Scale execution");
    auto* e = static_cast<ScaleF32Exec*>(ex);
    if (!e->resized) return fail(MNNB200_NO_EXECUTION, "scale_f32_execute before resize");
    if (!x || !y) return fail(MNNB200_INVALID_VALUE, "scale_f32_execute: NULL tensor");
    CK(launch_scale_f32(x, e->d_scale, e->d_bias, y, e->n, e->c, e->plane, e->rt->stream));
    return MNNB200_OK;
}

mnnb200_status mnnb200_softmax_f32(mnnb200_runtime* rt, const float* x, int outside, int axis, int inside, float* y) {
    if (!rt || !x || !y || outside <= 0 || axis <= 0 || inside <= 0) return fail(MNNB200_INVALID_VALUE, "softmax_f32: bad argument");
    CK(launch_softmax_f32(x, y, outside, axis, inside, rt->stream));
    return MNNB200_OK;
}
}  // extern "C"
