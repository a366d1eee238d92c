// deconv_capi.cu -- C ABI of libmnn_b200_deconv.so (include/mnn_b200_deconv.h): the float Deconvolution executions
// (CPUDeconvolution, CPUDeconvolutionDepthwise) on NCHW-linear fp32 tensors, over the kernels of deconv_f32_wgmma.cu, on the
// runtime and execution handles of libmnn_b200.so (exec.h).
#include <cuda.h>
#include <cuda_runtime.h>
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/mnn_b200_deconv.h"
#include "deconv_ops.h"
#include "exec.h"

using namespace mnnb200;

struct DeconvF32Exec : Tagged<kDeconvF32, ConvExec> {
    int act = 0, cp8 = 0, kp = 0, ocp = 0, bn = 0;
    int max_m_tiles = 0, max_kb = 0, max_taps = 0;
    DevBuf<float> d_hi, d_lo, d_bias;
    CUtensorMap tmap_hi, tmap_lo;
    DeconvF32Params p;
};
struct DwDeconvF32Exec : Tagged<kDwDeconvF32, ConvExec> {
    int act = 0;
    DevBuf<float> d_w, d_bias;
    DwF32Params p;
};

// The output size of a transposed conv: *oh / *ow when > 0, else the natural size.  NOT_SUPPORT for an empty tensor and for
// output rows (columns) past the last one a tap reaches plus the stride - 1 an out-pad can add, and for indices past 32 bits.
static mnnb200_status deconv_out_size(const mnnb200_conv_desc& d, int n, int ih, int iw, const int* oh, const int* ow, int* OH,
                                      int* OW, const char* what) {
    const long long reach_h = (long long)(ih - 1) * d.stride_h + (long long)d.dilate_h * (d.kh - 1) + 1;
    const long long reach_w = (long long)(iw - 1) * d.stride_w + (long long)d.dilate_w * (d.kw - 1) + 1;
    const long long H = oh && *oh > 0 ? *oh : reach_h - 2LL * d.pad_h, W = ow && *ow > 0 ? *ow : reach_w - 2LL * d.pad_w;
    if (n <= 0 || ih <= 0 || iw <= 0 || H <= 0 || W <= 0)
        return fail(MNNB200_NOT_SUPPORT, std::string(what) + ": empty tensor");
    if (H + d.pad_h > reach_h + d.stride_h - 1 || W + d.pad_w > reach_w + d.stride_w - 1)
        return fail(MNNB200_NOT_SUPPORT, std::string(what) + ": output size past what the pads and strides produce");
    if ((long long)n * H * W > 0x7fffffffLL - 128 || (long long)n * d.ic * ih * iw > 0x7fffffffLL ||
        (long long)n * d.oc * H * W > 0x7fffffffLL)
        return fail(MNNB200_NOT_SUPPORT, std::string(what) + ": tensor too large for 32-bit indexing");
    *OH = (int)H;
    *OW = (int)W;
    return MNNB200_OK;
}

extern "C" {
mnnb200_status mnnb200_deconv_f32_create(mnnb200_runtime* rt, const mnnb200_conv_desc* desc, const float* weight, const float* bias,
                                         int relu6, mnnb200_exec** out) {
    if (!rt || !desc || !weight || !out) return fail(MNNB200_INVALID_VALUE, "deconv_f32_create: NULL argument");
    if (!conv_desc_valid(desc)) return fail(MNNB200_INVALID_VALUE, "deconv_f32_create: bad descriptor");
    if (desc->group != 1) return fail(MNNB200_NOT_SUPPORT, "deconv_f32: group > 1 (depthwise has its own execution)");
    if (desc->stride_h > kDeconvMaxStride || desc->stride_w > kDeconvMaxStride)
        return fail(MNNB200_NOT_SUPPORT, "deconv_f32: stride > " + std::to_string(kDeconvMaxStride));
    auto e = new_exec<DeconvF32Exec>(rt);
    e->d = *desc; e->act = float_act(desc, relu6);
    e->cp8 = (desc->ic + 7) & ~7;
    // one K extent for every phase: the deepest phase's taps * cp8, rounded up to whole K blocks
    for (int ry = 0; ry < desc->stride_h; ++ry)
        for (int rx = 0; rx < desc->stride_w; ++rx) {
            const int taps = deconv_axis_taps(ry, desc->stride_h, desc->dilate_h, desc->kh).nk *
                             deconv_axis_taps(rx, desc->stride_w, desc->dilate_w, desc->kw).nk;
            e->kp = std::max(e->kp, (taps * e->cp8 + 31) & ~31);
        }
    e->ocp = (desc->oc + 127) & ~127;          // a whole number of tiles of every width: no weight tile crosses a phase
    const int phases = desc->stride_h * desc->stride_w;
    const size_t wn = (size_t)desc->ic * desc->oc * desc->kh * desc->kw, packed = (size_t)phases * e->ocp * e->kp;
    if ((size_t)phases * e->ocp > 0x7fffffffULL || (size_t)e->kp * 4 > 0x7fffffffULL)
        return fail(MNNB200_NOT_SUPPORT, "deconv_f32_create: weights too large");
    std::vector<float> hw(weight, weight + wn), hb(desc->oc, 0.f);
    if (bias) hb.assign(bias, bias + desc->oc);
    DevBuf<float> raw;
    mnnb200_status st;
    if ((st = raw.upload(hw, rt->stream)) || (st = e->d_bias.upload(hb, rt->stream)) || (st = e->d_hi.reserve(packed)) ||
        (st = e->d_lo.reserve(packed)))
        return st;
    cudaError_t ce = launch_pack_deconv_w_f32(raw, desc->ic, desc->oc, desc->kh, desc->kw, desc->stride_h, desc->stride_w,
                                              desc->dilate_h, desc->dilate_w, e->cp8, e->kp, e->ocp, e->d_hi, e->d_lo, rt->stream);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(rt->stream);
    raw.reset();
    if (ce != cudaSuccess) return fail(MNNB200_CUDA_ERROR, std::string("deconv_f32_create: ") + cudaGetErrorString(ce));
    *out = e.release();
    return MNNB200_OK;
}

mnnb200_status mnnb200_deconv_f32_set_pad(mnnb200_exec* ex, int pad_h, int pad_w) {
    auto* e = exec_as<ConvExec>(ex, kDeconvF32 | kDwDeconvF32);
    if (!e || pad_h < 0 || pad_w < 0)
        return fail(MNNB200_INVALID_VALUE, "deconv_f32_set_pad: bad argument (a float deconvolution, pads >= 0)");
    e->d.pad_h = pad_h; e->d.pad_w = pad_w;
    return MNNB200_OK;
}

mnnb200_status mnnb200_deconv_f32_resize(mnnb200_exec* ex, int n, int ih, int iw, int* oh, int* ow) {
    auto* e = exec_as<DeconvF32Exec>(ex);
    if (!e) return fail(MNNB200_INVALID_VALUE, "deconv_f32_resize: not a float deconvolution execution");
    const auto& d = e->d;
    int OH = 0, OW = 0;
    if (mnnb200_status st = deconv_out_size(d, n, ih, iw, oh, ow, &OH, &OW, "deconv_f32_resize")) return st;
    // the phases: per residue of each axis its outputs and taps, then the work items phase by phase
    DeconvF32Params p;
    memset(&p, 0, sizeof(p));
    p.bias = e->d_bias;
    p.N = n; p.IC = d.ic; p.IH = ih; p.IW = iw; p.OC = d.oc; p.OH = OH; p.OW = OW;
    p.sh = d.stride_h; p.sw = d.stride_w; p.Cp8 = e->cp8; p.ocp = e->ocp; p.act = e->act;
    auto axis = [](int r, int s, int dil, int k, int pad, int out, DeconvAxis& a) {
        const DeconvAxisTaps t = deconv_axis_taps(r, s, dil, k);
        a.o0 = ((r - pad) % s + s) % s;
        a.len = a.o0 < out ? (out - 1 - a.o0) / s + 1 : 0;
        a.q0 = (a.o0 + pad) / s;
        a.nk = t.nk; a.off0 = t.off0;
        return t.istep;
    };
    for (int r = 0; r < p.sh; ++r) p.istep_h = axis(r, p.sh, d.dilate_h, d.kh, d.pad_h, OH, p.ay[r]);
    for (int r = 0; r < p.sw; ++r) p.istep_w = axis(r, p.sw, d.dilate_w, d.kw, d.pad_w, OW, p.ax[r]);
    int max_m_tiles = 0, max_kb = 0, max_taps = 0;
    long long m_tiles = 0;
    for (int ry = 0; ry < p.sh; ++ry)
        for (int rx = 0; rx < p.sw; ++rx) {
            const int mt = (int)(((long long)n * p.ay[ry].len * p.ax[rx].len + 127) / 128), taps = p.ay[ry].nk * p.ax[rx].nk;
            m_tiles += mt;
            max_m_tiles = std::max(max_m_tiles, mt);
            max_taps = std::max(max_taps, taps);
            max_kb = std::max(max_kb, (taps * e->cp8 + 31) / 32);
        }
    const int sm = e->rt->prop.multiProcessorCount;
    int bn = d.oc <= 32 ? 32 : (d.oc <= 64 ? 64 : 128);
    while (bn > 32 && m_tiles * ((d.oc + bn - 1) / bn) < sm) bn >>= 1;
    p.n_chunks = (d.oc + bn - 1) / bn;
    long long items = 0;
    for (int ph = 0; ph < p.sh * p.sw; ++ph) {
        items += (((long long)n * p.ay[ph / p.sw].len * p.ax[ph % p.sw].len + 127) / 128) * p.n_chunks;
        p.item_end[ph] = (int)items;
    }
    if (items > 0x7fffffffLL) return fail(MNNB200_NOT_SUPPORT, "deconv_f32_resize: tensor too large for 32-bit indexing");
    p.items = (int)items;
    mnnb200_status st;
    if (bn != e->bn) {
        const int rows = p.sh * p.sw * e->ocp;
        if ((st = make_tmap_i8(&e->tmap_hi, e->d_hi, rows, e->kp * 4, bn)) || (st = make_tmap_i8(&e->tmap_lo, e->d_lo, rows, e->kp * 4, bn)))
            return st;
        e->bn = bn;
    }
    e->p = p;
    e->max_m_tiles = max_m_tiles; e->max_kb = max_kb; e->max_taps = max_taps;
    e->cost_bytes = 4.0 * ((double)n * d.ic * ih * iw + (double)n * d.oc * OH * OW + (double)d.oc * d.ic * d.kh * d.kw);
    e->cost_macs = (double)n * ih * iw * d.ic * d.oc * d.kh * d.kw;
    e->resized = true;
    if (oh) *oh = OH;
    if (ow) *ow = OW;
    return MNNB200_OK;
}

mnnb200_status mnnb200_deconv_f32_execute(mnnb200_exec* ex, const float* x, float* y) {
    auto* e = exec_as<DeconvF32Exec>(ex);
    if (!e) return fail(MNNB200_INVALID_VALUE, "deconv_f32_execute: not a float deconvolution execution");
    if (!e->resized) return fail(MNNB200_NO_EXECUTION, "deconv_f32_execute before resize");
    if (!x || !y) return fail(MNNB200_INVALID_VALUE, "deconv_f32_execute: NULL tensor");
    DeconvF32Params p = e->p;
    p.x = x; p.y = y;
    CK(launch_deconv_f32_wgmma(p, &e->tmap_hi, &e->tmap_lo, e->bn, e->rt->stream, e->rt->prop.multiProcessorCount));
    return MNNB200_OK;
}

mnnb200_status mnnb200_deconv_f32_plan(mnnb200_exec* ex, int* fields, int count) {
    auto* e = exec_as<DeconvF32Exec>(ex);
    if (!e || !fields || count < 0) return fail(MNNB200_INVALID_VALUE, "deconv_f32_plan: bad argument");
    if (!e->resized) return fail(MNNB200_NO_EXECUTION, "deconv_f32_plan before resize");
    const int v[] = {e->bn, e->p.n_chunks, e->p.sh * e->p.sw, e->max_m_tiles, e->max_kb, deconv_f32_stages(e->bn), e->max_taps};
    return copy_fields(v, fields, count);
}

mnnb200_status mnnb200_dwdeconv_f32_create(mnnb200_runtime* rt, const mnnb200_conv_desc* desc, const float* weight, const float* bias,
                                           int relu6, mnnb200_exec** out) {
    if (!rt || !desc || !weight || !out) return fail(MNNB200_INVALID_VALUE, "dwdeconv_f32_create: NULL argument");
    if (!conv_desc_valid(desc)) return fail(MNNB200_INVALID_VALUE, "dwdeconv_f32_create: bad descriptor");
    if (desc->group != desc->ic || desc->ic != desc->oc) return fail(MNNB200_NOT_SUPPORT, "dwdeconv_f32: group == ic == oc required");
    auto e = new_exec<DwDeconvF32Exec>(rt);
    e->d = *desc; e->act = float_act(desc, relu6);
    std::vector<float> hw(weight, weight + (size_t)desc->oc * desc->kh * desc->kw), hb(desc->oc, 0.f);
    if (bias) hb.assign(bias, bias + desc->oc);
    mnnb200_status st;
    if ((st = e->d_w.upload(hw, rt->stream)) || (st = e->d_bias.upload(hb, rt->stream))) return st;
    *out = e.release();
    return MNNB200_OK;
}

mnnb200_status mnnb200_dwdeconv_f32_resize(mnnb200_exec* ex, int n, int ih, int iw, int* oh, int* ow) {
    auto* e = exec_as<DwDeconvF32Exec>(ex);
    if (!e) return fail(MNNB200_INVALID_VALUE, "dwdeconv_f32_resize: not a float depthwise deconvolution execution");
    const auto& d = e->d;
    int OH = 0, OW = 0;
    if (mnnb200_status st = deconv_out_size(d, n, ih, iw, oh, ow, &OH, &OW, "dwdeconv_f32_resize")) return st;
    DwF32Params& p = e->p;
    memset(&p, 0, sizeof(p));
    p.w = e->d_w; p.bias = e->d_bias;
    p.N = n; p.C = d.oc; p.IH = ih; p.IW = iw; p.OH = OH; p.OW = OW; p.KH = d.kh; p.KW = d.kw;
    p.sh = d.stride_h; p.sw = d.stride_w; p.ph = d.pad_h; p.pw = d.pad_w; p.dh = d.dilate_h; p.dw = d.dilate_w; p.act = e->act;
    e->cost_bytes = 4.0 * ((double)n * d.oc * ih * iw + (double)n * d.oc * OH * OW + (double)d.oc * d.kh * d.kw);
    e->cost_macs = (double)n * ih * iw * d.oc * d.kh * d.kw;
    e->resized = true;
    if (oh) *oh = OH;
    if (ow) *ow = OW;
    return MNNB200_OK;
}

mnnb200_status mnnb200_dwdeconv_f32_execute(mnnb200_exec* ex, const float* x, float* y) {
    auto* e = exec_as<DwDeconvF32Exec>(ex);
    if (!e) return fail(MNNB200_INVALID_VALUE, "dwdeconv_f32_execute: not a float depthwise deconvolution execution");
    if (!e->resized) return fail(MNNB200_NO_EXECUTION, "dwdeconv_f32_execute before resize");
    if (!x || !y) return fail(MNNB200_INVALID_VALUE, "dwdeconv_f32_execute: NULL tensor");
    DwF32Params p = e->p;
    p.x = x; p.y = y;
    CK(launch_dwdeconv_f32(p, e->rt->stream));
    return MNNB200_OK;
}
}  // extern "C"

