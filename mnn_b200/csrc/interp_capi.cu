// interp_capi.cu -- C ABI of libmnn_b200_interp.so (include/mnn_b200_interp.h): the fp32 Interp execution (CPUInterp) on
// NCHW-linear fp32 tensors, over the kernel of interp_f32.cu, on the runtime and execution handles of libmnn_b200.so (exec.h).
//
// resize builds the kernel's tables the way CPUInterp::onResize and CPUResize.hpp build theirs, in the same float expressions
// (this host code is compiled with -ffp-contract=off, as the reference's CPU sources are compiled without -mfma):
//   nearest (1):        x1 = floor(dst * scale + offset), clamped
//   nearest-round (4):  x1 = floor(dst * scale + offset + 0.499f), clamped
//   bilinear (2):       src = dst * scale + offset, x1 = floor(src), f = src - x1; taps x1, x1 + 1 (clamped), weights 1 - f, f
//   cubic (3):          src = dst * scale + offset, taps (int)src - 1 .. + 2 (truncation, clamped), t = src - floor(src), and
//                       the weights of the Keys kernel with a = -0.75 with the CPU's mix of float and double (cubic_weights).
#include <cuda_runtime.h>
#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/mnn_b200_interp.h"
#include "exec.h"
#include "interp_ops.h"

using namespace mnnb200;

struct InterpF32Exec : Tagged<kInterpF32> {
    int resize_type = 0;
    float scale_w = 0.f, scale_h = 0.f, offset_w = 0.f, offset_h = 0.f;
    DevBuf<int> d_xi, d_yi;
    DevBuf<float> d_xw, d_yw;
    InterpF32Params p;
    int last_vec = -1, last_grid = 0, last_row_groups = 0;   // the last execute's launch since resize
};

namespace {

int taps_of(int type) { return type == 2 ? 2 : (type == 3 ? 4 : 1); }

// (int)v for a float v, saturated at the int range (the CPU's conversion of a coordinate far outside the image is undefined;
// any value past the range clamps to the same border)
int to_int(float v) {
    if (v <= -2147483648.f) return INT32_MIN;
    if (v >= 2147483648.f) return INT32_MAX;
    return (int)v;
}
int clamp_tap(long long v, int n) { return (int)std::min<long long>(std::max<long long>(v, 0), n - 1); }

// the four weights of CubicInterpolation2 (compute/ResizeFunction.cpp) at fraction t: b and c are float expressions except c's
// cubic term, which is double (a double constant); a and d are double, the product 5.0f * 0.75 being exactly 3.75; each is
// rounded to float where the CPU multiplies the taps by it
void cubic_weights(float t, float* w) {
    const float u = 1.0f - t, ta = 1.0f + t, td = 2.0f - t;
    const double a = (double)(3.0f - 6.0f * ta) + 3.75 * ta * ta - (double)(0.75f * ta * ta * ta);
    const float b = 1.0f - 2.25f * t * t + 1.25f * t * t * t;
    const double c = (double)(1.0f - 2.25f * u * u) + 1.25 * u * u * u;
    const double d = (double)(3.0f - 6.0f * td) + 3.75 * td * td - (double)(0.75f * td * td * td);
    w[0] = (float)a; w[1] = b; w[2] = (float)c; w[3] = (float)d;
}

// one axis' table: `out` destination positions of an `in`-long input axis
void axis_table(int type, float scale, float offset, int in, int out, std::vector<int>& idx, std::vector<float>& wt) {
    const int taps = taps_of(type);
    idx.resize((size_t)out * taps);
    wt.resize(taps > 1 ? (size_t)out * taps : 0);
    for (int o = 0; o < out; ++o) {
        const float src = (float)o * scale + offset;
        int* ix = &idx[(size_t)o * taps];
        if (type == 1) {
            ix[0] = clamp_tap(to_int(std::floor(src)), in);
        } else if (type == 4) {
            ix[0] = clamp_tap(to_int(std::floor(src + 0.499f)), in);
        } else if (type == 2) {
            const int x1 = to_int(std::floor(src));
            const float f = src - (float)x1;
            ix[0] = clamp_tap(x1, in);
            ix[1] = clamp_tap((long long)x1 + 1, in);
            wt[(size_t)o * 2 + 0] = 1.0f - f;
            wt[(size_t)o * 2 + 1] = f;
        } else {
            const int x1 = to_int(src);
            const float t = src - std::floor(src);
            for (int k = 0; k < 4; ++k) ix[k] = clamp_tap((long long)x1 - 1 + k, in);
            cubic_weights(t, &wt[(size_t)o * 4]);
        }
    }
}

}  // namespace

extern "C" {
mnnb200_status mnnb200_interp_f32_create(mnnb200_runtime* rt, int resize_type, float width_scale, float height_scale,
                                         float width_offset, float height_offset, mnnb200_exec** out) {
    if (!rt || !out) return fail(MNNB200_INVALID_VALUE, "interp_f32_create: NULL argument");
    auto e = new_exec<InterpF32Exec>(rt);
    e->resize_type = resize_type;
    e->scale_w = width_scale; e->scale_h = height_scale; e->offset_w = width_offset; e->offset_h = height_offset;
    *out = e.release();
    return MNNB200_OK;
}

mnnb200_status mnnb200_interp_f32_resize(mnnb200_exec* ex, int planes, int ih, int iw, int oh, int ow) {
    auto* e = exec_as<InterpF32Exec>(ex);
    if (!e) return fail(MNNB200_INVALID_VALUE, "interp_f32_resize: not a float Interp execution");
    if (e->resize_type < 1 || e->resize_type > 4)
        return fail(MNNB200_NOT_SUPPORT, "interp_f32_resize: resize type " + std::to_string(e->resize_type) + " (1-4 run here)");
    if (!std::isfinite(e->scale_w) || !std::isfinite(e->scale_h) || !std::isfinite(e->offset_w) || !std::isfinite(e->offset_h))
        return fail(MNNB200_NOT_SUPPORT, "interp_f32_resize: a non-finite scale or offset");
    if (planes <= 0 || ih <= 0 || iw <= 0 || oh <= 0 || ow <= 0) return fail(MNNB200_NOT_SUPPORT, "interp_f32_resize: empty tensor");
    const int taps = taps_of(e->resize_type);
    if ((long long)planes * ih * iw > 0x7fffffffLL || (long long)planes * oh * ow > 0x7fffffffLL ||
        (long long)oh * taps > 0x7fffffffLL || (long long)ow * taps > 0x7fffffffLL)
        return fail(MNNB200_NOT_SUPPORT, "interp_f32_resize: tensor too large for 32-bit indexing");
    std::vector<int> xi, yi;
    std::vector<float> xw, yw;
    axis_table(e->resize_type, e->scale_w, e->offset_w, iw, ow, xi, xw);
    axis_table(e->resize_type, e->scale_h, e->offset_h, ih, oh, yi, yw);
    cudaStream_t s = e->rt->stream;
    mnnb200_status st;
    if ((st = e->d_xi.upload(xi, s)) || (st = e->d_yi.upload(yi, s)) || (st = e->d_xw.upload(xw, s)) || (st = e->d_yw.upload(yw, s)))
        return st;
    InterpF32Params& p = e->p;
    memset(&p, 0, sizeof(p));
    p.xi = e->d_xi; p.xw = e->d_xw; p.yi = e->d_yi; p.yw = e->d_yw;
    p.planes = planes; p.ih = ih; p.iw = iw; p.oh = oh; p.ow = ow; p.taps = taps;
    e->last_vec = -1; e->last_grid = 0; e->last_row_groups = 0;
    e->cost_bytes = 4.0 * ((double)planes * ih * iw + (double)planes * oh * ow);
    e->cost_macs = (double)planes * oh * ow * (p.taps == 1 ? 0 : p.taps * (p.taps + 1));
    e->resized = true;
    return MNNB200_OK;
}

mnnb200_status mnnb200_interp_f32_execute(mnnb200_exec* ex, const float* x, float* y) {
    auto* e = exec_as<InterpF32Exec>(ex);
    if (!e) return fail(MNNB200_INVALID_VALUE, "interp_f32_execute: not a float Interp execution");
    if (!e->resized) return fail(MNNB200_NO_EXECUTION, "interp_f32_execute before resize");
    if (!x || !y) return fail(MNNB200_INVALID_VALUE, "interp_f32_execute: NULL tensor");
    InterpF32Params p = e->p;
    p.x = x; p.y = y;
    const int sm = e->rt->prop.multiProcessorCount;
    const bool vec = interp_f32_vec(p);
    int grid = 0, row_groups = 0;
    interp_f32_grid(p, vec, sm, &grid, &row_groups);
    CK(launch_interp_f32(p, sm, e->rt->stream));
    e->last_vec = vec ? 1 : 0; e->last_grid = grid; e->last_row_groups = row_groups;
    return MNNB200_OK;
}

mnnb200_status mnnb200_interp_f32_plan(mnnb200_exec* ex, int* fields, int count) {
    auto* e = exec_as<InterpF32Exec>(ex);
    if (!e || !fields || count < 0) return fail(MNNB200_INVALID_VALUE, "interp_f32_plan: bad argument");
    if (!e->resized) return fail(MNNB200_NO_EXECUTION, "interp_f32_plan before resize");
    const auto& p = e->p;
    const int v[] = {p.taps, e->last_vec, e->last_grid, kInterpThreads, e->last_row_groups, p.ow * p.taps, p.oh * p.taps};
    return copy_fields(v, fields, count);
}
}  // extern "C"
