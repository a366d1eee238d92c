// grid_sample_capi.cu -- C ABI of libmnn_b200_grid_sample.so (include/mnn_b200_grid_sample.h): the fp32 GridSample execution
// (CPUGridSample) on NCHW-linear fp32 tensors, over the kernel of grid_sample_f32.cu, on the runtime and execution handles of
// libmnn_b200.so (exec.h).
//
// resize fixes the shape, the per-axis coordinate constants (computed here in the CPU's float expressions; this host code is
// compiled with -ffp-contract=off) and the channel groups: a shape whose n * pixels work items fill the card (kFill per SM) runs
// one group of all channels, a shape with fewer pixels splits its channels into the fewest groups that reach kFill items per SM.
#include <cuda_runtime.h>
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <string>

#include "../../include/mnn_b200_grid_sample.h"
#include "exec.h"
#include "grid_sample_ops.h"

using namespace mnnb200;

namespace {
// work items (threads) per SM the channel groups aim for: 8 CTAs of 256 threads, one full wave at full occupancy
constexpr long long kFill = 2048;
}  // namespace

struct GridSampleF32Exec : Tagged<kGridSampleF32> {
    bool nearest = false, zeros = false, align = false;
    int rank = 0;
    GridSampleF32Params p;
    int grid = 0;
    int last_vec = -1;   // the last execute's grid-read path since resize
};

extern "C" {
mnnb200_status mnnb200_grid_sample_f32_create(mnnb200_runtime* rt, int mode, int padding, int align_corners, mnnb200_exec** out) {
    if (!rt || !out) return fail(MNNB200_INVALID_VALUE, "grid_sample_f32_create: NULL argument");
    if (mode < 0 || mode > 1) return fail(MNNB200_NOT_SUPPORT, "grid_sample_f32_create: mode " + std::to_string(mode) + " (0-1 run here)");
    if (padding < 0 || padding > 2)
        return fail(MNNB200_NOT_SUPPORT, "grid_sample_f32_create: padding " + std::to_string(padding) + " (0-2 run here)");
    auto e = new_exec<GridSampleF32Exec>(rt);
    e->nearest = mode == 1;
    e->zeros = padding == 0;   // REFLECTION (2) samples as CLAMP (1), as the CPU does
    e->align = align_corners != 0;
    *out = e.release();
    return MNNB200_OK;
}

mnnb200_status mnnb200_grid_sample_f32_resize(mnnb200_exec* ex, int rank, int n, int c, const int* in_dims, const int* out_dims) {
    auto* e = exec_as<GridSampleF32Exec>(ex);
    if (!e) return fail(MNNB200_INVALID_VALUE, "grid_sample_f32_resize: not a float GridSample execution");
    if (rank != 4 && rank != 5) return fail(MNNB200_NOT_SUPPORT, "grid_sample_f32_resize: rank " + std::to_string(rank) + " (4-5 run here)");
    if (!in_dims || !out_dims) return fail(MNNB200_INVALID_VALUE, "grid_sample_f32_resize: NULL dims");
    const int sp = rank - 2;
    long long in_el = 1, out_px = 1;
    bool empty = n <= 0 || c <= 0;
    for (int i = 0; i < sp; ++i) {
        empty = empty || in_dims[i] <= 0 || out_dims[i] <= 0;
        in_el *= std::max(in_dims[i], 0);
        out_px *= std::max(out_dims[i], 0);
    }
    if (empty) return fail(MNNB200_NOT_SUPPORT, "grid_sample_f32_resize: empty tensor");
    const long long lim = 0x7fffffffLL;
    if ((long long)n * c * in_el > lim || (long long)n * out_px * sp > lim || (long long)n * c * out_px > lim)
        return fail(MNNB200_NOT_SUPPORT, "grid_sample_f32_resize: tensor too large for 32-bit indexing");
    GridSampleF32Params& p = e->p;
    memset(&p, 0, sizeof(p));
    p.n = n; p.c = c; p.pixels = (int)out_px;
    p.id = rank == 5 ? in_dims[0] : 1;
    p.ih = in_dims[sp - 2];
    p.iw = in_dims[sp - 1];
    // the CPU's constants: a = 1, b = 0 with alignCorners, else a = 0, b = 1; axes in grid order x (W), y (H), z (D)
    const float a = e->align ? 1.0f : 0.0f, b = e->align ? 0.0f : 1.0f;
    const int axis_in[3] = {p.iw, p.ih, p.id};
    for (int i = 0; i < sp; ++i) {
        const float in = (float)axis_in[i];
        p.in_a[i] = in - a;                       // _mm512_set1_ps(inW) - a
        p.k[i] = 0.5f * (in - a);                 // kx = 0.5f * ((float)inW - a)
        p.k0[i] = 0.5f * (in - a - b);            // bx = 0.5f * ((float)inW - a - b)
    }
    p.b = b;
    const int sm = e->rt->prop.multiProcessorCount > 0 ? e->rt->prop.multiProcessorCount : 1;
    const long long items = (long long)n * out_px;
    const long long groups = std::min<long long>(c, std::max<long long>(1, (kFill * sm + items - 1) / items));
    p.cper = (int)((c + groups - 1) / groups);
    p.cgroups = (c + p.cper - 1) / p.cper;
    e->rank = rank;
    e->grid = grid_sample_f32_grid(p, sm);
    e->last_vec = -1;
    const int taps = e->nearest ? 1 : (rank == 5 ? 8 : 4);
    e->cost_bytes = 4.0 * ((double)n * c * in_el + (double)n * out_px * sp + (double)n * c * out_px);
    e->cost_macs = e->nearest ? 0.0 : (double)n * c * out_px * (taps - 1);
    e->resized = true;
    return MNNB200_OK;
}

mnnb200_status mnnb200_grid_sample_f32_execute(mnnb200_exec* ex, const float* x, const float* grid, float* y) {
    auto* e = exec_as<GridSampleF32Exec>(ex);
    if (!e) return fail(MNNB200_INVALID_VALUE, "grid_sample_f32_execute: not a float GridSample execution");
    if (!e->resized) return fail(MNNB200_NO_EXECUTION, "grid_sample_f32_execute before resize");
    if (!x || !grid || !y) return fail(MNNB200_INVALID_VALUE, "grid_sample_f32_execute: NULL tensor");
    GridSampleF32Params p = e->p;
    p.x = x; p.grid = grid; p.y = y;
    const bool vec2 = e->rank == 4 && ((uintptr_t)grid & 7) == 0;
    CK(launch_grid_sample_f32(p, e->rank, e->nearest, e->zeros, vec2, e->rt->prop.multiProcessorCount, e->rt->stream));
    e->last_vec = vec2 ? 1 : 0;
    return MNNB200_OK;
}

mnnb200_status mnnb200_grid_sample_f32_plan(mnnb200_exec* ex, int* fields, int count) {
    auto* e = exec_as<GridSampleF32Exec>(ex);
    if (!e || !fields || count < 0) return fail(MNNB200_INVALID_VALUE, "grid_sample_f32_plan: bad argument");
    if (!e->resized) return fail(MNNB200_NO_EXECUTION, "grid_sample_f32_plan before resize");
    const int taps = e->nearest ? 1 : (e->rank == 5 ? 8 : 4);
    const int v[] = {e->rank, taps, e->p.cgroups, e->p.cper, e->grid, kGridSampleThreads, e->last_vec};
    return copy_fields(v, fields, count);
}
}  // extern "C"
