// gather_capi.cu -- C ABI of libmnn_b200_gather.so (include/mnn_b200_gather.h): Gather / GatherV2 / GatherND / GatherElements
// and the int32 <-> fp32 Cast over the kernels of gather.cu, on the runtime and execution handles of libmnn_b200.so (exec.h).
//
// resize turns the two shapes into the kernels' geometry the way the reference's geometry stage lowers the ops to While loops
// (GeometryGather.cpp): Gather is outside x N slices of `inside` elements; GatherND is N tuples of d indices against the
// params' dims batch_dims .. batch_dims + d, with the strides buildGatherND computes (from the start of params: it adds no
// batch offset); GatherElements is GatherND with one full coordinate per output element.
#include <cuda_runtime.h>
#include <cstring>
#include <string>

#include "../../include/mnn_b200_gather.h"
#include "exec.h"
#include "gather_ops.h"

using namespace mnnb200;

struct GatherExec : Tagged<kGather> {
    int mode = 0;
    GatherParams p;
    GatherElementsParams pe;
    int last_path = -1, last_grid = 0, last_spt = 0;   // the last execute's launch since resize
};

namespace {

constexpr long long kMaxElems = 0x7fffffffLL;

long long product(const int* d, int from, int to) {
    long long n = 1;
    for (int i = from; i < to; ++i) n *= d[i];
    return n;
}

mnnb200_status refuse(const std::string& why) { return fail(MNNB200_NOT_SUPPORT, "gather_resize: " + why); }

}  // namespace

extern "C" {
mnnb200_status mnnb200_gather_create(mnnb200_runtime* rt, int mode, mnnb200_exec** out) {
    if (!rt || !out) return fail(MNNB200_INVALID_VALUE, "gather_create: NULL argument");
    if (mode < 0 || mode > 2) return fail(MNNB200_INVALID_VALUE, "gather_create: mode " + std::to_string(mode) + " (0-2)");
    auto e = new_exec<GatherExec>(rt);
    e->mode = mode;
    *out = e.release();
    return MNNB200_OK;
}

mnnb200_status mnnb200_gather_resize(mnnb200_exec* ex, const int* pd, int pr, const int* id, int ir, int axis) {
    auto* e = exec_as<GatherExec>(ex);
    if (!e) return fail(MNNB200_INVALID_VALUE, "gather_resize: not a gather execution");
    if ((pr > 0 && !pd) || (ir > 0 && !id)) return fail(MNNB200_INVALID_VALUE, "gather_resize: NULL shape");
    if (pr < 1 || ir < 1 || pr > kGatherMaxDims || ir > kGatherMaxDims) return refuse("rank outside 1-8");
    for (int i = 0; i < pr; ++i) if (pd[i] <= 0) return refuse("empty params");
    for (int i = 0; i < ir; ++i) if (id[i] <= 0) return refuse("empty indices");
    const long long np = product(pd, 0, pr), ni = product(id, 0, ir);
    if (np > kMaxElems || ni > kMaxElems) return refuse("more than 2^31 - 1 elements");
    GatherParams p;
    memset(&p, 0, sizeof(p));
    GatherElementsParams pe;
    memset(&pe, 0, sizeof(pe));
    long long nout;
    if (e->mode == 0) {
        if (axis < -pr || axis >= pr) return refuse("axis " + std::to_string(axis) + " of a rank-" + std::to_string(pr) + " tensor");
        if (axis < 0) axis += pr;
        p.outside = product(pd, 0, axis);
        p.n = ni;
        p.inside = product(pd, axis + 1, pr);
        p.d = 1;
        p.dim[0] = pd[axis];
        p.stride[0] = p.inside;
        p.x_outer = (long long)pd[axis] * p.inside;
        p.idx_outer = 0;
        nout = p.outside * p.n * p.inside;
    } else if (e->mode == 1) {
        const int d = id[ir - 1], b = axis;
        if (b < 0 || (b > 0 && b >= ir - 1)) return refuse("batch_dims " + std::to_string(b));
        if (d < 1 || d + b > pr) return refuse("an index tuple of " + std::to_string(d) + " past the params' rank");
        p.outside = 1;
        p.n = product(id, 0, ir - 1);
        p.inside = product(pd, b + d, pr);
        p.d = d;
        for (int k = 0; k < d; ++k) {
            p.dim[k] = pd[b + k];
            p.stride[k] = product(pd, b + k + 1, pr);
        }
        p.x_outer = 0;
        p.idx_outer = 0;
        nout = p.n * p.inside;
    } else {
        if (ir != pr) return refuse("indices of another rank than params");
        if (axis < -pr || axis >= pr) return refuse("axis " + std::to_string(axis) + " of a rank-" + std::to_string(pr) + " tensor");
        if (axis < 0) axis += pr;
        for (int k = 0; k < pr; ++k)
            if (k != axis && id[k] > pd[k]) return refuse("an index dimension past the params' outside the axis");
        pe.count = ni;
        pe.rank = pr;
        pe.axis = axis;
        pe.axis_len = pd[axis];
        for (int k = 0; k < pr; ++k) {
            pe.odim[k] = id[k];
            pe.xstride[k] = product(pd, k + 1, pr);
        }
        nout = ni;
    }
    if (nout > kMaxElems) return refuse("more than 2^31 - 1 output elements");
    e->p = p;
    e->pe = pe;
    e->last_path = -1;
    e->last_grid = 0;
    e->last_spt = 0;
    e->cost_bytes = 4.0 * (2.0 * (double)nout + (double)ni);
    e->cost_macs = 0;
    e->resized = true;
    return MNNB200_OK;
}

mnnb200_status mnnb200_gather_execute(mnnb200_exec* ex, const void* x, const int* idx, void* y) {
    auto* e = exec_as<GatherExec>(ex);
    if (!e) return fail(MNNB200_INVALID_VALUE, "gather_execute: not a gather execution");
    if (!e->resized) return fail(MNNB200_NO_EXECUTION, "gather_execute before resize");
    if (!x || !idx || !y) return fail(MNNB200_INVALID_VALUE, "gather_execute: NULL tensor");
    const int sm = e->rt->prop.multiProcessorCount;
    if (e->mode == 2) {
        GatherElementsParams pe = e->pe;
        pe.x = x; pe.idx = idx; pe.y = y;
        CK(launch_gather_elements(pe, sm, e->rt->stream));
        e->last_path = 0;
        e->last_grid = gather_elements_grid(pe.count, sm);
        return MNNB200_OK;
    }
    GatherParams p = e->p;
    p.x = x; p.idx = idx; p.y = y;
    CK(launch_gather(p, sm, e->rt->stream));
    const GatherLaunch l = gather_launch(p, sm);
    e->last_path = l.vec ? 1 : 0;
    e->last_grid = l.grid;
    e->last_spt = l.slices_per_tile;
    return MNNB200_OK;
}

mnnb200_status mnnb200_gather_plan(mnnb200_exec* ex, int* fields, int count) {
    auto* e = exec_as<GatherExec>(ex);
    if (!e || !fields || count < 0) return fail(MNNB200_INVALID_VALUE, "gather_plan: bad argument");
    if (!e->resized) return fail(MNNB200_NO_EXECUTION, "gather_plan before resize");
    const bool el = e->mode == 2;
    const int v[] = {e->mode, e->last_path, e->last_grid, kGatherThreads, e->last_spt, el ? 1 : (int)e->p.outside,
                     el ? (int)e->pe.count : (int)e->p.n, el ? 1 : (int)e->p.inside};
    return copy_fields(v, fields, count);
}

mnnb200_status mnnb200_cast_i32_f32(mnnb200_runtime* rt, const int* x, float* y, long long n) {
    if (!rt || n < 0 || (n > 0 && (!x || !y))) return fail(MNNB200_INVALID_VALUE, "cast_i32_f32: bad argument");
    CK(launch_cast_i32_f32(x, y, n, rt->prop.multiProcessorCount, rt->stream));
    return MNNB200_OK;
}

mnnb200_status mnnb200_cast_f32_i32(mnnb200_runtime* rt, const float* x, int* y, long long n) {
    if (!rt || n < 0 || (n > 0 && (!x || !y))) return fail(MNNB200_INVALID_VALUE, "cast_f32_i32: bad argument");
    CK(launch_cast_f32_i32(x, y, n, rt->prop.multiProcessorCount, rt->stream));
    return MNNB200_OK;
}
}  // extern "C"
