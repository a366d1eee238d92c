// scatter_capi.cu -- C ABI of libmnn_b200_scatter.so (include/mnn_b200_scatter.h): ScatterNd and ScatterElements over the
// kernels of scatter.cu, on the runtime and execution handles of libmnn_b200.so (exec.h).
//
// resize turns the shapes into the kernels' geometry the way GeometryScatter.cpp does before it builds its loop: ScatterNd
// (:176-205) has N = the indices' dims but the last, D = the last, S = the updates' dims from index D on, and strides the
// output's element strides of dims 0 .. D-1 (buildScatterND, :21-25); ScatterElements (:209-280) is the same loop over the
// indices' elements with one full coordinate each and S = 1.  Scratch is grown here, never in execute.
#include <cuda_runtime.h>
#include <algorithm>
#include <cstring>
#include <string>

#include "../../include/mnn_b200_scatter.h"
#include "exec.h"
#include "scatter_ops.h"

using namespace mnnb200;

struct ScatterExec : Tagged<kScatter> {
    int mode = 0, reduction = -1;
    bool with_data = true;
    ScatterParams p;
    int passes = 0;
    DevBuf<int> owner;
    DevBuf<unsigned> keys[2], vals[2], hist;
    ScatterLaunch last{};   // the last execute's launch since resize
    bool executed = false;
};

namespace {

constexpr long long kMaxElems = 0x7fffffffLL;

long long product(const int* d, int from, int to) {
    long long n = 1;
    for (int i = from; i < to; ++i) n *= d[i];
    return n;
}

mnnb200_status refuse(const std::string& why) { return fail(MNNB200_NOT_SUPPORT, "scatter_resize: " + why); }

}  // namespace

extern "C" {
mnnb200_status mnnb200_scatter_create(mnnb200_runtime* rt, int mode, int reduction, int with_data, mnnb200_exec** out) {
    if (!rt || !out) return fail(MNNB200_INVALID_VALUE, "scatter_create: NULL argument");
    if (mode < 0 || mode > 1) return fail(MNNB200_INVALID_VALUE, "scatter_create: mode " + std::to_string(mode) + " (0-1)");
    if (with_data < 0 || with_data > 1 || (mode == 1 && !with_data))
        return fail(MNNB200_INVALID_VALUE, "scatter_create: with_data " + std::to_string(with_data));
    if (reduction > 2)
        return fail(MNNB200_NOT_SUPPORT, "scatter_create: reduction " + std::to_string(reduction) + " (only ADD, SUB, MUL)");
    auto e = new_exec<ScatterExec>(rt);
    e->mode = mode;
    e->reduction = reduction < 0 ? -1 : reduction;
    e->with_data = with_data == 1;
    *out = e.release();
    return MNNB200_OK;
}

mnnb200_status mnnb200_scatter_resize(mnnb200_exec* ex, const int* od, int orank, const int* id, int irank, const int* ud,
                                      int urank, int axis, int is_int32) {
    auto* e = exec_as<ScatterExec>(ex);
    if (!e) return fail(MNNB200_INVALID_VALUE, "scatter_resize: not a scatter execution");
    if ((orank > 0 && !od) || (irank > 0 && !id) || (urank > 0 && !ud)) return fail(MNNB200_INVALID_VALUE, "scatter_resize: NULL shape");
    if (orank < 1 || irank < 1 || urank < 0 || orank > kScatterMaxDims || irank > kScatterMaxDims || urank > kScatterMaxDims)
        return refuse("rank outside 1-8");
    for (int i = 0; i < orank; ++i) if (od[i] <= 0) return refuse("empty output");
    for (int i = 0; i < irank; ++i) if (id[i] < 0) return refuse("a negative indices dimension");
    for (int i = 0; i < urank; ++i) if (ud[i] < 0) return refuse("a negative updates dimension");
    const long long total = product(od, 0, orank), ni = product(id, 0, irank), nu = product(ud, 0, urank);
    if (total > kMaxElems || ni > kMaxElems || nu > kMaxElems) return refuse("more than 2^31 - 1 elements");
    if (is_int32 && e->reduction >= 0) return refuse("an int32 scatter with a reduction");
    ScatterParams p;
    memset(&p, 0, sizeof(p));
    p.mode = e->mode;
    p.total = total;
    if (e->mode == 0) {
        const int d = id[irank - 1];
        if (d < 1 || d > orank) return refuse("an index tuple of " + std::to_string(d) + " into a rank-" + std::to_string(orank) + " output");
        p.d = d;
        p.n = product(id, 0, irank - 1);
        p.s = d < urank ? product(ud, d, urank) : 1;
        p.r = product(od, d, orank);
        for (int k = 0; k < d; ++k) p.stride[k] = (int)product(od, k + 1, orank);
    } else {
        if (irank != orank) return refuse("indices of another rank than the output");
        if (axis < -orank || axis >= orank) return refuse("axis " + std::to_string(axis) + " of a rank-" + std::to_string(orank) + " tensor");
        if (axis < 0) axis += orank;
        p.d = orank;
        p.axis = axis;
        p.n = ni;
        p.s = 1;
        p.r = 1;
        for (int k = 0; k < orank; ++k) {
            p.stride[k] = (int)product(od, k + 1, orank);
            p.idim[k] = id[k];
            p.istride[k] = product(id, k + 1, irank);
        }
    }
    if (p.s > p.r) return refuse("a slice of " + std::to_string(p.s) + " elements past the destination's " + std::to_string(p.r));
    if (nu < p.n * p.s) return refuse("fewer updates than N * S");
    p.x = p.total / p.r;
    const bool fold = e->reduction >= 0 && p.n > 0 && p.s > 0;
    const int passes = fold ? scatter_sort_passes(p.x) : 0;
    if (e->reduction < 0 && p.n > 0 && p.s > 0) {
        if (mnnb200_status st = e->owner.reserve((size_t)p.x)) return st;
        if (mnnb200_status st = e->keys[0].reserve((size_t)p.n)) return st;
    }
    if (fold) {
        const long long tiles = (p.n + kScatterTile - 1) / kScatterTile;
        for (int b = 0; b < 2; ++b) {
            if (mnnb200_status st = e->keys[b].reserve((size_t)p.n)) return st;
            if (mnnb200_status st = e->vals[b].reserve((size_t)p.n)) return st;
        }
        if (mnnb200_status st = e->hist.reserve((size_t)(kScatterDigits * (tiles + 1)))) return st;
    }
    e->p = p;
    e->passes = passes;
    e->last = ScatterLaunch{};
    e->executed = false;
    e->cost_bytes = 4.0 * ((e->with_data ? 2.0 : 1.0) * (double)total + (double)(p.n * p.s) + (double)p.n * (e->mode == 0 ? p.d : 1));
    e->cost_macs = 0;
    e->resized = true;
    return MNNB200_OK;
}

mnnb200_status mnnb200_scatter_execute(mnnb200_exec* ex, const void* data, const int* idx, const void* upd, void* y) {
    auto* e = exec_as<ScatterExec>(ex);
    if (!e) return fail(MNNB200_INVALID_VALUE, "scatter_execute: not a scatter execution");
    if (!e->resized) return fail(MNNB200_NO_EXECUTION, "scatter_execute before resize");
    if (!y || (e->with_data != (data != nullptr))) return fail(MNNB200_INVALID_VALUE, "scatter_execute: NULL output, or data against create");
    if (e->p.n > 0 && e->p.s > 0 && (!idx || !upd)) return fail(MNNB200_INVALID_VALUE, "scatter_execute: NULL indices or updates");
    const int sm = e->rt->prop.multiProcessorCount;
    ScatterParams p = e->p;
    p.data = data; p.idx = idx; p.upd = upd; p.y = y;
    const ScatterScratch w{e->owner, {e->keys[0], e->keys[1]}, {e->vals[0], e->vals[1]}, e->hist};
    CK(launch_scatter(p, e->reduction, std::max(e->passes, 1), w, sm, e->rt->stream));
    e->last = scatter_launch(p, e->reduction, e->passes, sm);
    e->executed = true;
    return MNNB200_OK;
}

mnnb200_status mnnb200_scatter_plan(mnnb200_exec* ex, int* fields, int count) {
    auto* e = exec_as<ScatterExec>(ex);
    if (!e || !fields || count < 0) return fail(MNNB200_INVALID_VALUE, "scatter_plan: bad argument");
    if (!e->resized) return fail(MNNB200_NO_EXECUTION, "scatter_plan before resize");
    const ScatterLaunch& l = e->last;
    const int v[] = {e->mode, e->reduction, (int)e->p.n, (int)e->p.s, (int)e->p.r, (int)e->p.x, e->executed ? l.path : -1,
                     e->passes, e->executed ? l.launches : 0, e->executed ? l.vec : 0, e->executed ? l.init_vec : 0,
                     e->executed ? l.grid : 0};
    return copy_fields(v, fields, count);
}
}  // extern "C"
