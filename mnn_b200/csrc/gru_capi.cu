// gru_capi.cu -- C ABI of libmnn_b200_gru.so (include/mnn_b200_gru.h): the GRU as a weight repack, the split-TF32 projection
// MatMul of libmnn_b200.so and the recurrence kernel of gru.cu, on the runtime and execution handles of libmnn_b200.so (exec.h).
//
// The repack writes the x parts of both directions' weights as one [I][D * 3H] matrix, so that one MatMul P[T * B][D * 3H] =
// X Wx + bx gives every step's x terms of both directions.  It runs every execute (a captured graph replays with new weights)
// and reads (I + H) * 3H * D floats once.  The scratch and the MatMul are made at resize; a new MatMul runs once there on zeroed
// operands so that it allocates its packing scratch then, and every execute allocates nothing and can be captured.
#include <cuda_runtime.h>
#include <algorithm>
#include <string>

#include "../../include/mnn_b200_gru.h"
#include "exec.h"
#include "gru_ops.h"

using namespace mnnb200;

struct GruExec : Tagged<kGru> {
    int lbr = 0;
    int t = 0, b = 0, i = 0, h = 0, d = 0;
    bool has_h0 = false;
    RnnPlan plan;
    mnnb200_exec* mm = nullptr;   // the projection, for (mm_rows, mm_i, mm_cols)
    long long mm_rows = 0, mm_i = 0, mm_cols = 0;
    DevBuf<float> gates, wx, r, bx, kb;
    ~GruExec() override {
        if (mm) mnnb200_exec_destroy(mm);
    }
};

namespace {

constexpr long long kMaxElems = 0x7fffffffLL;

mnnb200_status refuse(const std::string& why) { return fail(MNNB200_NOT_SUPPORT, "gru_resize: " + why); }

struct FitsCtx {
    int smem_cap;
    cudaError_t err;
};
bool cluster_fits(int lbr, const RnnPlan& pl, void* ctx) {
    auto* c = static_cast<FitsCtx*>(ctx);
    int n = 0;
    const cudaError_t e = gru_max_active_clusters(lbr, pl, c->smem_cap, &n);
    if (e != cudaSuccess) {
        cudaGetLastError();
        c->err = e;
        return false;
    }
    return n > 0;
}

}  // namespace

extern "C" {
mnnb200_status mnnb200_gru_create(mnnb200_runtime* rt, int linear_before_reset, mnnb200_exec** out) {
    if (!rt || !out) return fail(MNNB200_INVALID_VALUE, "gru_create: NULL argument");
    if (linear_before_reset < 0 || linear_before_reset > 1)
        return fail(MNNB200_INVALID_VALUE, "gru_create: linear_before_reset " + std::to_string(linear_before_reset) + " (0 or 1)");
    auto e = new_exec<GruExec>(rt);
    e->lbr = linear_before_reset;
    *out = e.release();
    return MNNB200_OK;
}

mnnb200_status mnnb200_gru_resize(mnnb200_exec* ex, int T, int B, int I, int H, int D, int has_h0) {
    auto* e = exec_as<GruExec>(ex);
    if (!e) return fail(MNNB200_INVALID_VALUE, "gru_resize: not a GRU execution");
    if (has_h0 < 0 || has_h0 > 1) return fail(MNNB200_INVALID_VALUE, "gru_resize: has_h0 " + std::to_string(has_h0));
    if (T < 1 || B < 1 || I < 1 || H < 1) return refuse("an empty dimension");
    if (D < 1 || D > 2) return refuse("D " + std::to_string(D) + " (1 or 2)");
    if (H > kRnnMaxHidden) return refuse("H " + std::to_string(H) + " past " + std::to_string(kRnnMaxHidden));
    const long long rows = (long long)T * B, cols = (long long)D * 3 * H;
    if (rows * I > kMaxElems || (long long)(I + H) * cols > kMaxElems || cols * H > kMaxElems || rows * D * H > kMaxElems ||
        rows * cols > kMaxElems)
        return refuse("a tensor of more than 2^31 - 1 elements");
    const cudaDeviceProp& prop = e->rt->prop;
    FitsCtx ctx{(int)prop.sharedMemPerBlockOptin, cudaSuccess};
    RnnPlan plan;
    if (!gru_choose_plan(e->lbr, B, H, D, prop.multiProcessorCount, ctx.smem_cap, cluster_fits, &ctx, &plan)) {
        if (ctx.err != cudaSuccess) return fail(MNNB200_CUDA_ERROR, std::string("gru_resize: ") + cudaGetErrorString(ctx.err));
        return refuse("no cluster of the recurrence fits on the device");
    }
    if (plan.groups > 65535) return refuse("more than 65535 batch groups");
    mnnb200_exec* mm = e->mm;
    if (!mm || e->mm_rows != rows || e->mm_i != I || e->mm_cols != cols) {
        mm = nullptr;
        if (mnnb200_status st = mnnb200_matmul_create(e->rt, 1, (int)rows, I, (int)cols, 0, 0, 0, &mm)) return st;
    }
    mnnb200_status st = e->gates.reserve((size_t)(rows * cols));
    if (!st) st = e->wx.reserve((size_t)(I * cols));
    if (!st) st = e->r.reserve((size_t)(cols * H));
    if (!st) st = e->bx.reserve((size_t)cols);
    if (!st) st = e->kb.reserve((size_t)D * 4 * H);
    if (!st && mm != e->mm) {   // the warm-up execute: the new MatMul allocates its packing scratch here, not in execute
        DevBuf<float> zeros;
        const size_t n = (size_t)std::max(rows, cols) * I;
        st = zeros.reserve(n);
        if (!st && cudaMemsetAsync(zeros, 0, n * sizeof(float), e->rt->stream) != cudaSuccess) {
            cudaGetLastError();
            st = fail(MNNB200_CUDA_ERROR, "gru_resize: memset");
        }
        if (!st) st = mnnb200_matmul_execute(mm, zeros, zeros, nullptr, e->gates);
        if (!st && cudaStreamSynchronize(e->rt->stream) != cudaSuccess) {   // before `zeros` is freed
            cudaGetLastError();
            st = fail(MNNB200_CUDA_ERROR, "gru_resize: warm-up");
        }
    }
    if (st) {
        if (mm != e->mm) mnnb200_exec_destroy(mm);
        return st;
    }
    if (mm != e->mm) {
        if (e->mm) mnnb200_exec_destroy(e->mm);
        e->mm = mm;
        e->mm_rows = rows;
        e->mm_i = I;
        e->mm_cols = cols;
    }
    e->t = T; e->b = B; e->i = I; e->h = H; e->d = D;
    e->has_h0 = has_h0 == 1;
    e->plan = plan;
    e->cost_bytes = 4.0 * ((double)rows * I + 2.0 * (double)cols * (I + H + 1) + 2.0 * (double)rows * cols + (double)rows * D * H);
    e->cost_macs = (double)rows * cols * I + (double)rows * cols * H;
    e->resized = true;
    return MNNB200_OK;
}

mnnb200_status mnnb200_gru_execute(mnnb200_exec* ex, const float* x, const float* const* params, const float* h0, float* y,
                                   float* y_h) {
    auto* e = exec_as<GruExec>(ex);
    if (!e) return fail(MNNB200_INVALID_VALUE, "gru_execute: not a GRU execution");
    if (!e->resized) return fail(MNNB200_NO_EXECUTION, "gru_execute before resize");
    if (!x || !params || (!y && !y_h)) return fail(MNNB200_INVALID_VALUE, "gru_execute: NULL x or params, or both outputs NULL");
    for (int k = 0; k < kGruParamsPerDir * e->d; ++k)
        if (!params[k]) return fail(MNNB200_INVALID_VALUE, "gru_execute: NULL weight " + std::to_string(k));
    if (e->has_h0 != (h0 != nullptr)) return fail(MNNB200_INVALID_VALUE, "gru_execute: h0 against resize");
    GruRepackParams rp = {};
    for (int k = 0; k < kGruParamsPerDir * e->d; ++k) rp.in[k] = params[k];
    rp.wx = e->wx;
    rp.r = e->r;
    rp.bx = e->bx;
    rp.kb = e->kb;
    rp.i = e->i; rp.h = e->h; rp.d = e->d;
    CK(launch_gru_repack(rp, e->rt->stream));
    if (mnnb200_status st = mnnb200_matmul_execute(e->mm, x, e->wx, e->bx, e->gates)) return st;
    GruParams p;
    p.g = e->gates;
    p.r = e->r;
    p.kb = e->kb;
    p.h0 = h0;
    p.y = y;
    p.yh = y_h;
    p.t = e->t; p.b = e->b; p.h = e->h; p.d = e->d;
    p.cs = e->plan.cs;
    p.rows = e->plan.rows;
    p.hs = e->plan.hs;
    p.rstride = e->plan.rstride;
    CK(launch_gru_recur(e->lbr, p, e->plan, e->rt->stream));
    return MNNB200_OK;
}

mnnb200_status mnnb200_gru_plan(mnnb200_exec* ex, int* fields, int count) {
    auto* e = exec_as<GruExec>(ex);
    if (!e || !fields || count < 0) return fail(MNNB200_INVALID_VALUE, "gru_plan: bad argument");
    if (!e->resized) return fail(MNNB200_NO_EXECUTION, "gru_plan before resize");
    const RnnPlan& l = e->plan;
    const long long cols = e->mm_cols;
    const long long scratch = 4LL * (e->mm_rows * cols + e->mm_i * cols + cols * e->h + cols + 4LL * e->d * e->h);
    const int v[] = {e->lbr, e->t, e->b, e->i, e->h, e->d, l.cs, l.groups, l.rows, l.resident, l.smem,
                     scratch > 0x7fffffffLL ? 0x7fffffff : (int)scratch, 3, l.ks};
    return copy_fields(v, fields, count);
}
}  // extern "C"
