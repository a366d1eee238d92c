// rnn_capi.cu -- C ABI of libmnn_b200_rnn.so (include/mnn_b200_rnn.h): LSTM and RNN as the split-TF32 projection MatMul of
// libmnn_b200.so followed by the recurrence kernel of rnn.cu, on the runtime and execution handles of libmnn_b200.so (exec.h).
//
// W is [D * G * H][I] and the bias [D * G * H], both contiguous, so one MatMul C[T * B][D * G * H] = X W^T + bias gives both
// directions' gates; rows are independent, so direction 1's reversal in time is only indexing in the recurrence.  The Gate
// scratch and the MatMul are made here; the MatMul allocates its own packing scratch at its first execute, so resize runs one
// warm-up execute of it (on the stream, no host read) and every later execute allocates nothing and can be captured.
#include <cuda_runtime.h>
#include <algorithm>
#include <string>

#include "../../include/mnn_b200_rnn.h"
#include "exec.h"
#include "rnn_ops.h"

using namespace mnnb200;

struct RnnExec : Tagged<kRnn> {
    int cell = 0;
    int t = 0, b = 0, i = 0, h = 0, d = 0;
    bool has_h0 = false, has_c0 = false;
    RnnPlan plan;
    mnnb200_exec* mm = nullptr;   // the projection, for (mm_rows, mm_i, mm_cols)
    long long mm_rows = 0, mm_i = 0, mm_cols = 0;
    DevBuf<float> gates;
    ~RnnExec() override {
        if (mm) mnnb200_exec_destroy(mm);
    }
};

namespace {

constexpr long long kMaxElems = 0x7fffffffLL;

mnnb200_status refuse(const std::string& why) { return fail(MNNB200_NOT_SUPPORT, "rnn_resize: " + why); }

struct FitsCtx {
    int smem_cap;
    cudaError_t err;
};
bool cluster_fits(int cell, const RnnPlan& pl, void* ctx) {
    auto* c = static_cast<FitsCtx*>(ctx);
    int n = 0;
    const cudaError_t e = rnn_max_active_clusters(cell, pl, c->smem_cap, &n);
    if (e != cudaSuccess) {
        cudaGetLastError();
        c->err = e;
        return false;
    }
    return n > 0;
}

}  // namespace

extern "C" {
mnnb200_status mnnb200_rnn_create(mnnb200_runtime* rt, int cell, mnnb200_exec** out) {
    if (!rt || !out) return fail(MNNB200_INVALID_VALUE, "rnn_create: NULL argument");
    if (cell < 0 || cell > 1) return fail(MNNB200_INVALID_VALUE, "rnn_create: cell " + std::to_string(cell) + " (0 LSTM, 1 RNN)");
    auto e = new_exec<RnnExec>(rt);
    e->cell = cell;
    *out = e.release();
    return MNNB200_OK;
}

mnnb200_status mnnb200_rnn_resize(mnnb200_exec* ex, int T, int B, int I, int H, int D, int has_h0, int has_c0) {
    auto* e = exec_as<RnnExec>(ex);
    if (!e) return fail(MNNB200_INVALID_VALUE, "rnn_resize: not an LSTM / RNN execution");
    if (has_h0 < 0 || has_h0 > 1 || has_c0 < 0 || has_c0 > 1 || (e->cell == 1 && has_c0))
        return fail(MNNB200_INVALID_VALUE, "rnn_resize: has_h0 / has_c0 (an RNN has no cell state)");
    if (T < 1 || B < 1 || I < 1 || H < 1) return refuse("an empty dimension");
    if (D < 1 || D > 2) return refuse("D " + std::to_string(D) + " (1 or 2)");
    if (H > kRnnMaxHidden) return refuse("H " + std::to_string(H) + " past " + std::to_string(kRnnMaxHidden));
    const long long ng = e->cell == 0 ? 4 : 1, rows = (long long)T * B, cols = (long long)D * ng * H;
    if (rows * I > kMaxElems || cols * I > kMaxElems || cols * H > kMaxElems || rows * D * H > kMaxElems || rows * cols > kMaxElems)
        return refuse("a tensor of more than 2^31 - 1 elements");
    const cudaDeviceProp& prop = e->rt->prop;
    FitsCtx ctx{(int)prop.sharedMemPerBlockOptin, cudaSuccess};
    RnnPlan plan;
    if (!rnn_choose_plan(e->cell, B, H, D, prop.multiProcessorCount, ctx.smem_cap, cluster_fits, &ctx, &plan)) {
        if (ctx.err != cudaSuccess) return fail(MNNB200_CUDA_ERROR, std::string("rnn_resize: ") + cudaGetErrorString(ctx.err));
        return refuse("no cluster of the recurrence fits on the device");
    }
    if (plan.groups > 65535) return refuse("more than 65535 batch groups");
    mnnb200_exec* mm = e->mm;
    if (!mm || e->mm_rows != rows || e->mm_i != I || e->mm_cols != cols) {
        mm = nullptr;
        if (mnnb200_status st = mnnb200_matmul_create(e->rt, 1, (int)rows, I, (int)cols, 0, 1, 0, &mm)) return st;
    }
    mnnb200_status st = e->gates.reserve((size_t)(rows * cols));
    if (!st && mm != e->mm) {   // the warm-up execute: the new MatMul allocates its packing scratch here, not in execute
        DevBuf<float> zeros;
        const size_t n = (size_t)std::max(rows, cols) * I;
        st = zeros.reserve(n);
        if (!st && cudaMemsetAsync(zeros, 0, n * sizeof(float), e->rt->stream) != cudaSuccess) {
            cudaGetLastError();
            st = fail(MNNB200_CUDA_ERROR, "rnn_resize: memset");
        }
        if (!st) st = mnnb200_matmul_execute(mm, zeros, zeros, nullptr, e->gates);
        if (!st && cudaStreamSynchronize(e->rt->stream) != cudaSuccess) {   // before `zeros` is freed
            cudaGetLastError();
            st = fail(MNNB200_CUDA_ERROR, "rnn_resize: warm-up");
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
    e->has_c0 = has_c0 == 1;
    e->plan = plan;
    e->cost_bytes = 4.0 * ((double)rows * I + (double)cols * (I + H + 1) + 2.0 * (double)rows * cols + (double)rows * D * H);
    e->cost_macs = (double)rows * cols * I + (double)rows * cols * H;
    e->resized = true;
    return MNNB200_OK;
}

mnnb200_status mnnb200_rnn_execute(mnnb200_exec* ex, const float* x, const float* w, const float* r, const float* bias,
                                   const float* h0, const float* c0, float* y, float* y_h, float* y_c) {
    auto* e = exec_as<RnnExec>(ex);
    if (!e) return fail(MNNB200_INVALID_VALUE, "rnn_execute: not an LSTM / RNN execution");
    if (!e->resized) return fail(MNNB200_NO_EXECUTION, "rnn_execute before resize");
    if (!x || !w || !r || !y) return fail(MNNB200_INVALID_VALUE, "rnn_execute: NULL x, w, r or y");
    if (e->has_h0 != (h0 != nullptr) || e->has_c0 != (c0 != nullptr))
        return fail(MNNB200_INVALID_VALUE, "rnn_execute: h0 / c0 against resize");
    if (mnnb200_status st = mnnb200_matmul_execute(e->mm, x, w, bias, e->gates)) return st;
    RnnParams p;
    p.g = e->gates;
    p.r = r;
    p.h0 = h0;
    p.c0 = c0;
    p.y = y;
    p.yh = y_h;
    p.yc = e->cell == 0 ? y_c : nullptr;
    p.t = e->t; p.b = e->b; p.h = e->h; p.d = e->d;
    p.cs = e->plan.cs;
    p.rows = e->plan.rows;
    p.hs = e->plan.hs;
    p.rstride = e->plan.rstride;
    CK(launch_rnn_recur(e->cell, p, e->plan, e->rt->stream));
    return MNNB200_OK;
}

mnnb200_status mnnb200_rnn_plan(mnnb200_exec* ex, int* fields, int count) {
    auto* e = exec_as<RnnExec>(ex);
    if (!e || !fields || count < 0) return fail(MNNB200_INVALID_VALUE, "rnn_plan: bad argument");
    if (!e->resized) return fail(MNNB200_NO_EXECUTION, "rnn_plan before resize");
    const RnnPlan& l = e->plan;
    const long long scratch = 4LL * e->mm_rows * e->mm_cols;
    const int v[] = {e->cell, e->t, e->b, e->i, e->h, e->d, l.cs, l.groups, l.rows, l.resident, l.smem,
                     scratch > 0x7fffffffLL ? 0x7fffffff : (int)scratch, 1, l.ks};
    return copy_fields(v, fields, count);
}
}  // extern "C"
