// llm_capi.cu -- C ABI of libmnn_b200_llm.so (include/mnn_b200_llm.h): the LayerNorm / RMSNorm and fused RoPE executions over
// the kernels of llm_ops.cu, on the runtime and execution handles of libmnn_b200.so (exec.h).
#include <cuda_runtime.h>
#include <string>
#include <vector>

#include "../../include/mnn_b200_llm.h"
#include "exec.h"
#include "llm_ops.h"

using namespace mnnb200;

// ---- LayerNorm / RMSNorm and fused RoPE of MNN-LLM's decoder layers (llm_ops.cu)
struct LayerNormF32Exec : Tagged<kLayerNormF32> {
    LayerNormParams p{};   // everything but the tensors; rows = 0 until the first resize
    DevBuf<float> d_gamma, d_beta;
};
struct RoPEF32Exec : Tagged<kRoPEF32> {
    RopeParams p{};
    DevBuf<float> d_qg, d_qb, d_kg, d_kb;
};

extern "C" {
// CPULayerNorm::makeResource (CPULayerNorm.cpp:25-68): gamma / beta copied once to the device; the affine transform exists only when
// both are given (:35), so a gamma alone is ignored as the CPU ignores it
mnnb200_status mnnb200_layernorm_f32_create(mnnb200_runtime* rt, int inner, float eps, int rms, const float* gamma, const float* beta,
                                            int affine_size, mnnb200_exec** out) {
    if (!rt || !out || inner <= 0) return fail(MNNB200_INVALID_VALUE, "layernorm_f32_create: bad argument");
    if (!layernorm_f32_threads(inner, nullptr))
        return fail(MNNB200_NOT_SUPPORT, "layernorm_f32_create: a row of more than 32768 elements does not fit in registers");
    const bool affine = gamma && beta;
    if (affine && affine_size != inner)
        return fail(MNNB200_NOT_SUPPORT, "layernorm_f32_create: gamma / beta size " + std::to_string(affine_size) + " != inner " +
                                             std::to_string(inner));
    auto e = new_exec<LayerNormF32Exec>(rt);
    mnnb200_status st;
    if (affine && ((st = e->d_gamma.upload(std::vector<float>(gamma, gamma + inner), rt->stream)) ||
                   (st = e->d_beta.upload(std::vector<float>(beta, beta + inner), rt->stream))))
        return st;
    e->p.inner = inner; e->p.eps = eps; e->p.rms = rms ? 1 : 0;
    e->p.gamma = affine ? (const float*)e->d_gamma : nullptr;
    e->p.beta = affine ? (const float*)e->d_beta : nullptr;
    *out = e.release();
    return MNNB200_OK;
}

// CPULayerNorm::onResize (CPULayerNorm.cpp:228-284): the caller passes the rows of the [rows][inner] view (outer size, or
// length(0) * group for a grouped norm).  A refused resize keeps the previous plan.
mnnb200_status mnnb200_layernorm_f32_resize(mnnb200_exec* ex, int rows) {
    auto* e = exec_as<LayerNormF32Exec>(ex);
    if (!e) return fail(MNNB200_INVALID_VALUE, "layernorm_f32_resize: not a LayerNorm execution");
    if (rows <= 0) return fail(MNNB200_NOT_SUPPORT, "layernorm_f32_resize: zero rows");
    if ((long long)rows * e->p.inner > 0x7fffffffLL) return fail(MNNB200_NOT_SUPPORT, "layernorm_f32_resize: tensor too large for 32-bit indexing");
    e->p.rows = rows;
    e->cost_bytes = 8.0 * rows * (double)e->p.inner;
    e->cost_macs = 0;
    e->resized = true;
    return MNNB200_OK;
}

// CPULayerNorm::onExecute (CPULayerNorm.cpp:70-226): y = norm(x); the residual form (NC4HW4 2-in / 2-out, :93-153) also takes
// residual and sum: sum = x + residual, y = norm(sum), one pass
mnnb200_status mnnb200_layernorm_f32_execute(mnnb200_exec* ex, const float* x, const float* residual, float* sum, float* y) {
    auto* e = exec_as<LayerNormF32Exec>(ex);
    if (!e) return fail(MNNB200_INVALID_VALUE, "layernorm_f32_execute: not a LayerNorm execution");
    if (!e->resized) return fail(MNNB200_NO_EXECUTION, "layernorm_f32_execute before resize");
    if (!x || !y || !residual != !sum) return fail(MNNB200_INVALID_VALUE, "layernorm_f32_execute: NULL tensor (residual and sum go together)");
    LayerNormParams p = e->p;
    p.x = x; p.r = residual; p.s = sum; p.y = y;
    CK(launch_layernorm_f32(p, e->rt->stream));
    return MNNB200_OK;
}

// CPURoPE's constructor (CPURoPE.cpp:20-49, 86-96): a q / k norm table (RoPEParam.q_norm / k_norm) is copied to the device, beta
// zero-filled when the table has none
mnnb200_status mnnb200_rope_f32_create(mnnb200_runtime* rt, int heads, int kv_heads, int head_dim, int rope_cut,
                                       const mnnb200_rope_norm* q_norm, const mnnb200_rope_norm* k_norm, mnnb200_exec** out) {
    if (!rt || !out) return fail(MNNB200_INVALID_VALUE, "rope_f32_create: NULL argument");
    if (heads <= 0 || kv_heads <= 0 || head_dim <= 0) return fail(MNNB200_NOT_SUPPORT, "rope_f32_create: heads, kv_heads and head_dim must be > 0");
    for (const mnnb200_rope_norm* n : {q_norm, k_norm})
        if (n && (!n->gamma || n->size != head_dim))
            return fail(MNNB200_NOT_SUPPORT, "rope_f32_create: a q / k norm needs gamma of head_dim values");
    auto e = new_exec<RoPEF32Exec>(rt);
    RopeParams& p = e->p;
    p.heads = heads; p.kv_heads = kv_heads; p.head_dim = head_dim;
    // ropeDim = rope_cut_head_dim in (0, head_dim], else head_dim, rounded down to even (CPURoPE.cpp:176-180)
    p.rope_dim = (rope_cut <= 0 || rope_cut > head_dim ? head_dim : rope_cut) / 2 * 2;
    auto table = [&](const mnnb200_rope_norm* n, DevBuf<float>& dg, DevBuf<float>& db, RopeNorm& rn) -> mnnb200_status {
        rn = RopeNorm{nullptr, nullptr, 0.f, 0};
        if (!n) return MNNB200_OK;
        std::vector<float> b(head_dim, 0.f);
        if (n->beta) b.assign(n->beta, n->beta + head_dim);
        mnnb200_status st;
        if ((st = dg.upload(std::vector<float>(n->gamma, n->gamma + head_dim), rt->stream)) || (st = db.upload(b, rt->stream))) return st;
        rn = RopeNorm{dg, db, n->eps, n->rms ? 1 : 0};
        return MNNB200_OK;
    };
    mnnb200_status st;
    if ((st = table(q_norm, e->d_qg, e->d_qb, p.qn)) || (st = table(k_norm, e->d_kg, e->d_kb, p.kn))) return st;
    *out = e.release();
    return MNNB200_OK;
}

// CPURoPE::onResize (CPURoPE.cpp:106-142, validRopeC4Input :71-84): q_width / k_width are the inputs' channel counts, which must be
// heads * head_dim and kv_heads * head_dim.  A refused resize keeps the previous plan.
mnnb200_status mnnb200_rope_f32_resize(mnnb200_exec* ex, int seq, int q_width, int k_width) {
    auto* e = exec_as<RoPEF32Exec>(ex);
    if (!e) return fail(MNNB200_INVALID_VALUE, "rope_f32_resize: not a RoPE execution");
    RopeParams& p = e->p;
    if (seq <= 0) return fail(MNNB200_NOT_SUPPORT, "rope_f32_resize: zero tokens");
    if ((long long)q_width != (long long)p.heads * p.head_dim || (long long)k_width != (long long)p.kv_heads * p.head_dim)
        return fail(MNNB200_NOT_SUPPORT, "rope_f32_resize: q / k width is not heads * head_dim / kv_heads * head_dim");
    if ((long long)seq * q_width > 0x7fffffffLL || (long long)seq * k_width > 0x7fffffffLL || (long long)seq * p.rope_dim > 0x7fffffffLL)
        return fail(MNNB200_NOT_SUPPORT, "rope_f32_resize: tensor too large for 32-bit indexing");
    p.seq = seq;
    e->cost_bytes = 4.0 * seq * (2.0 * (q_width + k_width) + 2.0 * p.rope_dim);
    e->cost_macs = 0;
    e->resized = true;
    return MNNB200_OK;
}

// CPURoPE::onExecute (CPURoPE.cpp:159-265): q [seq][heads * head_dim] and k [seq][kv_heads * head_dim] (the NC4HW4 [seq, C, 1, 1]
// inputs as the device stores them), cos / sin [seq][ropeDim] -> q_out [seq][heads][head_dim], k_out [seq][kv_heads][head_dim]
mnnb200_status mnnb200_rope_f32_execute(mnnb200_exec* ex, const float* q, const float* k, const float* cos, const float* sin,
                                        float* q_out, float* k_out) {
    auto* e = exec_as<RoPEF32Exec>(ex);
    if (!e) return fail(MNNB200_INVALID_VALUE, "rope_f32_execute: not a RoPE execution");
    if (!e->resized) return fail(MNNB200_NO_EXECUTION, "rope_f32_execute before resize");
    if (!q || !k || !cos || !sin || !q_out || !k_out) return fail(MNNB200_INVALID_VALUE, "rope_f32_execute: NULL tensor");
    RopeParams p = e->p;
    p.q = q; p.k = k; p.cos = cos; p.sin = sin; p.qo = q_out; p.ko = k_out;
    CK(launch_rope_f32(p, e->rt->stream));
    return MNNB200_OK;
}
}  // extern "C"
