// refdump_gather -- the reference's Gather family, Cast and (Batch)MatMul, for the tests of the gather kernels, the broadcast
// float MatMul and their plugin executions; and two transformer fixtures that use them.
//
//   refdump_gather op <request> <out>   one op (built as an OpT) through the Express executor on MNN_FORWARD_CPU
//                                       (REFDUMP_PLUGIN: on the plugin), once per input set given, on one executor.
//       request: int32 kind (0 Gather, 1 GatherV2, 2 GatherND, 3 GatherElements, 4 Cast, 5 MatMul, 6 BatchMatMul), axis_mode
//                (0 none, 1 the op's Axis, 2 a constant int32 third input), axis, ta, tb, dst (Cast: 0 fp32, 1 int32),
//                nin, then per input: dtype (0 fp32, 1 int32), rank, dims[rank]; int32 count, then count sets of the nin
//                inputs' raw data.
//       out:     int32 dtype, rank, dims[rank] of the output, then count raw outputs.
//   refdump_gather run <model.mnn> <batch> <seed> <outdir>   every command's fp32 outputs, as refdump's run writes them
//                                       (index.txt), with every input of the model filled by fillInputs; REFDUMP_RUN_REPEATS
//                                       as refdump's run.
//   refdump_gather bench <model.mnn> <batch> <threads> <warmup> <iters>   as refdump's bench, for models of several inputs.
//   refdump_gather bert <out.mnn> <seed>   a BERT-style encoder with seeded weights (cmdBert).
//   refdump_gather vit <out.mnn> <seed>    a ViT-style encoder with seeded weights (cmdVit).
#include <MNN/Interpreter.hpp>
#include <MNN/expr/Expr.hpp>
#include <MNN/expr/ExprCreator.hpp>
#include <MNN/expr/Executor.hpp>
#include <MNN/expr/ExecutorScope.hpp>
#include <dlfcn.h>
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <random>
#include <string>
#include <vector>
#include "MNN_generated.h"
#include "core/TensorUtils.hpp"

using namespace MNN;
using namespace MNN::Express;

static std::vector<char> readFile(const char* p) {
    std::ifstream f(p, std::ios::binary);
    return std::vector<char>((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
}
static void writeFile(const std::string& p, const void* d, size_t n) {
    std::ofstream f(p, std::ios::binary);
    f.write((const char*)d, n);
}

static void* g_plugin = nullptr;
static MNNForwardType forwardType() {
    const char* p = getenv("REFDUMP_PLUGIN");
    if (!p || !*p) return MNN_FORWARD_CPU;
    g_plugin = dlopen(p, RTLD_NOW | RTLD_GLOBAL);
    if (!g_plugin) { fprintf(stderr, "refdump_gather: dlopen(%s): %s\n", p, dlerror()); exit(3); }
    return MNN_FORWARD_CUDA;
}
static void pluginCounts(int* c, int* d) {
    *c = *d = -1;
    if (!g_plugin) return;
    typedef void (*Fn)(int*, int*);
    Fn fn = (Fn)dlsym(g_plugin, "mnnb200_plugin_stats");
    if (fn) fn(c, d);
}
static void pluginStats() {
    if (!g_plugin) return;
    int c, d;
    pluginCounts(&c, &d);
    printf("{\"plugin_created\": %d, \"plugin_declined\": %d}\n", c, d);
}

static halide_type_t dtypeOf(int t) { return t == 1 ? halide_type_of<int>() : halide_type_of<float>(); }

static int cmdOp(const char* reqPath, const char* outPath) {
    auto buf = readFile(reqPath);
    const int32_t* q = (const int32_t*)buf.data();
    const int kind = q[0], axisMode = q[1], axis = q[2], ta = q[3], tb = q[4], dst = q[5], nin = q[6];
    q += 7;
    std::vector<int> types(nin);
    std::vector<std::vector<int>> dims(nin);
    std::vector<size_t> counts(nin);
    for (int i = 0; i < nin; ++i) {
        types[i] = *q++;
        const int r = *q++;
        dims[i].assign(q, q + r);
        q += r;
        size_t n = 1;
        for (int d : dims[i]) n *= (size_t)d;
        counts[i] = n;
    }
    const int count = *q++;
    const char* data = (const char*)q;
    BackendConfig bc;
    bc.precision = BackendConfig::Precision_High;
    ExecutorScope scope(Executor::newExecutor(forwardType(), bc, 1));
    std::vector<VARP> xs;
    for (int i = 0; i < nin; ++i) xs.push_back(_Input(dims[i], NCHW, dtypeOf(types[i])));
    std::vector<VARP> in = xs;
    std::unique_ptr<OpT> op(new OpT);
    if (kind <= 3) {
        op->type = kind == 0 ? OpType_Gather : (kind == 1 ? OpType_GatherV2 : (kind == 2 ? OpType_GatherND : OpType_GatherElements));
        if (axisMode == 1) {
            op->main.type = OpParameter_Axis;
            op->main.value = new AxisT;
            op->main.AsAxis()->axis = axis;
        } else if (axisMode == 2) {
            in.push_back(_Scalar<int>(axis));
        }
    } else if (kind == 4) {
        op->type = OpType_Cast;
        op->main.type = OpParameter_CastParam;
        op->main.value = new CastParamT;
        op->main.AsCastParam()->srcT = types[0] == 1 ? DataType_DT_INT32 : DataType_DT_FLOAT;
        op->main.AsCastParam()->dstT = dst == 1 ? DataType_DT_INT32 : DataType_DT_FLOAT;
    } else if (kind == 5) {
        op->type = OpType_MatMul;
        op->main.type = OpParameter_MatMul;
        op->main.value = new MatMulT;
        op->main.AsMatMul()->transposeA = ta != 0;
        op->main.AsMatMul()->transposeB = tb != 0;
    } else {
        op->type = OpType_BatchMatMul;
        op->main.type = OpParameter_BatchMatMulParam;
        op->main.value = new BatchMatMulParamT;
        op->main.AsBatchMatMulParam()->adjX = ta != 0;
        op->main.AsBatchMatMulParam()->adjY = tb != 0;
    }
    VARP y = Variable::create(Expr::create(op.get(), in));
    std::ofstream o(outPath, std::ios::binary);
    for (int c = 0; c < count; ++c) {
        for (int i = 0; i < nin; ++i) {
            const size_t bytes = counts[i] * 4;
            memcpy(xs[i]->writeMap<char>(), data, bytes);
            data += bytes;
        }
        auto info = y->getInfo();
        const char* py = y->readMap<char>();
        if (!info || !py) { fprintf(stderr, "refdump_gather: compute failed\n"); return 2; }
        if (c == 0) {
            const int32_t hdr[2] = {info->type.code == halide_type_int ? 1 : 0, (int32_t)info->dim.size()};
            o.write((const char*)hdr, sizeof(hdr));
            o.write((const char*)info->dim.data(), info->dim.size() * 4);
        }
        o.write(py, (size_t)info->size * 4);
    }
    pluginStats();
    return 0;
}

// Every input of a session, batch dim set and filled from `seed`: fp32 inputs uniform in [-1, 1]; int32 inputs named *mask*
// [batch][seq] ones for the first seq - 8 * (b % 4) tokens of row b and zeros after; other int32 inputs token ids in
// [0, kIdRange)
static const int kIdRange = 2048;
static std::vector<Tensor*> sessionInputs(Interpreter* net, Session* s, int batch) {
    std::vector<Tensor*> ins;
    for (auto& kv : net->getSessionInputAll(s)) {
        auto shape = kv.second->shape();
        shape[0] = batch;
        net->resizeTensor(kv.second, shape);
        ins.push_back(kv.second);
    }
    net->resizeSession(s);
    return ins;
}
static void fillInputs(Interpreter* net, Session* s, int seed) {
    std::mt19937 rng(seed);
    for (auto& kv : net->getSessionInputAll(s)) {
        Tensor host(kv.second, Tensor::CAFFE);
        const int n = host.elementSize();
        if (host.getType().code == halide_type_int) {
            auto p = host.host<int>();
            const bool mask = kv.first.find("mask") != std::string::npos;
            const int seq = host.dimensions() > 1 ? host.length(1) : n;
            for (int i = 0; i < n; ++i) p[i] = mask ? ((i % seq) < seq - 8 * ((i / seq) % 4) ? 1 : 0) : (int)(rng() % kIdRange);
        } else {
            std::uniform_real_distribution<float> u(-1.f, 1.f);
            auto p = host.host<float>();
            for (int i = 0; i < n; ++i) p[i] = u(rng);
        }
        kv.second->copyFromHostTensor(&host);
    }
}
static Session* makeSession(Interpreter* net, int threads) {
    ScheduleConfig c; c.type = forwardType(); c.numThread = threads; c.backupType = MNN_FORWARD_CPU;
    BackendConfig bc; bc.precision = BackendConfig::Precision_High; c.backendConfig = &bc;
    return net->createSession(c);
}

static int cmdRun(const char* model, int batch, int seed, const std::string& dir) {
    std::shared_ptr<Interpreter> net(Interpreter::createFromFile(model), Interpreter::destroy);
    auto s = makeSession(net.get(), 4);
    if (!s) { fprintf(stderr, "refdump_gather run: createSession failed\n"); return 2; }
    sessionInputs(net.get(), s, batch);
    fillInputs(net.get(), s, seed);
    if (const char* rp = getenv("REFDUMP_RUN_REPEATS")) {
        const int reps = atoi(rp);
        auto output = net->getSessionOutput(s, nullptr);
        Tensor host(output, Tensor::CAFFE);
        for (int i = 0; i < reps; ++i) {
            fillInputs(net.get(), s, seed);
            if (net->runSession(s) != NO_ERROR) { fprintf(stderr, "refdump_gather run: plain runSession failed\n"); return 2; }
            output->copyToHostTensor(&host);
        }
        if (reps > 0) writeFile(dir + "/output_plain.f32", host.host<float>(), host.size());
        fillInputs(net.get(), s, seed);
    }
    FILE* idx = fopen((dir + "/index.txt").c_str(), "w");
    int n = 0;
    TensorCallBackWithInfo before = [&](const std::vector<Tensor*>&, const OperatorInfo*) { return true; };
    TensorCallBackWithInfo after = [&](const std::vector<Tensor*>& ts, const OperatorInfo* info) {
        for (size_t i = 0; i < ts.size(); ++i) {
            auto t = ts[i];
            if (t->elementSize() <= 0 || t->getType().code != halide_type_float) continue;
            Tensor host(t, Tensor::CAFFE);
            t->copyToHostTensor(&host);
            char name[64];
            snprintf(name, sizeof(name), "%04d_%zu.f32", n, i);
            writeFile(dir + "/" + name, host.host<float>(), host.size());
            fprintf(idx, "%s|%s|%s|", name, info->name().c_str(), info->type().c_str());
            for (int d = 0; d < host.dimensions(); ++d) fprintf(idx, "%d%s", host.length(d), d + 1 < host.dimensions() ? "," : "");
            fprintf(idx, "|0|0|0|0|0\n");
        }
        ++n;
        return true;
    };
    auto code = net->runSessionWithCallBackInfo(s, before, after, true);
    fclose(idx);
    if (code != NO_ERROR) { fprintf(stderr, "refdump_gather run: runSession -> %d\n", (int)code); return 2; }
    auto output = net->getSessionOutput(s, nullptr);
    Tensor host(output, Tensor::CAFFE);
    output->copyToHostTensor(&host);
    writeFile(dir + "/output.f32", host.host<float>(), host.size());
    pluginStats();
    return 0;
}

static int cmdBench(const char* model, int batch, int threads, int warmup, int iters) {
    std::shared_ptr<Interpreter> net(Interpreter::createFromFile(model), Interpreter::destroy);
    auto s = makeSession(net.get(), threads);
    if (!s) { fprintf(stderr, "refdump_gather bench: createSession failed\n"); return 2; }
    auto ins = sessionInputs(net.get(), s, batch);
    fillInputs(net.get(), s, 1000);
    std::vector<std::shared_ptr<Tensor>> hosts;
    size_t inBytes = 0;
    for (auto t : ins) {
        hosts.emplace_back(new Tensor(t, Tensor::CAFFE));
        t->copyToHostTensor(hosts.back().get());
        inBytes += hosts.back()->size();
    }
    auto output = net->getSessionOutput(s, nullptr);
    Tensor hostOut(output, Tensor::CAFFE);
    auto step = [&]() {
        for (size_t i = 0; i < ins.size(); ++i) ins[i]->copyFromHostTensor(hosts[i].get());
        net->runSession(s);
        output->copyToHostTensor(&hostOut);
    };
    for (int i = 0; i < warmup; ++i) step();
    int windows = 1;
    if (const char* w = getenv("REFDUMP_BENCH_WINDOWS")) windows = std::max(1, atoi(w));
    std::vector<double> win;
    double total = 0;
    for (int wdx = 0; wdx < windows; ++wdx) {
        auto t0 = std::chrono::steady_clock::now();
        for (int i = 0; i < iters; ++i) step();
        auto t1 = std::chrono::steady_clock::now();
        const double ms = std::chrono::duration<double, std::milli>(t1 - t0).count() / iters;
        win.push_back(ms);
        total += ms;
    }
    std::vector<double> sorted = win;
    std::sort(sorted.begin(), sorted.end());
    int created, declined;
    pluginCounts(&created, &declined);
    printf("{\"ms_per_iter\": %.6f, \"ms_median_window\": %.6f, \"ms_min_window\": %.6f, \"windows\": %d, \"batch\": %d, \"threads\": %d, "
           "\"iters\": %d, \"plugin_created\": %d, \"plugin_declined\": %d, \"h2d_bytes\": %zu, \"d2h_bytes\": %zu}\n",
           total / windows, sorted[sorted.size() / 2], sorted[0], windows, batch, threads, iters, created, declined, inBytes,
           (size_t)hostOut.size());
    return 0;
}

// ---- the fixtures
static VARP seeded(std::mt19937& rng, std::vector<int> shape, float scale) {
    std::uniform_real_distribution<float> u(-1.f, 1.f);
    size_t n = 1;
    for (int d : shape) n *= (size_t)d;
    std::vector<float> v(n);
    for (auto& f : v) f = u(rng) * scale;
    return _Const(v.data(), shape, NCHW, halide_type_of<float>());
}
// x [..., d] @ w [d, o] + b: a MatMul whose batch dims broadcast against a 2-D weight
static VARP linear(std::mt19937& rng, VARP x, int d, int o) {
    return _Add(_MatMul(x, seeded(rng, {d, o}, std::sqrt(3.f / d))), seeded(rng, {o}, 0.02f));
}
// LayerNorm over the last axis from Reductions and BinaryOps, eps 1e-5
static VARP layerNorm(std::mt19937& rng, VARP x, int d) {
    VARP c = _Subtract(x, _ReduceMean(x, {-1}, true));
    VARP r = _Rsqrt(_Add(_ReduceMean(_Multiply(c, c), {-1}, true), _Scalar<float>(1e-5f)));
    return _Add(_Multiply(_Multiply(c, r), _Add(seeded(rng, {d}, 0.1f), _Scalar<float>(1.f))), seeded(rng, {d}, 0.1f));
}
// one post-LN encoder layer on x [B, S, D]: H heads, QK^T as a BatchMatMul with adjY, PV as a BatchMatMul; `bias` [B, 1, 1, S]
// (or nullptr) is added to the scores
static VARP encoder(std::mt19937& rng, VARP x, int S, int D, int H, VARP bias) {
    const int dh = D / H;
    auto heads = [&](VARP t) { return _Transpose(_Reshape(t, {-1, S, H, dh}), {0, 2, 1, 3}); };   // [B, H, S, dh]
    VARP q = heads(linear(rng, x, D, D)), k = heads(linear(rng, x, D, D)), v = heads(linear(rng, x, D, D));
    VARP s = _Multiply(_BatchMatMul(q, k, false, true), _Scalar<float>(1.f / std::sqrt((float)dh)));
    if (bias.get()) s = _Add(s, bias);
    VARP ctx = _Reshape(_Transpose(_BatchMatMul(_Softmax(s, -1), v), {0, 2, 1, 3}), {-1, S, D});
    x = layerNorm(rng, _Add(x, linear(rng, ctx, D, D)), D);
    VARP f = linear(rng, _Gelu(linear(rng, x, D, 4 * D)), 4 * D, D);
    return layerNorm(rng, _Add(x, f), D);
}
static void save(VARP h, const char* out) {
    h->setName("output");
    Variable::save({h}, out);
}

// BERT-style: int32 input_ids and attention_mask [1, 64]; word (vocab 2048) and position embeddings by GatherV2, LayerNorm,
// 4 layers of D 256, 4 heads, FFN 1024, the mask Cast to fp32 into an additive -10000 score bias; a GatherV2 pooler on token 0
// (a scalar index), a dense layer and tanh.
static int cmdBert(const char* out, int seed) {
    std::mt19937 rng(seed);
    const int S = 64, D = 256, H = 4, V = kIdRange;
    VARP ids = _Input({1, S}, NCHW, halide_type_of<int>());
    ids->setName("input_ids");
    VARP mask = _Input({1, S}, NCHW, halide_type_of<int>());
    mask->setName("attention_mask");
    std::vector<int> pos(S);
    for (int i = 0; i < S; ++i) pos[i] = i;
    VARP x = _GatherV2(seeded(rng, {V, D}, 1.f), ids, _Scalar<int>(0));
    x = _Add(x, _GatherV2(seeded(rng, {S, D}, 0.5f), _Const(pos.data(), {S}, NCHW, halide_type_of<int>()), _Scalar<int>(0)));
    x = layerNorm(rng, x, D);
    VARP keep = _Cast<float>(mask);
    VARP bias = _Reshape(_Multiply(_Subtract(_Scalar<float>(1.f), keep), _Scalar<float>(-10000.f)), {-1, 1, 1, S});
    for (int l = 0; l < 4; ++l) x = encoder(rng, x, S, D, H, bias);
    VARP cls = _GatherV2(x, _Scalar<int>(0), _Scalar<int>(1));   // [B, D]
    save(_Tanh(linear(rng, cls, D, D)), out);
    return 0;
}

// ViT-style on a 3 x 64 x 64 image: a 8 x 8 stride-8 patch conv to D 192 (64 patches), a class token (a learned row, made
// [B, 1, D] by adding it to a zeroed mean of the patches), position embeddings, 4 layers of 3 heads, a final LayerNorm, a Gather
// (the op with an Axis parameter) of the class token and a 10-way head.
static int cmdVit(const char* out, int seed) {
    std::mt19937 rng(seed);
    const int D = 192, H = 3, P = 64, S = P + 1;
    VARP img = _Input({1, 3, 64, 64}, NCHW, halide_type_of<float>());
    img->setName("input");
    std::vector<float> w(D * 3 * 8 * 8), b(D);
    std::uniform_real_distribution<float> u(-1.f, 1.f);
    for (auto& f : w) f = u(rng) * std::sqrt(3.f / (3 * 64));
    for (auto& f : b) f = u(rng) * 0.02f;
    VARP p = _Conv(std::move(w), std::move(b), img, {3, D}, {8, 8}, VALID, {8, 8}, {1, 1}, 1, {0, 0}, false, false);
    p = _Transpose(_Reshape(_Convert(p, NCHW), {-1, D, P}), {0, 2, 1});                     // [B, 64, D]
    VARP cls = _Add(_Multiply(_ReduceMean(p, {1}, true), _Scalar<float>(0.f)), seeded(rng, {1, 1, D}, 0.5f));
    VARP x = _Add(_Concat({cls, p}, 1), seeded(rng, {1, S, D}, 0.5f));
    for (int l = 0; l < 4; ++l) x = encoder(rng, x, S, D, H, nullptr);
    x = layerNorm(rng, x, D);
    std::unique_ptr<OpT> g(new OpT);
    g->type = OpType_Gather;
    g->main.type = OpParameter_Axis;
    g->main.value = new AxisT;
    g->main.AsAxis()->axis = 1;
    VARP tok = Variable::create(Expr::create(g.get(), {x, _Scalar<int>(0)}));                // [B, D]
    save(linear(rng, tok, D, 10), out);
    return 0;
}

int main(int argc, char** argv) {
    const std::string cmd = argc > 1 ? argv[1] : "";
    if (cmd == "op" && argc >= 4) return cmdOp(argv[2], argv[3]);
    if (cmd == "run" && argc >= 6) return cmdRun(argv[2], atoi(argv[3]), atoi(argv[4]), argv[5]);
    if (cmd == "bench" && argc >= 7) return cmdBench(argv[2], atoi(argv[3]), atoi(argv[4]), atoi(argv[5]), atoi(argv[6]));
    if (cmd == "bert" && argc >= 4) return cmdBert(argv[2], atoi(argv[3]));
    if (cmd == "vit" && argc >= 4) return cmdVit(argv[2], atoi(argv[3]));
    fprintf(stderr, "usage: refdump_gather op <request> <out> | run <model> <batch> <seed> <outdir> | "
                    "bench <model> <batch> <threads> <warmup> <iters> | bert <out.mnn> <seed> | vit <out.mnn> <seed>\n");
    return 1;
}
