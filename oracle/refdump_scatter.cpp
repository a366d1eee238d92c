// refdump_scatter -- the reference's ScatterNd and ScatterElements, for the tests of the scatter kernels and their plugin
// execution.
//
//   refdump_scatter op <request> <out>   one op (built as an OpT) through the Express executor on MNN_FORWARD_CPU
//                                        (REFDUMP_PLUGIN: on the plugin), once per input set given, on one executor.
//       request: int32 kind (0 ScatterNd, 1 ScatterElements), reduction (a BinaryOpOperation code, or -1 none), torch_style
//                (1: a BinaryOp parameter whose opType is left at its default), axis_mode (0 none, 1 a constant int32 fourth
//                input: ScatterElements' axis), axis, out_rank, out_dims[out_rank] (ScatterNd's shape, a constant input), nin,
//                then per input: dtype (0 fp32, 1 int32), rank, dims[rank]; int32 count, then count sets of the nin inputs'
//                raw data.  Inputs: ScatterNd indices, updates[, data]; ScatterElements data, indices, updates.
//       out:     int32 dtype, rank, dims[rank] of the output, then count raw outputs.
//   refdump_scatter run <model.mnn> <batch> <seed> <outdir>   every command's fp32 outputs (index.txt), with every input of the
//                                        model filled by fillInputs; REFDUMP_RUN_REPEATS: that many plain runSessions first (on
//                                        the plugin: eager, then a captured graph replayed), the last output in output_plain.f32.
//   refdump_scatter bench <model.mnn> <batch> <threads> <warmup> <iters>   copy in + runSession + copy out, ms per iteration.
//   refdump_scatter pillars <out.mnn> <seed>   a PointPillars-style BEV net with seeded weights (cmdPillars).
//   refdump_scatter gnn <out.mnn> <seed>       a two-layer GraphSAGE-mean-style net with seeded weights (cmdGnn).
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
    if (!g_plugin) { fprintf(stderr, "refdump_scatter: dlopen(%s): %s\n", p, dlerror()); exit(3); }
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
    const int kind = q[0], reduction = q[1], torchStyle = q[2], axisMode = q[3], axis = q[4], orank = q[5];
    q += 6;
    std::vector<int> oshape(q, q + orank);
    q += orank;
    const int nin = *q++;
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
    std::vector<VARP> in;
    std::unique_ptr<OpT> op(new OpT);
    if (kind == 0) {
        op->type = OpType_ScatterNd;
        in = {xs[0], xs[1], _Const(oshape.data(), {(int)oshape.size()}, NCHW, halide_type_of<int>())};
        if (nin > 2) in.push_back(xs[2]);
    } else {
        op->type = OpType_ScatterElements;
        in = xs;
        if (axisMode == 1) in.push_back(_Scalar<int>(axis));
    }
    if (torchStyle || reduction >= 0 || kind == 1) {
        op->main.type = OpParameter_BinaryOp;
        op->main.value = new BinaryOpT;
        if (!torchStyle) op->main.AsBinaryOp()->opType = (BinaryOpOperation)reduction;
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
        if (!info || !py) { fprintf(stderr, "refdump_scatter: compute failed\n"); return 2; }
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

// ---- the fixtures' geometry, shared by their writers and fillInputs
static const int kH = 64, kW = 48, kPillars = 2048, kPillarIn = 16, kPillarC = 32;   // BEV canvas, pillars, features
static const int kV = 512, kE = 4096, kF = 32;                                         // graph nodes, edges, features

// Every input of a session, batch dim set and filled from `seed`: fp32 inputs uniform in [-1, 1]; int32 `cells` [1, P, 1]: the
// first 3/4 of the pillars on distinct random cells of the kH x kW canvas, the rest padding pillars on cell 0 (as exporters pad
// to a fixed pillar count); int32 `src` [1, E]: uniform nodes; int32 `dst` [1, E]: skewed, a quarter of the edges into four
// hub nodes (hundreds of updates each), the rest uniform.
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
            if (kv.first == "cells") {
                std::vector<int> cells(kH * kW);
                for (int i = 0; i < kH * kW; ++i) cells[i] = i;
                const int real = n * 3 / 4;
                for (int i = 0; i < n; ++i) {
                    if (i < real) {
                        std::swap(cells[i], cells[i + rng() % (kH * kW - i)]);
                        p[i] = cells[i];
                    } else {
                        p[i] = 0;
                    }
                }
            } else if (kv.first == "dst") {
                for (int i = 0; i < n; ++i) p[i] = rng() % 4 == 0 ? (int)(rng() % 4) * 97 : (int)(rng() % kV);
            } else {
                for (int i = 0; i < n; ++i) p[i] = (int)(rng() % kV);
            }
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
    if (!s) { fprintf(stderr, "refdump_scatter run: createSession failed\n"); return 2; }
    sessionInputs(net.get(), s, batch);
    fillInputs(net.get(), s, seed);
    if (const char* rp = getenv("REFDUMP_RUN_REPEATS")) {
        const int reps = atoi(rp);
        auto output = net->getSessionOutput(s, nullptr);
        Tensor host(output, Tensor::CAFFE);
        for (int i = 0; i < reps; ++i) {
            fillInputs(net.get(), s, seed);
            if (net->runSession(s) != NO_ERROR) { fprintf(stderr, "refdump_scatter run: plain runSession failed\n"); return 2; }
            output->copyToHostTensor(&host);
        }
        if (reps > 0) writeFile(dir + "/output_plain.f32", host.host<float>(), host.size());
        fillInputs(net.get(), s, seed);
    }
    FILE* idx = fopen((dir + "/index.txt").c_str(), "w");
    if (!idx) { fprintf(stderr, "refdump_scatter run: cannot write %s/index.txt\n", dir.c_str()); return 2; }
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
    if (code != NO_ERROR) { fprintf(stderr, "refdump_scatter run: runSession -> %d\n", (int)code); return 2; }
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
    if (!s) { fprintf(stderr, "refdump_scatter bench: createSession failed\n"); return 2; }
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

static std::vector<float> uniform(std::mt19937& rng, size_t n, float scale) {
    std::uniform_real_distribution<float> u(-1.f, 1.f);
    std::vector<float> v(n);
    for (auto& f : v) f = u(rng) * scale;
    return v;
}
static VARP seeded(std::mt19937& rng, std::vector<int> shape, float scale) {
    size_t n = 1;
    for (int d : shape) n *= (size_t)d;
    auto v = uniform(rng, n, scale);
    return _Const(v.data(), shape, NCHW, halide_type_of<float>());
}
static VARP conv(std::mt19937& rng, VARP x, int ic, int oc, int k, int stride, bool relu) {
    return _Conv(uniform(rng, (size_t)oc * ic * k * k, std::sqrt(3.f / (ic * k * k))), uniform(rng, oc, 0.05f), x, {ic, oc}, {k, k},
                 SAME, {stride, stride}, {1, 1}, 1, {0, 0}, relu, false);
}
static void save(VARP h, const char* out) {
    h->setName("output");
    Variable::save({h}, out);
}

// PointPillars-style, batch 1: `pillars` [1, P, 16] through a pillar-feature MatMul + ReLU to [P, 32]; ScatterNd of the
// pillar vectors by the int32 `cells` [1, P, 1] into a zero canvas [H * W, 32] (padding pillars write cell 0); a Raster to NCHW
// [1, 32, H, W]; a backbone of a stride-2 and a stride-1 3x3 conv (ReLU), a 2x2 stride-2 deconv upsample back to H x W, and
// 1x1 heads of 2 class and 7 box channels.
static int cmdPillars(const char* out, int seed) {
    std::mt19937 rng(seed);
    VARP pil = _Input({1, kPillars, kPillarIn}, NCHW, halide_type_of<float>());
    pil->setName("pillars");
    VARP cells = _Input({1, kPillars, 1}, NCHW, halide_type_of<int>());
    cells->setName("cells");
    VARP f = _MatMul(_Reshape(pil, {kPillars, kPillarIn}), seeded(rng, {kPillarIn, kPillarC}, std::sqrt(3.f / kPillarIn)));
    f = _Relu(_Add(f, seeded(rng, {kPillarC}, 0.05f)));
    const int shape[2] = {kH * kW, kPillarC};
    VARP canvas = _ScatterNd(_Reshape(cells, {kPillars, 1}), f, _Const(shape, {2}, NCHW, halide_type_of<int>()));
    VARP img = _Convert(_Transpose(_Reshape(canvas, {1, kH, kW, kPillarC}), {0, 3, 1, 2}), NC4HW4);
    VARP x = conv(rng, img, kPillarC, 64, 3, 2, true);
    x = conv(rng, x, 64, 64, 3, 1, true);
    x = _Deconv(uniform(rng, 64 * 32 * 4, std::sqrt(3.f / 64)), uniform(rng, 32, 0.05f), x, {64, 32}, {2, 2}, VALID, {2, 2}, {1, 1},
                1, {0, 0}, true, false);
    save(_Convert(conv(rng, x, 32, 9, 1, 1, false), NCHW), out);
    return 0;
}

// GraphSAGE-mean-style, batch 1: node features `x` [1, V, 32], int32 edges `src`, `dst` [1, E].  Each of two layers gathers the
// source nodes' features (GatherV2), adds them into their destination nodes (ScatterElements ADD on axis 0, the destination
// index broadcast over the features), divides by the in-degree (a ScatterElements ADD of ones, MAXIMUM with 1, REALDIV) and
// applies ReLU(mean W_n + h W_s + b).
static int cmdGnn(const char* out, int seed) {
    std::mt19937 rng(seed);
    VARP x = _Input({1, kV, kF}, NCHW, halide_type_of<float>());
    x->setName("x");
    VARP src = _Input({1, kE}, NCHW, halide_type_of<int>());
    src->setName("src");
    VARP dst = _Input({1, kE}, NCHW, halide_type_of<int>());
    dst->setName("dst");
    const int ef[2] = {kE, kF};
    VARP s = _Reshape(src, {kE});
    VARP d = _Reshape(dst, {kE, 1});
    VARP didx = _BroadcastTo(d, _Const(ef, {2}, NCHW, halide_type_of<int>()));
    std::vector<float> zf((size_t)kV * kF, 0.f), z1(kV, 0.f), ones(kE, 1.f);
    VARP deg = _ScatterElements(_Const(z1.data(), {kV, 1}, NCHW, halide_type_of<float>()), d,
                                _Const(ones.data(), {kE, 1}, NCHW, halide_type_of<float>()), _Scalar<int>(0), BinaryOpOperation_ADD);
    VARP inv = _Maximum(deg, _Scalar<float>(1.f));
    VARP h = _Reshape(x, {kV, kF});
    for (int l = 0; l < 2; ++l) {
        VARP msg = _GatherV2(h, s, _Scalar<int>(0));
        VARP agg = _ScatterElements(_Const(zf.data(), {kV, kF}, NCHW, halide_type_of<float>()), didx, msg, _Scalar<int>(0),
                                    BinaryOpOperation_ADD);
        VARP mean = _Divide(agg, inv);
        const float sc = std::sqrt(3.f / kF);
        h = _Relu(_Add(_Add(_MatMul(mean, seeded(rng, {kF, kF}, sc)), _MatMul(h, seeded(rng, {kF, kF}, sc))), seeded(rng, {kF}, 0.05f)));
    }
    save(_Reshape(h, {1, kV, kF}), out);
    return 0;
}

int main(int argc, char** argv) {
    const std::string cmd = argc > 1 ? argv[1] : "";
    if (cmd == "op" && argc >= 4) return cmdOp(argv[2], argv[3]);
    if (cmd == "run" && argc >= 6) return cmdRun(argv[2], atoi(argv[3]), atoi(argv[4]), argv[5]);
    if (cmd == "bench" && argc >= 7) return cmdBench(argv[2], atoi(argv[3]), atoi(argv[4]), atoi(argv[5]), atoi(argv[6]));
    if (cmd == "pillars" && argc >= 4) return cmdPillars(argv[2], atoi(argv[3]));
    if (cmd == "gnn" && argc >= 4) return cmdGnn(argv[2], atoi(argv[3]));
    fprintf(stderr, "usage: refdump_scatter op <request> <out> | run <model> <batch> <seed> <outdir> | "
                    "bench <model> <batch> <threads> <warmup> <iters> | pillars <out.mnn> <seed> | gnn <out.mnn> <seed>\n");
    return 1;
}
