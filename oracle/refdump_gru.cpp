// refdump_gru -- the reference's GRU (OpType_RNNSequenceGRU), for the tests of the GRU kernel and its plugin execution.
//
//   refdump_gru op <request> <out>     one op (built as an OpT, as the ONNX converter builds it) through the Express executor on
//                                      MNN_FORWARD_CPU (REFDUMP_PLUGIN: on the plugin), once per input set given, on one executor.
//       request: int32 lbr, T, B, I, H, D, has_h0, keep_all (keepAllOutputs), n_out (1 or 2), count; then count sets of the
//                op's fp32 inputs' raw data: X [T, B, I], per direction Wg [I + H, 2H], bg [1, 2H], Wc [I + H, H], bc [1, H],
//                rb [1, 3H], then h0 [D, B, H] when has_h0.
//       out:     per set, the op's outputs' raw fp32 data in order (keep_all: Y [T, D, B, H][, Y_h [D, B, H]]; else Y_h).
//   refdump_gru run <model.mnn> <batch> <seed> <outdir>   every command's fp32 outputs (index.txt), with every input filled by
//                                      fillInputs; REFDUMP_RUN_REPEATS: that many plain runSessions first, the last first output
//                                      in output_plain.f32.
//   refdump_gru chunks <model.mnn> <batch> <seed> <n> <outdir>   denoise_f32.mnn over n chained chunks: each chunk's outputs
//                                      (chunk<k>_<name>.f32), the final states fed back as the next chunk's initial states.
//   refdump_gru bench <model.mnn> <batch> <threads> <warmup> <iters>   copy in + runSession + copy out, ms per iteration.
//   refdump_gru denoise <out.mnn> <seed>   an RNNoise-style streaming denoiser chunk with seeded weights (cmdDenoise).
//   refdump_gru tagger <out.mnn> <seed>    a BiGRU sequence tagger with seeded weights (cmdTagger).
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
#include <map>
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
    if (!g_plugin) g_plugin = dlopen(p, RTLD_NOW | RTLD_GLOBAL);
    if (!g_plugin) { fprintf(stderr, "refdump_gru: dlopen(%s): %s\n", p, dlerror()); exit(3); }
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

// the GRU op as the ONNX converter writes it (OnnxSequenceGRUMerge.cpp): the RNNParam with the weights as inputs
static std::vector<VARP> gruOp(int lbr, int H, int D, bool keepAll, int nout, const std::vector<VARP>& in) {
    std::unique_ptr<OpT> op(new OpT);
    op->type = OpType_RNNSequenceGRU;
    op->main.type = OpParameter_RNNParam;
    op->main.value = new RNNParamT;
    auto p = op->main.AsRNNParam();
    p->numUnits = H;
    p->isBidirectionalRNN = D == 2;
    p->linearBeforeReset = lbr != 0;
    p->keepAllOutputs = keepAll;
    EXPRP e = Expr::create(op.get(), in, nout);
    std::vector<VARP> out;
    for (int i = 0; i < nout; ++i) out.push_back(Variable::create(e, i));
    return out;
}

static int cmdOp(const char* reqPath, const char* outPath) {
    auto buf = readFile(reqPath);
    const int32_t* q = (const int32_t*)buf.data();
    const int lbr = q[0], T = q[1], B = q[2], I = q[3], H = q[4], D = q[5], hasH0 = q[6], keepAll = q[7], nout = q[8];
    const int count = q[9];
    q += 10;
    std::vector<std::vector<int>> dims = {{T, B, I}};
    for (int d = 0; d < D; ++d) {
        dims.push_back({I + H, 2 * H});
        dims.push_back({1, 2 * H});
        dims.push_back({I + H, H});
        dims.push_back({1, H});
        dims.push_back({1, 3 * H});
    }
    if (hasH0) dims.push_back({D, B, H});
    BackendConfig bc;
    bc.precision = BackendConfig::Precision_High;
    ExecutorScope scope(Executor::newExecutor(forwardType(), bc, 1));
    std::vector<VARP> xs;
    for (auto& d : dims) xs.push_back(_Input(d, NCHW, halide_type_of<float>()));
    auto ys = gruOp(lbr, H, D, keepAll != 0, nout, xs);
    const char* data = (const char*)q;
    std::ofstream o(outPath, std::ios::binary);
    for (int c = 0; c < count; ++c) {
        for (size_t i = 0; i < dims.size(); ++i) {
            size_t n = 1;
            for (int d : dims[i]) n *= (size_t)d;
            memcpy(xs[i]->writeMap<char>(), data, n * 4);
            data += n * 4;
        }
        for (auto& y : ys) {
            auto info = y->getInfo();
            const char* py = y->readMap<char>();
            if (!info || !py) { fprintf(stderr, "refdump_gru: compute failed\n"); return 2; }
            o.write(py, (size_t)info->size * 4);
        }
    }
    pluginStats();
    return 0;
}

// ---- the fixtures' geometry, shared by their writers and fillInputs
static const int kDnT = 16, kDnF = 42, kDnD = 24, kDnH1 = 24, kDnH2 = 48, kDnH3 = 96, kDnG = 22;  // denoiser
static const int kTgT = 64, kTgV = 8000, kTgE = 128, kTgH = 256, kTgK = 17;                    // tagger

// the batch axis of a fixture input: dim 1 of every sequence and state
static std::vector<Tensor*> sessionInputs(Interpreter* net, Session* s, int batch) {
    std::vector<Tensor*> ins;
    for (auto& kv : net->getSessionInputAll(s)) {
        auto shape = kv.second->shape();
        shape[1] = batch;
        net->resizeTensor(kv.second, shape);
        ins.push_back(kv.second);
    }
    net->resizeSession(s);
    return ins;
}
// every fp32 input uniform in [-1, 1] from `seed` (states at half that); token ids uniform in [0, 8000)
static void fillInputs(Interpreter* net, Session* s, int seed) {
    std::mt19937 rng(seed);
    for (auto& kv : net->getSessionInputAll(s)) {
        Tensor host(kv.second, Tensor::CAFFE);
        if (kv.second->getType().code == halide_type_int) {
            std::uniform_int_distribution<int> u(0, kTgV - 1);
            for (int i = 0; i < host.elementSize(); ++i) host.host<int>()[i] = u(rng);
        } else {
            std::uniform_real_distribution<float> u(-1.f, 1.f);
            const float sc = kv.first == "feats" ? 1.f : 0.5f;
            for (int i = 0; i < host.elementSize(); ++i) host.host<float>()[i] = u(rng) * sc;
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
    if (!s) { fprintf(stderr, "refdump_gru run: createSession failed\n"); return 2; }
    sessionInputs(net.get(), s, batch);
    fillInputs(net.get(), s, seed);
    auto output = net->getSessionOutput(s, "output");
    if (const char* rp = getenv("REFDUMP_RUN_REPEATS")) {
        const int reps = atoi(rp);
        Tensor host(output, Tensor::CAFFE);
        for (int i = 0; i < reps; ++i) {
            fillInputs(net.get(), s, seed);
            if (net->runSession(s) != NO_ERROR) { fprintf(stderr, "refdump_gru run: plain runSession failed\n"); return 2; }
            output->copyToHostTensor(&host);
        }
        if (reps > 0) writeFile(dir + "/output_plain.f32", host.host<float>(), host.size());
        fillInputs(net.get(), s, seed);
    }
    FILE* idx = fopen((dir + "/index.txt").c_str(), "w");
    if (!idx) { fprintf(stderr, "refdump_gru run: cannot write %s/index.txt\n", dir.c_str()); return 2; }
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
            fprintf(idx, "\n");
        }
        ++n;
        return true;
    };
    auto code = net->runSessionWithCallBackInfo(s, before, after, true);
    fclose(idx);
    if (code != NO_ERROR) { fprintf(stderr, "refdump_gru run: runSession -> %d\n", (int)code); return 2; }
    Tensor host(output, Tensor::CAFFE);
    output->copyToHostTensor(&host);
    writeFile(dir + "/output.f32", host.host<float>(), host.size());
    pluginStats();
    return 0;
}

// denoise_f32.mnn over n chunks: chunk k's features from seed + 1 + k, its final states the next chunk's initial states
static int cmdChunks(const char* model, int batch, int seed, int chunks, const std::string& dir) {
    std::shared_ptr<Interpreter> net(Interpreter::createFromFile(model), Interpreter::destroy);
    auto s = makeSession(net.get(), 4);
    if (!s) { fprintf(stderr, "refdump_gru chunks: createSession failed\n"); return 2; }
    sessionInputs(net.get(), s, batch);
    fillInputs(net.get(), s, seed);
    const std::map<std::string, std::string> feed = {{"h1_n", "h1_0"}, {"h2_n", "h2_0"}, {"h3_n", "h3_0"}};
    for (int k = 0; k < chunks; ++k) {
        Tensor feats(net->getSessionInput(s, "feats"), Tensor::CAFFE);
        std::mt19937 rng(seed + 1 + k);
        std::uniform_real_distribution<float> u(-1.f, 1.f);
        for (int i = 0; i < feats.elementSize(); ++i) feats.host<float>()[i] = u(rng);
        net->getSessionInput(s, "feats")->copyFromHostTensor(&feats);
        if (net->runSession(s) != NO_ERROR) { fprintf(stderr, "refdump_gru chunks: runSession failed\n"); return 2; }
        for (const char* name : {"output", "h1_n", "h2_n", "h3_n"}) {
            auto t = net->getSessionOutput(s, name);
            Tensor host(t, Tensor::CAFFE);
            t->copyToHostTensor(&host);
            writeFile(dir + "/chunk" + std::to_string(k) + "_" + name + ".f32", host.host<float>(), host.size());
            auto it = feed.find(name);
            if (it != feed.end()) net->getSessionInput(s, it->second.c_str())->copyFromHostTensor(&host);
        }
    }
    pluginStats();
    return 0;
}

static int cmdBench(const char* model, int batch, int threads, int warmup, int iters) {
    std::shared_ptr<Interpreter> net(Interpreter::createFromFile(model), Interpreter::destroy);
    auto s = makeSession(net.get(), threads);
    if (!s) { fprintf(stderr, "refdump_gru bench: createSession failed\n"); return 2; }
    auto ins = sessionInputs(net.get(), s, batch);
    fillInputs(net.get(), s, 1000);
    std::vector<std::shared_ptr<Tensor>> hosts;
    size_t inBytes = 0;
    for (auto t : ins) {
        hosts.emplace_back(new Tensor(t, Tensor::CAFFE));
        t->copyToHostTensor(hosts.back().get());
        inBytes += hosts.back()->size();
    }
    auto output = net->getSessionOutput(s, "output");
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

static VARP seeded(std::mt19937& rng, std::vector<int> shape, float scale) {
    size_t n = 1;
    for (int d : shape) n *= (size_t)d;
    std::uniform_real_distribution<float> u(-1.f, 1.f);
    std::vector<float> v(n);
    for (auto& f : v) f = u(rng) * scale;
    return _Const(v.data(), shape, NCHW, halide_type_of<float>());
}
// a GRU layer of D directions on x [T, B, I] with seeded constant weights (uniform in +-1/sqrt(H), biases +-0.1), in the op's
// input order, h0 appended when given
static std::vector<VARP> layer(std::mt19937& rng, int lbr, VARP x, int I, int H, int D, int nout, VARP h0 = nullptr) {
    const float s = 1.f / std::sqrt((float)H);
    std::vector<VARP> in = {x};
    for (int d = 0; d < D; ++d) {
        in.push_back(seeded(rng, {I + H, 2 * H}, s));
        in.push_back(seeded(rng, {1, 2 * H}, 0.1f));
        in.push_back(seeded(rng, {I + H, H}, s));
        in.push_back(seeded(rng, {1, H}, 0.1f));
        in.push_back(seeded(rng, {1, 3 * H}, 0.1f));
    }
    if (h0.get()) in.push_back(h0);
    return gruOp(lbr, H, D, true, nout, in);
}
static VARP dense(std::mt19937& rng, VARP x, int i, int o) {
    return _Add(_MatMul(x, seeded(rng, {i, o}, std::sqrt(3.f / i))), seeded(rng, {o}, 0.05f));
}

// RNNoise-style streaming denoiser chunk (linear_before_reset 0, ONNX's default): `feats` [16, B, 42] and the states `h1_0`,
// `h2_0`, `h3_0` [1, B, 24 / 48 / 96] as graph inputs; a dense layer with tanh to 24; a GRU of H 24 on it; a GRU of H 48 on
// [feats, dense, gru1]; a GRU of H 96 on [feats, gru1, gru2]; a dense layer with sigmoid to 22 band gains.  Outputs: `output`
// [16, B, 22] and every final state `h1_n`, `h2_n`, `h3_n` [1, B, H], so that a caller can feed the next chunk.
static int cmdDenoise(const char* out, int seed) {
    std::mt19937 rng(seed);
    VARP feats = _Input({kDnT, 1, kDnF}, NCHW, halide_type_of<float>());
    feats->setName("feats");
    VARP h0[3];
    const int hs[3] = {kDnH1, kDnH2, kDnH3};
    for (int l = 0; l < 3; ++l) {
        h0[l] = _Input({1, 1, hs[l]}, NCHW, halide_type_of<float>());
        h0[l]->setName("h" + std::to_string(l + 1) + "_0");
    }
    VARP d = _Tanh(dense(rng, feats, kDnF, kDnD));                                          // [16, B, 24]
    auto g1 = layer(rng, 0, d, kDnD, kDnH1, 1, 2, h0[0]);
    VARP y1 = _Reshape(g1[0], {kDnT, -1, kDnH1});
    auto g2 = layer(rng, 0, _Concat({feats, d, y1}, 2), kDnF + kDnD + kDnH1, kDnH2, 1, 2, h0[1]);
    VARP y2 = _Reshape(g2[0], {kDnT, -1, kDnH2});
    auto g3 = layer(rng, 0, _Concat({feats, y1, y2}, 2), kDnF + kDnH1 + kDnH2, kDnH3, 1, 2, h0[2]);
    VARP y3 = _Reshape(g3[0], {kDnT, -1, kDnH3});
    VARP y = _Sigmoid(dense(rng, y3, kDnH3, kDnG));
    y->setName("output");
    std::vector<VARP> outs = {y};
    const std::vector<VARP>* gs[3] = {&g1, &g2, &g3};
    for (int l = 0; l < 3; ++l) {   // the states through a Reshape each, so that every output has a name of its own
        VARP hn = _Reshape((*gs[l])[1], {1, -1, hs[l]});
        hn->setName("h" + std::to_string(l + 1) + "_n");
        outs.push_back(hn);
    }
    Variable::save(outs, out);
    return 0;
}

// BiGRU sequence tagger (linear_before_reset 1): `ids` int32 [64, B] into a GatherV2 embedding [8000, 128]; two bidirectional
// GRUs of H 256 (the second on the first's [64, B, 512]), each consuming Y only; a MatMul to 17 tags and a Softmax:
// `output` [64, B, 17].
static int cmdTagger(const char* out, int seed) {
    std::mt19937 rng(seed);
    VARP ids = _Input({kTgT, 1}, NCHW, halide_type_of<int>());
    ids->setName("ids");
    VARP seq = _GatherV2(seeded(rng, {kTgV, kTgE}, 1.f), ids, _Scalar<int>(0));          // [64, B, 128]
    int I = kTgE;
    for (int l = 0; l < 2; ++l) {
        VARP y = layer(rng, 1, seq, I, kTgH, 2, 1)[0];                                     // [64, 2, B, 256]
        y->setName("bigru" + std::to_string(l));
        seq = _Reshape(_Transpose(y, {0, 2, 1, 3}), {kTgT, -1, 2 * kTgH});
        I = 2 * kTgH;
    }
    VARP y = _Softmax(dense(rng, seq, 2 * kTgH, kTgK), -1);
    y->setName("output");
    Variable::save({y}, out);
    return 0;
}

int main(int argc, char** argv) {
    const std::string cmd = argc > 1 ? argv[1] : "";
    if (cmd == "op" && argc >= 4) return cmdOp(argv[2], argv[3]);
    if (cmd == "run" && argc >= 6) return cmdRun(argv[2], atoi(argv[3]), atoi(argv[4]), argv[5]);
    if (cmd == "chunks" && argc >= 7) return cmdChunks(argv[2], atoi(argv[3]), atoi(argv[4]), atoi(argv[5]), argv[6]);
    if (cmd == "bench" && argc >= 7) return cmdBench(argv[2], atoi(argv[3]), atoi(argv[4]), atoi(argv[5]), atoi(argv[6]));
    if (cmd == "denoise" && argc >= 4) return cmdDenoise(argv[2], atoi(argv[3]));
    if (cmd == "tagger" && argc >= 4) return cmdTagger(argv[2], atoi(argv[3]));
    fprintf(stderr, "usage: refdump_gru op <request> <out> | run <model> <batch> <seed> <outdir> | chunks <model> <batch> <seed> "
                    "<n> <outdir> | bench <model> <batch> <threads> <warmup> <iters> | denoise <out.mnn> <seed> | "
                    "tagger <out.mnn> <seed>\n");
    return 1;
}
