// refdump_rnn -- the reference's ONNX LSTM and RNN (OpType_LSTM / OpType_RNN), for the tests of the recurrence kernel and its
// plugin execution.
//
//   refdump_rnn op <request> <out>     one op (built as an OpT) through the Express executor on MNN_FORWARD_CPU
//                                      (REFDUMP_PLUGIN: on the plugin), once per input set given, on one executor.
//       request: int32 cell (0 LSTM, 1 RNN), T, B, I, H, D, nin (4: X, W, R, B; 5: + h0; 6: + c0), clip (the LSTM parameter's
//                clippingThreshold, as a float's bits), count; then count sets of the nin fp32 inputs' raw data.
//       out:     per set, the op's outputs' raw fp32 data in order (Y [T, D, B, H], Y_h [D, B, H][, Y_c [D, B, H]]).
//   refdump_rnn run <model.mnn> <batch> <seed> <outdir>   every command's fp32 outputs (index.txt), with every input filled by
//                                      fillInputs; REFDUMP_RUN_REPEATS: that many plain runSessions first (on the plugin: eager,
//                                      then a captured graph replayed), the last first output in output_plain.f32.
//   refdump_rnn chunks <model.mnn> <batch> <seed> <n> <outdir>   kws_f32.mnn over n chained chunks: each chunk's outputs
//                                      (chunk<k>_<name>.f32), the final states fed back as the next chunk's initial states.
//   refdump_rnn bench <model.mnn> <batch> <threads> <warmup> <iters>   copy in + runSession + copy out, ms per iteration.
//   refdump_rnn crnn <out.mnn> <seed>  a CRNN-style text recogniser with seeded weights (cmdCrnn).
//   refdump_rnn kws <out.mnn> <seed>   a streaming keyword-spotter chunk with seeded weights (cmdKws).
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
    if (!g_plugin) { fprintf(stderr, "refdump_rnn: dlopen(%s): %s\n", p, dlerror()); exit(3); }
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

// the LSTM / RNN op of ONNX models as the converter writes it: the LSTM parameter carries only outputCount (H)
static std::vector<VARP> rnnOp(int cell, int H, float clip, const std::vector<VARP>& in) {
    std::unique_ptr<OpT> op(new OpT);
    op->type = cell == 0 ? OpType_LSTM : OpType_RNN;
    op->main.type = OpParameter_LSTM;
    op->main.value = new LSTMT;
    op->main.AsLSTM()->outputCount = H;
    op->main.AsLSTM()->clippingThreshold = clip;
    const int nout = cell == 0 ? 3 : 2;
    EXPRP e = Expr::create(op.get(), in, nout);
    std::vector<VARP> out;
    for (int i = 0; i < nout; ++i) out.push_back(Variable::create(e, i));
    return out;
}

static int cmdOp(const char* reqPath, const char* outPath) {
    auto buf = readFile(reqPath);
    const int32_t* q = (const int32_t*)buf.data();
    const int cell = q[0], T = q[1], B = q[2], I = q[3], H = q[4], D = q[5], nin = q[6];
    float clip;
    memcpy(&clip, &q[7], 4);
    const int count = q[8];
    q += 9;
    const int G = cell == 0 ? 4 : 1;
    std::vector<std::vector<int>> dims = {{T, B, I}, {D, G * H, I}, {D, G * H, H}, {D, G * H}, {D, B, H}, {D, B, H}};
    dims.resize(nin);
    BackendConfig bc;
    bc.precision = BackendConfig::Precision_High;
    ExecutorScope scope(Executor::newExecutor(forwardType(), bc, 1));
    std::vector<VARP> xs;
    for (int i = 0; i < nin; ++i) xs.push_back(_Input(dims[i], NCHW, halide_type_of<float>()));
    auto ys = rnnOp(cell, H, clip, xs);
    const char* data = (const char*)q;
    std::ofstream o(outPath, std::ios::binary);
    for (int c = 0; c < count; ++c) {
        for (int i = 0; i < nin; ++i) {
            size_t n = 1;
            for (int d : dims[i]) n *= (size_t)d;
            memcpy(xs[i]->writeMap<char>(), data, n * 4);
            data += n * 4;
        }
        for (auto& y : ys) {
            auto info = y->getInfo();
            const char* py = y->readMap<char>();
            if (!info || !py) { fprintf(stderr, "refdump_rnn: compute failed\n"); return 2; }
            o.write(py, (size_t)info->size * 4);
        }
    }
    pluginStats();
    return 0;
}

// ---- the fixtures' geometry, shared by their writers and fillInputs
static const int kImgH = 32, kImgW = 128, kCrnnH = 256, kClasses = 37;    // CRNN: grey 32 x 128 -> T = 32, 2 x BiLSTM(256)
static const int kKwsT = 16, kKwsF = 40, kKwsH = 128, kKwsR = 64, kKwsK = 12;  // KWS: 16 frames of 40 features, LSTM 128, RNN 64

// the batch axis of a fixture input: the image's dim 0; the sequences' and states' dim 1
static int batchAxis(const Tensor* t) { return t->dimensions() == 4 ? 0 : 1; }
static std::vector<Tensor*> sessionInputs(Interpreter* net, Session* s, int batch) {
    std::vector<Tensor*> ins;
    for (auto& kv : net->getSessionInputAll(s)) {
        auto shape = kv.second->shape();
        shape[batchAxis(kv.second)] = batch;
        net->resizeTensor(kv.second, shape);
        ins.push_back(kv.second);
    }
    net->resizeSession(s);
    return ins;
}
// every fp32 input uniform in [-1, 1] from `seed` (states at half that)
static void fillInputs(Interpreter* net, Session* s, int seed) {
    std::mt19937 rng(seed);
    for (auto& kv : net->getSessionInputAll(s)) {
        Tensor host(kv.second, Tensor::CAFFE);
        std::uniform_real_distribution<float> u(-1.f, 1.f);
        const float sc = kv.first == "feats" || kv.first == "image" ? 1.f : 0.5f;
        auto p = host.host<float>();
        for (int i = 0; i < host.elementSize(); ++i) p[i] = u(rng) * sc;
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
    if (!s) { fprintf(stderr, "refdump_rnn run: createSession failed\n"); return 2; }
    sessionInputs(net.get(), s, batch);
    fillInputs(net.get(), s, seed);
    auto output = net->getSessionOutput(s, "output");
    if (const char* rp = getenv("REFDUMP_RUN_REPEATS")) {
        const int reps = atoi(rp);
        Tensor host(output, Tensor::CAFFE);
        for (int i = 0; i < reps; ++i) {
            fillInputs(net.get(), s, seed);
            if (net->runSession(s) != NO_ERROR) { fprintf(stderr, "refdump_rnn run: plain runSession failed\n"); return 2; }
            output->copyToHostTensor(&host);
        }
        if (reps > 0) writeFile(dir + "/output_plain.f32", host.host<float>(), host.size());
        fillInputs(net.get(), s, seed);
    }
    FILE* idx = fopen((dir + "/index.txt").c_str(), "w");
    if (!idx) { fprintf(stderr, "refdump_rnn run: cannot write %s/index.txt\n", dir.c_str()); return 2; }
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
    if (code != NO_ERROR) { fprintf(stderr, "refdump_rnn run: runSession -> %d\n", (int)code); return 2; }
    Tensor host(output, Tensor::CAFFE);
    output->copyToHostTensor(&host);
    writeFile(dir + "/output.f32", host.host<float>(), host.size());
    pluginStats();
    return 0;
}

// kws_f32.mnn over n chunks: chunk k's features from seed + k, its final states the next chunk's initial states
static int cmdChunks(const char* model, int batch, int seed, int chunks, const std::string& dir) {
    std::shared_ptr<Interpreter> net(Interpreter::createFromFile(model), Interpreter::destroy);
    auto s = makeSession(net.get(), 4);
    if (!s) { fprintf(stderr, "refdump_rnn chunks: createSession failed\n"); return 2; }
    sessionInputs(net.get(), s, batch);
    fillInputs(net.get(), s, seed);
    const std::map<std::string, std::string> feed = {{"h_n", "h0"}, {"c_n", "c0"}, {"hr_n", "h0r"}};
    for (int k = 0; k < chunks; ++k) {
        Tensor feats(net->getSessionInput(s, "feats"), Tensor::CAFFE);
        std::mt19937 rng(seed + 1 + k);
        std::uniform_real_distribution<float> u(-1.f, 1.f);
        for (int i = 0; i < feats.elementSize(); ++i) feats.host<float>()[i] = u(rng);
        net->getSessionInput(s, "feats")->copyFromHostTensor(&feats);
        if (net->runSession(s) != NO_ERROR) { fprintf(stderr, "refdump_rnn chunks: runSession failed\n"); return 2; }
        for (const char* name : {"output", "h_n", "c_n", "hr_n"}) {
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
    if (!s) { fprintf(stderr, "refdump_rnn bench: createSession failed\n"); return 2; }
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
static VARP conv(std::mt19937& rng, VARP x, int ic, int oc) {
    return _Conv(uniform(rng, (size_t)oc * ic * 9, std::sqrt(3.f / (ic * 9))), uniform(rng, oc, 0.05f), x, {ic, oc}, {3, 3}, SAME,
                 {1, 1}, {1, 1}, 1, {0, 0}, true, false);
}
// an LSTM / RNN layer of D directions on x [T, B, I] with seeded constant weights (W, R uniform in +-1/sqrt(H), bias +-0.1)
static std::vector<VARP> layer(std::mt19937& rng, int cell, VARP x, int I, int H, int D, std::vector<VARP> states = {}) {
    const int G = cell == 0 ? 4 : 1;
    const float s = 1.f / std::sqrt((float)H);
    std::vector<VARP> in = {x, seeded(rng, {D, G * H, I}, s), seeded(rng, {D, G * H, H}, s), seeded(rng, {D, G * H}, 0.1f)};
    in.insert(in.end(), states.begin(), states.end());
    return rnnOp(cell, H, 0.f, in);
}

// CRNN-style recogniser: `image` [B, 1, 32, 128]; 3x3 conv + ReLU stages 1->64 (pool 2x2), 64->128 (pool 2x2), 128->256, 256->256
// (pool 2x1), 256->256 (pool 4x1) to [B, 256, 1, 32]; a Raster to [T = 32, B, 256]; two bidirectional LSTMs of H = 256 with the
// transpose / reshape of Y [T, 2, B, 256] to [T, B, 512] between them; a MatMul to 37 classes and a Softmax: `output` [32, B, 37].
static int cmdCrnn(const char* out, int seed) {
    std::mt19937 rng(seed);
    VARP img = _Input({1, 1, kImgH, kImgW}, NCHW, halide_type_of<float>());
    img->setName("image");
    VARP x = _Convert(img, NC4HW4);
    x = _MaxPool(conv(rng, x, 1, 64), {2, 2}, {2, 2});
    x = _MaxPool(conv(rng, x, 64, 128), {2, 2}, {2, 2});
    x = conv(rng, x, 128, 256);
    x = _MaxPool(conv(rng, x, 256, 256), {2, 1}, {2, 1});
    x = _MaxPool(conv(rng, x, 256, 256), {4, 1}, {4, 1});
    x = _Convert(x, NCHW);                                                  // [B, 256, 1, 32]
    VARP seq = _Transpose(_Reshape(x, {0, kCrnnH, kImgW / 4}), {2, 0, 1});  // [32, B, 256]
    for (int l = 0; l < 2; ++l) {
        VARP y = layer(rng, 0, seq, l == 0 ? kCrnnH : 2 * kCrnnH, kCrnnH, 2)[0];   // [32, 2, B, 256]
        y->setName("bilstm" + std::to_string(l));
        seq = _Reshape(_Transpose(y, {0, 2, 1, 3}), {kImgW / 4, -1, 2 * kCrnnH});
    }
    VARP logits = _Add(_MatMul(seq, seeded(rng, {2 * kCrnnH, kClasses}, std::sqrt(3.f / (2 * kCrnnH)))), seeded(rng, {kClasses}, 0.05f));
    VARP y = _Softmax(logits, -1);
    y->setName("output");
    Variable::save({y}, out);
    return 0;
}

// streaming keyword-spotter chunk: `feats` [16, B, 40] and the states `h0`, `c0` [1, B, 128], `h0r` [1, B, 64] as graph inputs;
// an LSTM of H = 128, an RNN of H = 64 with its own h0 over the LSTM's Y, then a MatMul of the RNN's last state to 12 keywords
// and a Softmax.  Outputs: `output` [B, 12] and every final state, `h_n`, `c_n` [1, B, 128] and `hr_n` [1, B, 64], so that a
// caller can feed the next chunk.
static int cmdKws(const char* out, int seed) {
    std::mt19937 rng(seed);
    VARP feats = _Input({kKwsT, 1, kKwsF}, NCHW, halide_type_of<float>());
    feats->setName("feats");
    VARP h0 = _Input({1, 1, kKwsH}, NCHW, halide_type_of<float>());
    h0->setName("h0");
    VARP c0 = _Input({1, 1, kKwsH}, NCHW, halide_type_of<float>());
    c0->setName("c0");
    VARP h0r = _Input({1, 1, kKwsR}, NCHW, halide_type_of<float>());
    h0r->setName("h0r");
    auto l1 = layer(rng, 0, feats, kKwsF, kKwsH, 1, {h0, c0});
    VARP seq = _Reshape(l1[0], {kKwsT, -1, kKwsH});
    auto l2 = layer(rng, 1, seq, kKwsH, kKwsR, 1, {h0r});
    VARP last = _Reshape(l2[1], {-1, kKwsR});
    VARP y = _Softmax(_Add(_MatMul(last, seeded(rng, {kKwsR, kKwsK}, std::sqrt(3.f / kKwsR))), seeded(rng, {kKwsK}, 0.05f)), -1);
    y->setName("output");
    l1[0]->setName("lstm");
    l2[0]->setName("rnn");
    // the states through a Reshape each, so that every output has a name of its own (the LSTM's outputs share its expr's)
    VARP hn = _Reshape(l1[1], {1, -1, kKwsH}), cn = _Reshape(l1[2], {1, -1, kKwsH}), hrn = _Reshape(l2[1], {1, -1, kKwsR});
    hn->setName("h_n");
    cn->setName("c_n");
    hrn->setName("hr_n");
    Variable::save({y, hn, cn, hrn}, out);
    return 0;
}

int main(int argc, char** argv) {
    const std::string cmd = argc > 1 ? argv[1] : "";
    if (cmd == "op" && argc >= 4) return cmdOp(argv[2], argv[3]);
    if (cmd == "run" && argc >= 6) return cmdRun(argv[2], atoi(argv[3]), atoi(argv[4]), argv[5]);
    if (cmd == "chunks" && argc >= 7) return cmdChunks(argv[2], atoi(argv[3]), atoi(argv[4]), atoi(argv[5]), argv[6]);
    if (cmd == "bench" && argc >= 7) return cmdBench(argv[2], atoi(argv[3]), atoi(argv[4]), atoi(argv[5]), atoi(argv[6]));
    if (cmd == "crnn" && argc >= 4) return cmdCrnn(argv[2], atoi(argv[3]));
    if (cmd == "kws" && argc >= 4) return cmdKws(argv[2], atoi(argv[3]));
    fprintf(stderr, "usage: refdump_rnn op <request> <out> | run <model> <batch> <seed> <outdir> | chunks <model> <batch> <seed> "
                    "<n> <outdir> | bench <model> <batch> <threads> <warmup> <iters> | crnn <out.mnn> <seed> | kws <out.mnn> <seed>\n");
    return 1;
}
