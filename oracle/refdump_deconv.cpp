// refdump_deconv -- the reference's fp32 Deconvolution, for the tests of the deconvolution kernels and their plugin execution.
//
//   refdump_deconv deconv <request> <out>   one Deconvolution / DeconvolutionDepthwise op, built as an OpT the way Express's
//                                           _Deconv (express/NeuralNetWorkOp.cpp) builds it plus the fields _Deconv leaves out
//                                           (pads [t, l, b, r], outPads, an output-shape input, ReLU / ReLU6), run through the
//                                           Express executor on MNN_FORWARD_CPU (REFDUMP_PLUGIN: on the plugin).
//       request: int32 n, ic, ih, iw, oc, kh, kw, sh, sw, pt, pl, pb, pr, dh, dw, oph, opw, same, out_h, out_w, depthwise, relu,
//                relu6, has_bias, then fp32 x [n][ic][ih][iw], w [ic][oc][kh][kw] ([c][kh][kw] depthwise), bias [oc].
//                out_h > 0: an output-shape input {n, out_h, out_w, oc} (hasOutputShape).
//       out:     int32 n, oc, oh, ow, then fp32 y.
//   refdump_deconv chain <batch> <seed> <dir>   conv 3x3 -> deconv 4x4 stride 2 -> depthwise deconv 3x3 -> conv 1x1 on an
//                                           8-channel 10x10 NCHW input, run twice with two inputs (cmdChain).
#include <MNN/expr/Expr.hpp>
#include <MNN/expr/ExprCreator.hpp>
#include <MNN/expr/Executor.hpp>
#include <MNN/expr/ExecutorScope.hpp>
#include <dlfcn.h>
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

static void* g_plugin = nullptr;
static MNNForwardType forwardType() {
    const char* p = getenv("REFDUMP_PLUGIN");
    if (!p || !*p) return MNN_FORWARD_CPU;
    g_plugin = dlopen(p, RTLD_NOW | RTLD_GLOBAL);
    if (!g_plugin) { fprintf(stderr, "refdump_deconv: dlopen(%s): %s\n", p, dlerror()); exit(3); }
    return MNN_FORWARD_CUDA;
}
// the plugin's counts of executions it created and declined, as one JSON line
static void pluginStats() {
    if (!g_plugin) return;
    typedef void (*Fn)(int*, int*);
    Fn fn = (Fn)dlsym(g_plugin, "mnnb200_plugin_stats");
    int c = 0, d = 0;
    if (fn) fn(&c, &d);
    printf("{\"plugin_created\": %d, \"plugin_declined\": %d}\n", c, d);
}

struct Req {
    int32_t n, ic, ih, iw, oc, kh, kw, sh, sw, pt, pl, pb, pr, dh, dw, oph, opw, same, out_h, out_w, depthwise, relu, relu6, has_bias;
};

static VARP deconvOp(VARP x, const Req& r, const float* w, const float* b, VARP outShape) {
    std::unique_ptr<OpT> op(new OpT);
    op->type = r.depthwise ? OpType_DeconvolutionDepthwise : OpType_Deconvolution;
    op->main.type = OpParameter_Convolution2D;
    op->main.value = new Convolution2DT;
    auto conv = op->main.AsConvolution2D();
    conv->common.reset(new Convolution2DCommonT);
    auto& c = *conv->common;
    c.padMode = r.same ? PadMode_SAME : PadMode_CAFFE;
    c.pads = {r.pt, r.pl, r.pb, r.pr};
    if (r.oph || r.opw) c.outPads = {r.oph, r.opw};
    c.strideX = r.sw; c.strideY = r.sh; c.dilateX = r.dw; c.dilateY = r.dh; c.kernelX = r.kw; c.kernelY = r.kh;
    c.group = r.depthwise ? r.oc : 1;
    c.outputCount = r.oc; c.inputCount = r.ic;
    c.relu = r.relu != 0; c.relu6 = r.relu6 != 0;
    c.hasOutputShape = outShape.get() != nullptr;
    const size_t wn = (size_t)(r.depthwise ? 1 : r.ic) * r.oc * r.kh * r.kw;
    conv->weight.assign(w, w + wn);
    conv->bias.assign(r.oc, 0.f);
    if (b) conv->bias.assign(b, b + r.oc);
    std::vector<VARP> in{x};
    if (outShape.get()) in.push_back(outShape);
    return Variable::create(Expr::create(op.get(), in));
}

static int cmdDeconv(const char* reqPath, const char* outPath) {
    auto buf = readFile(reqPath);
    Req r;
    memcpy(&r, buf.data(), sizeof(r));
    const float* x = (const float*)(buf.data() + sizeof(r));
    const size_t xn = (size_t)r.n * r.ic * r.ih * r.iw, wn = (size_t)(r.depthwise ? 1 : r.ic) * r.oc * r.kh * r.kw;
    const float* w = x + xn;
    const float* b = r.has_bias ? w + wn : nullptr;
    BackendConfig bc;
    bc.precision = BackendConfig::Precision_High;
    ExecutorScope scope(Executor::newExecutor(forwardType(), bc, 1));
    VARP in = _Input({r.n, r.ic, r.ih, r.iw}, NCHW, halide_type_of<float>());
    memcpy(in->writeMap<float>(), x, xn * 4);
    VARP shape;
    if (r.out_h > 0) {
        shape = _Input({4}, NCHW, halide_type_of<int>());
        int* s = shape->writeMap<int>();
        s[0] = r.n; s[1] = r.out_h; s[2] = r.out_w; s[3] = r.oc;
    }
    VARP y = deconvOp(in, r, w, b, shape);
    y = _Convert(y, NCHW);
    auto info = y->getInfo();
    if (!info || info->dim.size() != 4) { fprintf(stderr, "refdump_deconv: no output shape\n"); return 2; }
    const float* p = y->readMap<float>();
    if (!p) { fprintf(stderr, "refdump_deconv: compute failed\n"); return 2; }
    std::ofstream o(outPath, std::ios::binary);
    int32_t dims[4] = {info->dim[0], info->dim[1], info->dim[2], info->dim[3]};
    o.write((const char*)dims, sizeof(dims));
    o.write((const char*)p, (size_t)dims[0] * dims[1] * dims[2] * dims[3] * 4);
    pluginStats();
    return 0;
}

static std::vector<float> seeded(std::mt19937& rng, size_t n, float scale) {
    std::uniform_real_distribution<float> u(-1.f, 1.f);
    std::vector<float> v(n);
    for (auto& f : v) f = u(rng) * scale;
    return v;
}

// conv 3x3 -> deconv 4x4 stride 2 -> depthwise deconv 3x3 -> conv 1x1, seeded float weights, run twice on one executor: first
// on the seeded input, then on a second seeded input written into the same input variable.  Each run writes the deconvolution's
// and the graph's output (NCHW fp32) to <dir>/{deconv,output}_<run>.f32.
static int cmdChain(int batch, int seed, const std::string& dir) {
    BackendConfig bc;
    bc.precision = BackendConfig::Precision_High;
    ExecutorScope scope(Executor::newExecutor(forwardType(), bc, 1));
    std::mt19937 rng(seed);
    VARP x = _Input({batch, 8, 10, 10}, NCHW, halide_type_of<float>());
    VARP h = _Conv(seeded(rng, 16 * 8 * 9, 0.4f), seeded(rng, 16, 0.2f), x, {8, 16}, {3, 3}, CAFFE, {1, 1}, {1, 1}, 1, {1, 1},
                   true, false);
    Req r{};
    r.ic = 16; r.oc = 12; r.kh = r.kw = 4; r.sh = r.sw = 2; r.pt = r.pl = r.pb = r.pr = 1; r.dh = r.dw = 1; r.relu = 1;
    auto w1 = seeded(rng, 16 * 12 * 16, 0.25f), b1 = seeded(rng, 12, 0.2f);
    VARP dc = deconvOp(h, r, w1.data(), b1.data(), nullptr);
    Req d{};
    d.ic = d.oc = 12; d.kh = d.kw = 3; d.sh = d.sw = 1; d.pt = d.pl = d.pb = d.pr = 1; d.dh = d.dw = 1; d.depthwise = 1; d.relu6 = 1;
    auto w2 = seeded(rng, 12 * 9, 0.5f), b2 = seeded(rng, 12, 0.2f);
    h = deconvOp(dc, d, w2.data(), b2.data(), nullptr);
    VARP y = _Conv(seeded(rng, 6 * 12, 0.4f), seeded(rng, 6, 0.2f), h, {12, 6}, {1, 1}, VALID, {1, 1}, {1, 1}, 1, {0, 0});
    VARP dcOut = _Convert(dc, NCHW), yOut = _Convert(y, NCHW);
    for (int run = 0; run < 2; ++run) {
        auto in = seeded(rng, (size_t)batch * 8 * 10 * 10, 1.f);
        memcpy(x->writeMap<float>(), in.data(), in.size() * 4);
        for (auto& v : {std::make_pair(std::string("deconv"), dcOut), std::make_pair(std::string("output"), yOut)}) {
            auto info = v.second->getInfo();
            const float* p = v.second->readMap<float>();
            if (!info || !p) { fprintf(stderr, "refdump_deconv chain: compute failed\n"); return 2; }
            std::ofstream o(dir + "/" + v.first + "_" + std::to_string(run) + ".f32", std::ios::binary);
            o.write((const char*)p, (size_t)info->size * 4);
        }
    }
    pluginStats();
    return 0;
}

int main(int argc, char** argv) {
    if (argc >= 4 && std::string(argv[1]) == "deconv") return cmdDeconv(argv[2], argv[3]);
    if (argc >= 5 && std::string(argv[1]) == "chain") return cmdChain(atoi(argv[2]), atoi(argv[3]), argv[4]);
    fprintf(stderr, "usage: refdump_deconv deconv <request> <out> | chain <batch> <seed> <dir>\n");
    return 1;
}
