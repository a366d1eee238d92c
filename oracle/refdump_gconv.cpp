// refdump_gconv -- the reference's grouped fp32 Convolution, for the tests of the grouped conv kernel and its plugin execution.
//
//   refdump_gconv conv <request> <out>      one Convolution op, built as an OpT the way Express's _Conv (express/NeuralNetWorkOp.cpp)
//                                           builds it, with group and inputCount set independently (ConvolutionFloatFactory takes
//                                           group = channels / inputCount when inputCount > 0 differs from the input's channels),
//                                           pads [t, l, b, r] and ReLU / ReLU6, run through the Express executor on
//                                           MNN_FORWARD_CPU (REFDUMP_PLUGIN: on the plugin).
//       request: int32 n, ic, ih, iw, oc, kh, kw, sh, sw, pt, pl, pb, pr, dh, dw, group, input_count, relu, relu6, has_bias, wn,
//                then fp32 x [n][ic][ih][iw], w (wn values, [oc][ic / group][kh][kw]), bias [oc].
//       out:     int32 n, oc, oh, ow, then fp32 y.
//   refdump_gconv block <batch> <seed> <dir>   a ResNeXt stride-2 bottleneck (1x1 -> grouped 3x3, 32 groups, stride 2 -> 1x1, plus a
//                                           1x1 stride-2 projection shortcut, add, ReLU) on a 64-channel 16x16 NCHW input, then a
//                                           stride-1 bottleneck with an identity shortcut, run twice with two inputs (cmdBlock).
//   refdump_gconv resnext <out.mnn> <seed>  writes ResNeXt-50 32x4d built with Express, seeded fp32 weights (cmdResnext).
#include <MNN/expr/Expr.hpp>
#include <MNN/expr/ExprCreator.hpp>
#include <MNN/expr/Executor.hpp>
#include <MNN/expr/ExecutorScope.hpp>
#include <dlfcn.h>
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

static void* g_plugin = nullptr;
static MNNForwardType forwardType() {
    const char* p = getenv("REFDUMP_PLUGIN");
    if (!p || !*p) return MNN_FORWARD_CPU;
    g_plugin = dlopen(p, RTLD_NOW | RTLD_GLOBAL);
    if (!g_plugin) { fprintf(stderr, "refdump_gconv: dlopen(%s): %s\n", p, dlerror()); exit(3); }
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
    int32_t n, ic, ih, iw, oc, kh, kw, sh, sw, pt, pl, pb, pr, dh, dw, group, input_count, relu, relu6, has_bias, wn;
};

static VARP convOp(VARP x, const Req& r, const float* w, const float* b) {
    std::unique_ptr<OpT> op(new OpT);
    op->type = OpType_Convolution;
    op->main.type = OpParameter_Convolution2D;
    op->main.value = new Convolution2DT;
    auto conv = op->main.AsConvolution2D();
    conv->common.reset(new Convolution2DCommonT);
    auto& c = *conv->common;
    c.padMode = PadMode_CAFFE;
    c.pads = {r.pt, r.pl, r.pb, r.pr};
    c.strideX = r.sw; c.strideY = r.sh; c.dilateX = r.dw; c.dilateY = r.dh; c.kernelX = r.kw; c.kernelY = r.kh;
    c.group = r.group;
    c.outputCount = r.oc; c.inputCount = r.input_count;
    c.relu = r.relu != 0; c.relu6 = r.relu6 != 0;
    conv->weight.assign(w, w + r.wn);
    conv->bias.assign(r.oc, 0.f);
    if (b) conv->bias.assign(b, b + r.oc);
    return Variable::create(Expr::create(op.get(), {x}));
}

static int cmdConv(const char* reqPath, const char* outPath) {
    auto buf = readFile(reqPath);
    Req r;
    memcpy(&r, buf.data(), sizeof(r));
    const float* x = (const float*)(buf.data() + sizeof(r));
    const size_t xn = (size_t)r.n * r.ic * r.ih * r.iw;
    const float* w = x + xn;
    const float* b = r.has_bias ? w + r.wn : nullptr;
    BackendConfig bc;
    bc.precision = BackendConfig::Precision_High;
    ExecutorScope scope(Executor::newExecutor(forwardType(), bc, 1));
    VARP in = _Input({r.n, r.ic, r.ih, r.iw}, NCHW, halide_type_of<float>());
    memcpy(in->writeMap<float>(), x, xn * 4);
    VARP y = _Convert(convOp(in, r, w, b), NCHW);
    auto info = y->getInfo();
    if (!info || info->dim.size() != 4) { fprintf(stderr, "refdump_gconv: no output shape\n"); return 2; }
    const float* p = y->readMap<float>();
    if (!p) { fprintf(stderr, "refdump_gconv: compute failed\n"); return 2; }
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

// a seeded float conv with pads (k - 1) / 2, weights uniform in +-gain sqrt(3 / fan_in) (fan_in = ic / group * k * k)
static VARP conv(std::mt19937& rng, VARP x, int ic, int oc, int k, int stride, int group, bool relu, float gain = 1.41f) {
    const int fan = ic / group * k * k;
    auto w = seeded(rng, (size_t)oc * fan, gain * std::sqrt(3.f / fan));
    auto b = seeded(rng, oc, 0.1f);
    return _Conv(std::move(w), std::move(b), x, {ic, oc}, {k, k}, CAFFE, {stride, stride}, {1, 1}, group, {(k - 1) / 2, (k - 1) / 2},
                 relu, false);
}

// ResNeXt bottleneck (32 groups): 1x1 -> grouped 3x3 (stride) -> 1x1, shortcut (a 1x1 projection when the shape changes), add,
// ReLU.  *grouped, when given, receives the grouped 3x3's output.
static VARP bottleneck(std::mt19937& rng, VARP x, int ic, int width, int oc, int stride, VARP* grouped = nullptr) {
    VARP h = conv(rng, x, ic, width, 1, 1, 1, true);
    h = conv(rng, h, width, width, 3, stride, 32, true);
    if (grouped) *grouped = h;
    h = conv(rng, h, width, oc, 1, 1, 1, false, 0.5f);
    VARP s = (stride != 1 || ic != oc) ? conv(rng, x, ic, oc, 1, stride, 1, false, 0.5f) : x;
    return _Relu(_Add(h, s));
}

// two bottlenecks on one executor, each run twice with two seeded inputs written into the same input variable.  Each run writes
// the first block's grouped conv output and the graph's output (NCHW fp32) to <dir>/{grouped,output}_<run>.f32.
static int cmdBlock(int batch, int seed, const std::string& dir) {
    BackendConfig bc;
    bc.precision = BackendConfig::Precision_High;
    ExecutorScope scope(Executor::newExecutor(forwardType(), bc, 1));
    std::mt19937 rng(seed);
    VARP x = _Input({batch, 64, 16, 16}, NCHW, halide_type_of<float>());
    VARP grouped;
    VARP h = bottleneck(rng, x, 64, 128, 256, 2, &grouped);
    VARP y = bottleneck(rng, h, 256, 128, 256, 1);
    VARP gOut = _Convert(grouped, NCHW), yOut = _Convert(y, NCHW);
    for (int run = 0; run < 2; ++run) {
        auto in = seeded(rng, (size_t)batch * 64 * 16 * 16, 1.f);
        memcpy(x->writeMap<float>(), in.data(), in.size() * 4);
        for (auto& v : {std::make_pair(std::string("grouped"), gOut), std::make_pair(std::string("output"), yOut)}) {
            auto info = v.second->getInfo();
            const float* p = v.second->readMap<float>();
            if (!info || !p) { fprintf(stderr, "refdump_gconv block: compute failed\n"); return 2; }
            std::ofstream o(dir + "/" + v.first + "_" + std::to_string(run) + ".f32", std::ios::binary);
            o.write((const char*)p, (size_t)info->size * 4);
        }
    }
    pluginStats();
    return 0;
}

// ResNeXt-50 32x4d (Xie et al. 2017): 7x7 / 2 stem, 3x3 / 2 max pool, stages of 3 / 4 / 6 / 3 bottlenecks of group width 4
// (width 128 / 256 / 512 / 1024, outputs 256 / 512 / 1024 / 2048, the first block of stages 2-4 with stride 2), 7x7 average
// pool and the 1000-way classifier as a 1x1 conv.  No batch norm (a converted model has it folded into the conv weights).
static int cmdResnext(const char* out, int seed) {
    std::mt19937 rng(seed);
    VARP x = _Input({1, 3, 224, 224}, NCHW, halide_type_of<float>());
    x->setName("input");
    VARP h = conv(rng, x, 3, 64, 7, 2, 1, true);
    h = _MaxPool(h, {3, 3}, {2, 2}, CAFFE, {1, 1});
    const int blocks[4] = {3, 4, 6, 3};
    int ic = 64;
    for (int s = 0; s < 4; ++s) {
        const int width = 128 << s, oc = 256 << s;
        for (int b = 0; b < blocks[s]; ++b) {
            h = bottleneck(rng, h, ic, width, oc, (s > 0 && b == 0) ? 2 : 1);
            ic = oc;
        }
    }
    h = _AvePool(h, {7, 7}, {1, 1}, VALID);
    h = conv(rng, h, 2048, 1000, 1, 1, 1, false, 1.f);
    h = _Convert(h, NCHW);
    h->setName("output");
    Variable::save({h}, out);
    return 0;
}

int main(int argc, char** argv) {
    if (argc >= 4 && std::string(argv[1]) == "conv") return cmdConv(argv[2], argv[3]);
    if (argc >= 5 && std::string(argv[1]) == "block") return cmdBlock(atoi(argv[2]), atoi(argv[3]), argv[4]);
    if (argc >= 4 && std::string(argv[1]) == "resnext") return cmdResnext(argv[2], atoi(argv[3]));
    fprintf(stderr, "usage: refdump_gconv conv <request> <out> | block <batch> <seed> <dir> | resnext <out.mnn> <seed>\n");
    return 1;
}
