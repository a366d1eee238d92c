// refdump_interp -- the reference's fp32 Interp / Resize, for the tests of the Interp kernel and its plugin execution.
//
//   refdump_interp op <request> <out>   one Interp op, built as an OpT the way Express's _Interp (express/NeuralNetWorkOp.cpp)
//                                       builds it plus the fields _Interp leaves out (ctm, halfPixelCenters, a scales or size
//                                       input), run through the Express executor on MNN_FORWARD_CPU (REFDUMP_PLUGIN: on the
//                                       plugin), once per input given, on one executor.
//       request: int32 n, c, ih, iw, resizeType, ctm, alignCorners, halfPixelCenters, outputHeight, outputWidth, nhwc, mode,
//                fp32 heightScale, widthScale, s0, s1, int32 count, then count fp32 inputs in the input's layout (NCHW, or NHWC
//                when nhwc).  mode 1: a float scales input {1, 1, s0, s1}; mode 2: an int32 size input {s0, s1}.
//       out:     int32 n, c, oh, ow, then count fp32 outputs, NCHW.
//   refdump_interp seg <out.mnn> <seed>   writes a compact DeepLab-v3-style segmentation net with seeded weights (cmdSeg).
//   refdump_interp fpn <out.mnn> <seed>   writes a nearest x2 FPN / YOLO-style neck with one Resize (cmdFpn).
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
    if (!g_plugin) { fprintf(stderr, "refdump_interp: dlopen(%s): %s\n", p, dlerror()); exit(3); }
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
    int32_t n, c, ih, iw, resizeType, ctm, alignCorners, halfPixel, outH, outW, nhwc, mode;
    float heightScale, widthScale, s0, s1;
    int32_t count;
};

static int cmdOp(const char* reqPath, const char* outPath) {
    auto buf = readFile(reqPath);
    Req r;
    memcpy(&r, buf.data(), sizeof(r));
    const float* data = (const float*)(buf.data() + sizeof(r));
    const size_t xn = (size_t)r.n * r.c * r.ih * r.iw;
    BackendConfig bc;
    bc.precision = BackendConfig::Precision_High;
    ExecutorScope scope(Executor::newExecutor(forwardType(), bc, 1));
    VARP x = r.nhwc ? _Input({r.n, r.ih, r.iw, r.c}, NHWC, halide_type_of<float>())
                    : _Input({r.n, r.c, r.ih, r.iw}, NCHW, halide_type_of<float>());
    std::unique_ptr<OpT> op(new OpT);
    op->type = OpType_Interp;
    op->main.type = OpParameter_Interp;
    auto p = new InterpT;
    op->main.value = p;
    p->resizeType = r.resizeType;
    p->ctm = (CoordinateTransformationMode)r.ctm;
    p->alignCorners = r.alignCorners != 0;
    p->halfPixelCenters = r.halfPixel != 0;
    p->outputHeight = r.outH; p->outputWidth = r.outW;
    p->heightScale = r.heightScale; p->widthScale = r.widthScale;
    std::vector<VARP> in{x};
    if (r.mode == 1) {
        const float s[4] = {1.f, 1.f, r.s0, r.s1};
        in.push_back(_Const(s, {4}, NCHW, halide_type_of<float>()));
    } else if (r.mode == 2) {
        const int s[2] = {(int)r.s0, (int)r.s1};
        in.push_back(_Const(s, {2}, NCHW, halide_type_of<int>()));
    }
    VARP y = _Convert(Variable::create(Expr::create(op.get(), in)), NCHW);
    std::ofstream o(outPath, std::ios::binary);
    for (int i = 0; i < r.count; ++i) {
        memcpy(x->writeMap<float>(), data + i * xn, xn * 4);
        auto info = y->getInfo();
        const float* py = y->readMap<float>();
        if (!info || info->dim.size() != 4 || !py) { fprintf(stderr, "refdump_interp: compute failed\n"); return 2; }
        if (i == 0) {
            int32_t dims[4] = {info->dim[0], info->dim[1], info->dim[2], info->dim[3]};
            o.write((const char*)dims, sizeof(dims));
        }
        o.write((const char*)py, (size_t)info->size * 4);
    }
    pluginStats();
    return 0;
}

static std::vector<float> seeded(std::mt19937& rng, size_t n, float scale) {
    std::uniform_real_distribution<float> u(-1.f, 1.f);
    std::vector<float> v(n);
    for (auto& f : v) f = u(rng) * scale;
    return v;
}
// a k x k conv (group 1, or depthwise when group == ic == oc) with "same" pads for its dilation, seeded He-like weights
static VARP conv(std::mt19937& rng, VARP x, int ic, int oc, int k, int stride, bool relu, int dilate = 1, int group = 1) {
    const int fan = ic / group * k * k;
    auto w = seeded(rng, (size_t)oc * fan, 1.41f * std::sqrt(3.f / fan));
    auto b = seeded(rng, oc, 0.1f);
    const int pad = dilate * (k - 1) / 2;
    return _Conv(std::move(w), std::move(b), x, {ic, oc}, {k, k}, CAFFE, {stride, stride}, {dilate, dilate}, group, {pad, pad},
                 relu, false);
}
// ArgMax over `axis` with topK 1, as the model converters write it (Express's _ArgMax leaves topK 0)
static VARP argMax(VARP x, int axis) {
    std::unique_ptr<OpT> op(new OpT);
    op->type = OpType_ArgMax;
    op->main.type = OpParameter_ArgMax;
    op->main.value = new ArgMaxT;
    op->main.AsArgMax()->axis = axis;
    op->main.AsArgMax()->topK = 1;
    return Variable::create(Expr::create(std::move(op), {x}));
}
static void save(VARP h, const char* out) {
    h->setName("output");
    Variable::save({h}, out);
}

// DeepLab-v3 in small (Chen et al. 2017, with the v3+ decoder): a 3 x 128 x 128 input, a strided conv / depthwise backbone to
// stride 8 with a stride-2 low-level branch, ASPP (1x1, 3x3 at dilations 2 and 4, and image pooling: global average pool ->
// 1x1 -> bilinear upsample from 1x1), concat -> 1x1, x4 bilinear align-corners, concat with the projected low-level features,
// 3x3 to 21 classes, x2 bilinear to the input size, ArgMax over the classes.
static int cmdSeg(const char* out, int seed) {
    std::mt19937 rng(seed);
    VARP x = _Input({1, 3, 128, 128}, NCHW, halide_type_of<float>());
    x->setName("input");
    VARP low = conv(rng, x, 3, 16, 3, 2, true);                       // 64 x 64
    VARP h = conv(rng, low, 16, 32, 3, 2, true);                      // 32 x 32
    h = conv(rng, h, 32, 32, 3, 2, true, 1, 32);                      // 16 x 16, depthwise
    h = conv(rng, h, 32, 64, 1, 1, true);
    VARP b0 = conv(rng, h, 64, 32, 1, 1, true);
    VARP b1 = conv(rng, h, 64, 32, 3, 1, true, 2);
    VARP b2 = conv(rng, h, 64, 32, 3, 1, true, 4);
    VARP pool = conv(rng, _AvePool(h, {16, 16}, {1, 1}, VALID), 64, 32, 1, 1, true);
    VARP b3 = _Interp({pool}, 0.f, 0.f, 16, 16, 2, false);
    h = conv(rng, _Concat({b0, b1, b2, b3}, 1), 128, 32, 1, 1, true);
    h = _Interp({h}, 0.f, 0.f, 64, 64, 2, true);                      // x4, align corners
    h = _Concat({h, conv(rng, low, 16, 8, 1, 1, true)}, 1);
    h = conv(rng, h, 40, 21, 3, 1, false);
    h = _Interp({h}, 0.f, 0.f, 128, 128, 2, false);                   // x2 to the input size
    save(argMax(_Convert(h, NCHW), 1), out);
    return 0;
}

// A YOLO / FPN-style neck on a 3 x 160 x 160 input: a stride-2 conv backbone (C3 at 40, C4 at 20, C5 at 10), top-down nearest
// x2 upsamples concatenated with the lateral features and fused by 3x3 convs, then one Resize (x2, bilinear) and a 1x1 head.
static int cmdFpn(const char* out, int seed) {
    std::mt19937 rng(seed);
    VARP x = _Input({1, 3, 160, 160}, NCHW, halide_type_of<float>());
    x->setName("input");
    VARP h = conv(rng, x, 3, 16, 3, 2, true);                         // 80
    VARP c3 = conv(rng, h, 16, 32, 3, 2, true);                       // 40
    VARP c4 = conv(rng, c3, 32, 64, 3, 2, true);                      // 20
    VARP c5 = conv(rng, c4, 64, 128, 3, 2, true);                     // 10
    VARP p5 = conv(rng, c5, 128, 64, 1, 1, true);
    VARP p4 = conv(rng, _Concat({_Interp({p5}, 2.f, 2.f, 0, 0, 1, false), c4}, 1), 128, 64, 3, 1, true);
    VARP l4 = conv(rng, p4, 64, 32, 1, 1, true);
    VARP p3 = conv(rng, _Concat({_Interp({l4}, 2.f, 2.f, 0, 0, 1, false), c3}, 1), 64, 32, 3, 1, true);
    h = conv(rng, _Resize(p3, 2.f, 2.f), 32, 8, 1, 1, false);
    save(_Convert(h, NCHW), out);
    return 0;
}

int main(int argc, char** argv) {
    if (argc >= 4 && std::string(argv[1]) == "op") return cmdOp(argv[2], argv[3]);
    if (argc >= 4 && std::string(argv[1]) == "seg") return cmdSeg(argv[2], atoi(argv[3]));
    if (argc >= 4 && std::string(argv[1]) == "fpn") return cmdFpn(argv[2], atoi(argv[3]));
    fprintf(stderr, "usage: refdump_interp op <request> <out> | seg <out.mnn> <seed> | fpn <out.mnn> <seed>\n");
    return 1;
}
