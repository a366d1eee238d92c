// refdump_grid_sample -- the reference's fp32 GridSample, for the tests of the GridSample kernel and its plugin execution.
//
//   refdump_grid_sample op <request> <out>   one GridSample op, built by Express's _GridSample, run through the Express executor
//                                            on MNN_FORWARD_CPU (REFDUMP_PLUGIN: on the plugin), once per input set given, on one
//                                            executor.
//       request: int32 rank, n, c, id, ih, iw, od, oh, ow, mode (0 bilinear, 1 nearest), padding (0 zeros, 1 border, 2
//                reflection), alignCorners, count, linear, then count sets of (x NCHW fp32, grid fp32).  Rank 4 ignores id and
//                od.  x reaches the op in NC4HW4, as the model converter feeds it; linear 1 hands it over in its NCHW layout
//                instead (CPUGridSample then reads the linear buffer as if it were packed: oracle/grid_sample_oracle.py).
//       out:     int32 rank, then rank dims, then count fp32 outputs, NCHW.
//   refdump_grid_sample flow <out.mnn> <seed>   writes a two-frame flow-warp net with seeded weights (cmdFlow).
//   refdump_grid_sample lut <out.mnn> <seed>    writes an image-adaptive 3D-LUT enhancer with seeded weights (cmdLut).
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
    if (!g_plugin) { fprintf(stderr, "refdump_grid_sample: dlopen(%s): %s\n", p, dlerror()); exit(3); }
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
    int32_t rank, n, c, id, ih, iw, od, oh, ow, mode, padding, align, count, linear;
};

static int cmdOp(const char* reqPath, const char* outPath) {
    auto buf = readFile(reqPath);
    Req r;
    memcpy(&r, buf.data(), sizeof(r));
    const float* data = (const float*)(buf.data() + sizeof(r));
    const bool d3 = r.rank == 5;
    INTS xs = d3 ? INTS{r.n, r.c, r.id, r.ih, r.iw} : INTS{r.n, r.c, r.ih, r.iw};
    INTS gs = d3 ? INTS{r.n, r.od, r.oh, r.ow, 3} : INTS{r.n, r.oh, r.ow, 2};
    size_t xn = 1, gn = 1;
    for (int v : xs) xn *= v;
    for (int v : gs) gn *= v;
    BackendConfig bc;
    bc.precision = BackendConfig::Precision_High;
    ExecutorScope scope(Executor::newExecutor(forwardType(), bc, 1));
    VARP x = _Input(xs, NCHW, halide_type_of<float>());
    VARP g = _Input(gs, NCHW, halide_type_of<float>());
    const GridSamplePaddingMode pad = r.padding == 1 ? GRID_SAMPLE_PADDING_BORDER
                                      : (r.padding == 2 ? GRID_SAMPLE_PADDING_REFLECTION : GRID_SAMPLE_PADDING_ZEROS);
    // the CPU samples x in its packed NC4HW4 layout, as a converted model feeds it (the converter inserts the conversion)
    VARP y = _Convert(_GridSample(r.linear ? x : _Convert(x, NC4HW4), g, r.mode == 1 ? NEAREST : BILINEAR, pad, r.align != 0), NCHW);
    std::ofstream o(outPath, std::ios::binary);
    for (int i = 0; i < r.count; ++i) {
        const float* set = data + (size_t)i * (xn + gn);
        memcpy(x->writeMap<float>(), set, xn * 4);
        memcpy(g->writeMap<float>(), set + xn, gn * 4);
        auto info = y->getInfo();
        const float* py = y->readMap<float>();
        if (!info || (int)info->dim.size() != r.rank || !py) { fprintf(stderr, "refdump_grid_sample: compute failed\n"); return 2; }
        if (i == 0) {
            o.write((const char*)&r.rank, 4);
            for (int d : info->dim) o.write((const char*)&d, 4);
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
// seeded He-like weights of a k x k conv, gain times the usual scale
struct ConvW {
    std::vector<float> w, b;
    int ic, oc, k;
};
static ConvW convW(std::mt19937& rng, int ic, int oc, int k, float gain = 1.41f) {
    const int fan = ic * k * k;
    return {seeded(rng, (size_t)oc * fan, gain * std::sqrt(3.f / fan)), seeded(rng, oc, 0.1f), ic, oc, k};
}
static VARP conv(const ConvW& c, VARP x, int stride, bool relu) {
    const int pad = (c.k - 1) / 2;
    return _Conv(std::vector<float>(c.w), std::vector<float>(c.b), x, {c.ic, c.oc}, {c.k, c.k}, CAFFE, {stride, stride}, {1, 1}, 1,
                 {pad, pad}, relu, false);
}
static void save(VARP h, const char* out) {
    h->setName("output");
    Variable::save({h}, out);
}

// A two-frame flow-warp net (PWC-Net / RAFT-style warping, in small) on one 6 x 64 x 64 input (frame 1's and frame 2's RGB
// stacked on the channels): a shared stride-4 conv encoder for both frames, a conv flow head [N, 2, 16, 16] in normalised grid
// units, permuted to [N, 16, 16, 2] by a Raster and added to a constant identity base grid (broadcast over the batch); a bilinear /
// zeros GridSample of frame 2's features at that grid, concatenated with frame 1's features, a conv refinement, and a x4 bilinear
// Interp of the refined flow to the input size.
static int cmdFlow(const char* out, int seed) {
    std::mt19937 rng(seed);
    const int H = 64, h = 16;
    VARP x = _Input({1, 6, H, H}, NCHW, halide_type_of<float>());
    x->setName("input");
    auto frames = _Split(x, {3, 3}, 1);
    ConvW e1 = convW(rng, 3, 16, 3), e2 = convW(rng, 16, 32, 3);
    auto enc = [&](VARP f) { return conv(e2, conv(e1, f, 2, true), 2, true); };   // 16 x 16, shared weights
    VARP f1 = enc(frames[0]), f2 = enc(frames[1]);
    VARP fh = conv(convW(rng, 64, 32, 3), _Concat({f1, f2}, 1), 1, true);
    VARP flow = conv(convW(rng, 32, 2, 3, 0.1f), fh, 1, false);                     // [N, 2, 16, 16], about +-0.1
    std::vector<float> base((size_t)h * h * 2);
    for (int i = 0; i < h; ++i)
        for (int j = 0; j < h; ++j) {
            base[(i * h + j) * 2 + 0] = -1.f + (2.f * j + 1.f) / h;   // x: pixel centres, alignCorners false
            base[(i * h + j) * 2 + 1] = -1.f + (2.f * i + 1.f) / h;
        }
    VARP grid = _Transpose(_Convert(flow, NCHW), {0, 2, 3, 1}) + _Const(base.data(), {1, h, h, 2}, NCHW, halide_type_of<float>());
    // the feature map in NC4HW4, as the model converter feeds a GridSample (AddTensorFormatConverter: NC4HW4_SINGLE)
    VARP warped = _GridSample(_Convert(f2, NC4HW4), grid, BILINEAR, GRID_SAMPLE_PADDING_ZEROS, false);
    VARP r = conv(convW(rng, 64, 32, 3), _Concat({f1, warped}, 1), 1, true);
    r = conv(convW(rng, 32, 2, 3, 0.1f), r, 1, false);
    r = _Interp({r}, 0.f, 0.f, H, H, 2, false);                                       // x4 to the input size
    save(_Convert(r, NCHW), out);
    return 0;
}

// An image-adaptive 3D-LUT enhancer (Zeng et al. 2020, in small) on a 3 x 64 x 64 image: a small CNN on a 4x average-pooled copy
// gives, through a MatMul, the weights of 3 basis LUTs; a MatMul with the constant basis [3, 3 * 33^3] (an identity LUT and two
// seeded ones) gives the image's LUT [N, 3, 33, 33, 33].  The image, rescaled from [0, 1] to [-1, 1] and permuted to
// [N, 1, 64, 64, 3] (R, G, B = x, y, z), is the grid of a trilinear / border GridSample with alignCorners; the result, reshaped
// back to the image, is added to it.
static int cmdLut(const char* out, int seed) {
    std::mt19937 rng(seed);
    const int H = 64, L = 33, L3 = L * L * L;
    VARP x = _Input({1, 3, H, H}, NCHW, halide_type_of<float>());
    x->setName("input");
    VARP h = _AvePool(x, {4, 4}, {4, 4}, VALID);                                        // 16 x 16
    h = conv(convW(rng, 3, 16, 3), h, 2, true);                                         // 8 x 8
    h = conv(convW(rng, 16, 32, 3), h, 2, true);                                        // 4 x 4
    h = _AvePool(h, {4, 4}, {1, 1}, VALID);                                             // [N, 32, 1, 1]
    VARP feat = _Reshape(_Convert(h, NCHW), {-1, 32});
    auto w1 = seeded(rng, 32 * 3, 0.2f), b1 = seeded(rng, 3, 0.1f);
    b1[0] += 1.f;                                                                       // mostly the identity LUT
    VARP wts = _MatMul(feat, _Const(w1.data(), {32, 3}, NCHW, halide_type_of<float>())) +
               _Const(b1.data(), {1, 3}, NCHW, halide_type_of<float>());
    std::vector<float> basis((size_t)3 * 3 * L3);
    auto more = seeded(rng, (size_t)2 * 3 * L3, 0.05f);
    for (int c = 0; c < 3; ++c)
        for (int d = 0; d < L; ++d)
            for (int i = 0; i < L; ++i)
                for (int j = 0; j < L; ++j) {
                    const int v = c == 0 ? j : (c == 1 ? i : d);
                    basis[(size_t)c * L3 + ((size_t)d * L + i) * L + j] = (float)v / (L - 1);
                }
    std::copy(more.begin(), more.end(), basis.begin() + 3 * L3);
    VARP lut = _MatMul(wts, _Const(basis.data(), {3, 3 * L3}, NCHW, halide_type_of<float>()));
    lut = _Reshape(lut, {-1, 3, L, L, L});
    VARP grid = _Transpose(_Convert(x, NCHW), {0, 2, 3, 1}) * _Scalar<float>(2.f) - _Scalar<float>(1.f);
    grid = _Reshape(grid, {-1, 1, H, H, 3});
    VARP y = _GridSample(_Convert(lut, NC4HW4), grid, BILINEAR, GRID_SAMPLE_PADDING_BORDER, true);   // [N, 3, 1, 64, 64]
    y = _Reshape(_Convert(y, NCHW), {-1, 3, H, H}) + x;
    save(_Convert(y, NCHW), out);
    return 0;
}

int main(int argc, char** argv) {
    if (argc >= 4 && std::string(argv[1]) == "op") return cmdOp(argv[2], argv[3]);
    if (argc >= 4 && std::string(argv[1]) == "flow") return cmdFlow(argv[2], atoi(argv[3]));
    if (argc >= 4 && std::string(argv[1]) == "lut") return cmdLut(argv[2], atoi(argv[3]));
    fprintf(stderr, "usage: refdump_grid_sample op <request> <out> | flow <out.mnn> <seed> | lut <out.mnn> <seed>\n");
    return 1;
}
