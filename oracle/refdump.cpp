// refdump -- drives the UNMODIFIED reference (oracle/_ref/libMNN.so, MNN_FORWARD_CPU) and dumps
// tensors so that tests can pin oracle/mnn_oracle.c and the CUDA path against the real thing.
//
// TEST INFRASTRUCTURE ONLY (see oracle/mnn_oracle.c header).  Built by oracle/build_ref.py in
// this container (needs the reference headers); the GPU box only runs the prebuilt binary.
// Uses nothing but the reference's public / exported API:
//   Express op builders  include/MNN/expr/NeuralNetWorkOp.hpp:137-157 (the same calls
//                        test/op/ConvInt8Test.cpp:225-243 makes)
//   Interpreter/Session  include/MNN/Interpreter.hpp (createSession, runSessionWithCallBackInfo)
//   Revert               tools/cpp/revertMNNModel.cpp:143-231 (random-weight int8 PTQ of benchmark graphs)
//   ConvolutionCommon::load  source/core/ConvolutionCommon.hpp:15 (IDST weight decode, SURVEY a1)
#include <algorithm>
#include <MNN/Interpreter.hpp>
#include <MNN/Tensor.hpp>
#include <MNN/AutoTime.hpp>
#include <MNN/expr/Expr.hpp>
#include <MNN/expr/ExprCreator.hpp>
#include <MNN/expr/Executor.hpp>
#include <MNN/expr/ExecutorScope.hpp>
#include <MNN/expr/Module.hpp>
#include "MNN_generated.h"
#include "core/TensorUtils.hpp"
#include "core/ConvolutionCommon.hpp"
#include "core/IDSTEncoder.hpp"
#include "core/WinogradInt8Attr.hpp"
#include "revertMNNModel.hpp"
#include <cstdio>
#include <cstring>
#include <fstream>
#include <random>
#include <string>
#include <vector>
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <dlfcn.h>

using namespace MNN;
using namespace MNN::Express;

static std::vector<char> readFile(const char* p) {
    std::ifstream f(p, std::ios::binary);
    return std::vector<char>((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
}
static void writeFile(const std::string& p, const void* d, size_t n) {
    std::ofstream o(p, std::ios::binary);
    o.write((const char*)d, n);
}

// REFDUMP_PLUGIN=<libmnn_b200_plugin.so>: load the plugin (its static initialiser registers an MNN_FORWARD_CUDA
// RuntimeCreator through MNNInsertExtraRuntimeCreator) and schedule the session on it instead of MNN_FORWARD_CPU.
static void* g_plugin = nullptr;
static MNNForwardType forwardType() {
    const char* p = getenv("REFDUMP_PLUGIN");
    if (!p || !*p) return MNN_FORWARD_CPU;
    if (!g_plugin) {
        g_plugin = dlopen(p, RTLD_NOW | RTLD_GLOBAL);
        if (!g_plugin) { fprintf(stderr, "refdump: dlopen(%s): %s\n", p, dlerror()); exit(3); }
    }
    return MNN_FORWARD_CUDA;
}
static void pluginStats() {
    if (!g_plugin) return;
    typedef void (*Fn)(int*, int*);
    Fn fn = (Fn)dlsym(g_plugin, "mnnb200_plugin_stats");
    int c = 0, d = 0;
    if (fn) fn(&c, &d);
    printf("{\"plugin_created\": %d, \"plugin_declined\": %d}\n", c, d);
}

struct ConvReq {
    int32_t mode;  // 0 legacy (int32 bias + fused scale), 1 modern (float bias + weight scale + scaleIn/Out)
    int32_t n, ic, ih, iw, oc, kh, kw, sh, sw, ph, pw, dh, dw, group, relu, zin, zout, minv, maxv;
    float scaleIn, scaleOut;
};


// Modern wire form (what FullQuantAndCoding / Revert emit, tools/cpp/revertMNNModel.cpp:79-123): op stays
// OpType_Convolution(/Depthwise) with IDST-coded int8 weights + per-channel alpha + float bias, and the
// activation quantisation lives on the TENSORS (Net.extraTensorDescribe[].quantInfo).  The CPU executor reads
// scaleX from the tensors' quant info (compute/ConvInt8TiledExecutor.cpp:1967-1976), so this form can only be
// exercised through a real model + Pipeline (quant propagation, source/core/Pipeline.cpp:241-400).  We
// assemble a 2-op net {Input, Convolution}, feed x as float (q - z_in)*s_in and read y back dequantised.
static int convModern(const ConvReq& r, const std::vector<int8_t>& x, const std::vector<int8_t>& w,
                      const std::vector<float>& biasF, const std::vector<float>& scale, const char* outPath) {
    std::unique_ptr<NetT> net(new NetT);
    net->tensorName = {"x", "y"};
    net->outputName = {"y"};
    net->sourceType = NetSource_CAFFE;
    {
        std::unique_ptr<OpT> in(new OpT);
        in->type = OpType_Input; in->name = "x"; in->outputIndexes = {0};
        in->main.type = OpParameter_Input; in->main.value = new InputT;
        auto ip = in->main.AsInput();
        ip->dims = {r.n, r.ic, r.ih, r.iw}; ip->dtype = DataType_DT_FLOAT; ip->dformat = MNN_DATA_FORMAT_NC4HW4;
        net->oplists.emplace_back(std::move(in));
    }
    {
        std::unique_ptr<OpT> convOp(new OpT);
        bool dw = (r.ic == r.oc && r.ic == r.group && r.group > 1);
        convOp->type = dw ? OpType_ConvolutionDepthwise : OpType_Convolution;
        convOp->name = "y"; convOp->inputIndexes = {0}; convOp->outputIndexes = {1};
        convOp->main.type = OpParameter_Convolution2D;
        convOp->main.value = new Convolution2DT;
        auto conv2D = convOp->main.AsConvolution2D();
        conv2D->common.reset(new Convolution2DCommonT);
        auto cm = conv2D->common.get();
        cm->padMode = PadMode_CAFFE; cm->padX = r.pw; cm->padY = r.ph; cm->strideX = r.sw; cm->strideY = r.sh;
        cm->group = r.group; cm->outputCount = r.oc; cm->inputCount = r.ic; cm->dilateX = r.dw; cm->dilateY = r.dh;
        cm->kernelX = r.kw; cm->kernelY = r.kh; cm->relu = r.relu != 0;
        int ks = (r.ic / r.group) * r.kh * r.kw;
        conv2D->quanParameter = IDSTEncoder::encode(nullptr, scale, ks, r.oc, false, w.data(), -128);
        conv2D->quanParameter->scaleIn = r.scaleIn;
        conv2D->quanParameter->scaleOut = r.scaleOut;
        conv2D->bias = biasF;
        conv2D->symmetricQuan.reset(new QuantizedFloatParamT);
        conv2D->symmetricQuan->nbits = 8;
        if (getenv("REFDUMP_WINO_UNIT")) {
            // attach a winogradAttr (core/WinogradInt8Attr.hpp:45-63 layout) => CPUConvInt8Creator picks ConvInt8Winograd for the
            // modern wire form too (CPUBackend.cpp:658-667, CPUConvolution.cpp:336-339).  ConvInt8Winograd reads the output scale /
            // zero point from the OP (mResource), so they are set consistently with the tensor quant info.
            const int unit = atoi(getenv("REFDUMP_WINO_UNIT"));
            const float inS = getenv("REFDUMP_WINO_INSCALE") ? (float)atof(getenv("REFDUMP_WINO_INSCALE")) : 1.0f;
            const float wS = getenv("REFDUMP_WINO_WSCALE") ? (float)atof(getenv("REFDUMP_WINO_WSCALE")) : 1.0f;
            const int a2 = (unit + r.kh - 1) * (unit + r.kw - 1);
            std::vector<int32_t> body = {0, 0, r.kh, r.kw, unit, unit};
            auto pushf = [&](float v) { int32_t b; memcpy(&b, &v, 4); body.push_back(b); };
            for (int i = 0; i < a2; ++i) pushf(inS);
            for (int i = 0; i < a2; ++i) body.push_back(0);
            for (int i = 0; i < a2 * r.oc; ++i) pushf(wS);
            std::vector<int32_t> blob = {0, 1, (int32_t)body.size()};
            blob.insert(blob.end(), body.begin(), body.end());
            conv2D->symmetricQuan->winogradAttr = blob;
            conv2D->symmetricQuan->zeroPoint = (int8_t)r.zin;
            conv2D->symmetricQuan->outputZeroPoint = (int8_t)r.zout;
            conv2D->symmetricQuan->clampMin = (int8_t)r.minv;
            conv2D->symmetricQuan->clampMax = (int8_t)r.maxv;
        }
        net->oplists.emplace_back(std::move(convOp));
    }
    float qs[2] = {r.scaleIn, r.scaleOut};
    int qz[2] = {r.zin, r.zout};
    for (int i = 0; i < 2; ++i) {
        std::unique_ptr<TensorDescribeT> d(new TensorDescribeT);
        d->index = i;
        d->quantInfo.reset(new TensorQuantInfoT);
        d->quantInfo->scale = qs[i]; d->quantInfo->zero = (float)qz[i];
        d->quantInfo->min = i == 0 ? -128.f : (float)r.minv; d->quantInfo->max = i == 0 ? 127.f : (float)r.maxv;
        d->quantInfo->type = DataType_DT_INT8;
        net->extraTensorDescribe.emplace_back(std::move(d));
    }
    flatbuffers::FlatBufferBuilder fb(1024);
    fb.Finish(Net::Pack(fb, net.get()));
    if (getenv("REFDUMP_SAVE_MODEL")) writeFile(getenv("REFDUMP_SAVE_MODEL"), fb.GetBufferPointer(), fb.GetSize());
    std::shared_ptr<Interpreter> itp(Interpreter::createFromBuffer(fb.GetBufferPointer(), fb.GetSize()), Interpreter::destroy);
    ScheduleConfig c; c.type = MNN_FORWARD_CPU; c.numThread = 1;
    BackendConfig bc; bc.precision = BackendConfig::Precision_High; c.backendConfig = &bc;
    auto s = itp->createSession(c);
    auto input = itp->getSessionInput(s, nullptr);
    {
        Tensor host(input, Tensor::CAFFE);
        auto p = host.host<float>();
        for (size_t i = 0; i < x.size(); ++i) p[i] = ((float)x[i] - (float)r.zin) * r.scaleIn;
        input->copyFromHostTensor(&host);
    }
    itp->runSession(s);
    auto output = itp->getSessionOutput(s, nullptr);
    Tensor hostOut(output, Tensor::CAFFE);
    output->copyToHostTensor(&hostOut);
    int32_t hdr[4] = {hostOut.length(0), hostOut.length(1), hostOut.length(2), hostOut.length(3)};
    std::vector<int8_t> q(hostOut.elementSize());
    auto po = hostOut.host<float>();
    for (size_t i = 0; i < q.size(); ++i) q[i] = (int8_t)std::lrintf(po[i] / r.scaleOut + (float)r.zout);
    std::ofstream o(outPath, std::ios::binary);
    o.write((const char*)hdr, sizeof(hdr));
    o.write((const char*)q.data(), q.size());
    return 0;
}

// conv <req.bin> <out.bin>: one ConvInt8 / DepthwiseConvInt8 op on the CPU backend.
static int cmdConv(const char* reqPath, const char* outPath) {
    auto buf = readFile(reqPath);
    ConvReq r;
    memcpy(&r, buf.data(), sizeof(r));
    const char* p = buf.data() + sizeof(r);
    size_t xs = (size_t)r.n * r.ic * r.ih * r.iw, ws = (size_t)r.oc * (r.ic / r.group) * r.kh * r.kw;
    std::vector<int8_t> x(p, p + xs); p += xs;
    std::vector<int8_t> w(p, p + ws); p += ws;
    std::vector<float> scale(r.oc);
    std::vector<int> biasI(r.oc);
    std::vector<float> biasF(r.oc);
    if (r.mode == 0) { memcpy(biasI.data(), p, 4 * r.oc); } else { memcpy(biasF.data(), p, 4 * r.oc); }
    p += 4 * r.oc;
    memcpy(scale.data(), p, 4 * r.oc);

    VARP xin = _Input({r.n, r.ic, r.ih, r.iw}, NCHW, halide_type_of<int8_t>());
    memcpy(xin->writeMap<int8_t>(), x.data(), xs);
    auto xC4 = _Convert(xin, NC4HW4);
    // same entry sequence as test/op/ConvInt8Test.cpp:225-227 (hides the x86 uint8 storage)
    xC4 = _FloatToInt8(_Cast<float>(xC4), _Scalar<float>(1.0f), -128, 127);
    VARP y;
    INTS channel = {r.ic, r.oc}, kernel = {r.kw, r.kh}, stride = {r.sw, r.sh}, dilate = {r.dw, r.dh}, pads = {r.pw, r.ph};
    if (r.mode == 0) {
        y = _Conv(std::move(w), std::move(biasI), std::move(scale), xC4, channel, kernel, CAFFE, stride, dilate,
                  r.group, pads, r.relu != 0, (int8_t)r.zin, (int8_t)r.zout, (int8_t)r.minv, (int8_t)r.maxv, false);
    } else {
        return convModern(r, x, w, biasF, scale, outPath);
    }
    y = _Int8ToFloat(y, _Scalar<float>(1.0f));
    y = _Cast<int8_t>(y);
    y = _Convert(y, NCHW);
    auto info = y->getInfo();
    auto yp = y->readMap<int8_t>();
    if (!info || !yp) { fprintf(stderr, "refdump conv: run failed\n"); return 2; }
    int32_t hdr[4] = {info->dim[0], info->dim[1], info->dim[2], info->dim[3]};
    std::ofstream o(outPath, std::ios::binary);
    o.write((const char*)hdr, sizeof(hdr));
    o.write((const char*)yp, info->size);
    return 0;
}

// pad = padY (rows), padW = padX (columns)
struct WinoReq { int32_t n, ic, ih, iw, oc, k, pad, unit, relu, zin, zout, minv, maxv; float scaleIn, scaleOut; int32_t padW; };
// wino <req.bin> <out.bin>: OpType_ConvInt8 carrying a winogradAttr => ConvInt8Winograd on the CPU backend
// (source/backend/cpu/CPUConvolution.cpp:336-339).  Op built exactly as test/op/ConvInt8Test.cpp:585-610 does
// (_Conv float-bias overload + WinogradInt8Attr::turnToWinogradConv).  Must be linked against the AVX2 build
// (libMNN_avx2.so): the AVX512 build of this op is wrong upstream (SURVEY F8).
static int cmdWino(const char* reqPath, const char* outPath) {
    auto buf = readFile(reqPath);
    WinoReq r;
    memcpy(&r, buf.data(), sizeof(r));
    const char* p = buf.data() + sizeof(r);
    int alpha = r.unit + r.k - 1, alpha2 = alpha * alpha;
    size_t xs = (size_t)r.n * r.ic * r.ih * r.iw, ws = (size_t)r.oc * r.ic * r.k * r.k;
    std::vector<int8_t> x(p, p + xs); p += xs;
    std::vector<int8_t> w(p, p + ws); p += ws;
    std::vector<float> bias(r.oc), wscale(r.oc), inS(alpha2), wS((size_t)alpha2 * r.oc);
    std::vector<int> inZ(alpha2);
    memcpy(bias.data(), p, 4 * r.oc); p += 4 * r.oc;
    memcpy(wscale.data(), p, 4 * r.oc); p += 4 * r.oc;
    memcpy(inS.data(), p, 4 * alpha2); p += 4 * alpha2;
    memcpy(inZ.data(), p, 4 * alpha2); p += 4 * alpha2;
    memcpy(wS.data(), p, 4 * (size_t)alpha2 * r.oc);

    VARP xin = _Input({r.n, r.ic, r.ih, r.iw}, NCHW, halide_type_of<int8_t>());
    memcpy(xin->writeMap<int8_t>(), x.data(), xs);
    auto xC4 = _Convert(xin, NC4HW4);
    xC4 = _FloatToInt8(_Cast<float>(xC4), _Scalar<float>(1.0f), -128, 127);
    INTS channel = {r.ic, r.oc}, kernel = {r.k, r.k}, pads = {r.padW, r.pad};   // {padX, padY}, as convModern
    WinogradInt8Attr attrs;
    attrs.add(0, 0, r.k, r.k, r.unit, r.unit, inS, wS, inZ);
    auto y = _Conv(std::move(w), std::move(bias), std::move(wscale), xC4, channel, kernel, CAFFE, {1, 1}, {1, 1}, 1, pads,
                   r.relu != 0, r.scaleIn, r.scaleOut, (int8_t)r.zin, (int8_t)r.zout, (int8_t)r.minv, (int8_t)r.maxv, 127, false);
    y = attrs.turnToWinogradConv(y);
    y = _Int8ToFloat(y, _Scalar<float>(1.0f));
    y = _Cast<int8_t>(y);
    y = _Convert(y, NCHW);
    auto info = y->getInfo();
    auto yp = y->readMap<int8_t>();
    if (!info || !yp) { fprintf(stderr, "refdump wino: run failed\n"); return 2; }
    int32_t hdr[4] = {info->dim[0], info->dim[1], info->dim[2], info->dim[3]};
    std::ofstream o(outPath, std::ios::binary);
    o.write((const char*)hdr, sizeof(hdr));
    o.write((const char*)yp, info->size);
    return 0;
}

struct MatReq { int32_t batch, e, l, h, ta, tb, hasBias, pad; };
// matmul <req.bin> <out.bin>: float MatMul / BatchMatMul on the CPU backend through the Express builders the reference's
// own tests use (test/op/MatMulTest.cpp, BatchMatMulTest.cpp: _MatMul(a, b, tranposeA, tranposeB), _BatchMatMul(a, b, adjX, adjY)).
static int cmdMatMul(const char* reqPath, const char* outPath) {
    auto buf = readFile(reqPath);
    BackendConfig bcm; bcm.precision = BackendConfig::Precision_High;
    auto exem = Executor::newExecutor(forwardType(), bcm, 1);
    ExecutorScope scopem(exem);
    MatReq r; memcpy(&r, buf.data(), sizeof(r));
    const char* p = buf.data() + sizeof(r);
    size_t as = (size_t)r.batch * r.e * r.l, bs = (size_t)r.batch * r.l * r.h;
    std::vector<int> sa = r.ta ? std::vector<int>{r.batch, r.l, r.e} : std::vector<int>{r.batch, r.e, r.l};
    std::vector<int> sb = r.tb ? std::vector<int>{r.batch, r.h, r.l} : std::vector<int>{r.batch, r.l, r.h};
    VARP y;
    if (r.batch == 1) {
        sa.erase(sa.begin()); sb.erase(sb.begin());
        VARP a = _Input(sa, NCHW, halide_type_of<float>()), b = _Input(sb, NCHW, halide_type_of<float>());
        memcpy(a->writeMap<float>(), p, as * 4); memcpy(b->writeMap<float>(), p + as * 4, bs * 4);
        y = _MatMul(a, b, r.ta != 0, r.tb != 0);
        auto yp = y->readMap<float>();
        if (!yp) return 2;
        writeFile(outPath, yp, (size_t)r.e * r.h * 4);
        return 0;
    }
    VARP a = _Input(sa, NCHW, halide_type_of<float>()), b = _Input(sb, NCHW, halide_type_of<float>());
    memcpy(a->writeMap<float>(), p, as * 4); memcpy(b->writeMap<float>(), p + as * 4, bs * 4);
    y = _BatchMatMul(a, b, r.ta != 0, r.tb != 0);
    auto yp = y->readMap<float>();
    if (!yp) return 2;
    writeFile(outPath, yp, (size_t)r.batch * r.e * r.h * 4);
    return 0;
}

struct PoolReq { int32_t n, c, ih, iw, kh, kw, sh, sw, ph, pw, isAvg, zero; float scale; };
// pool <req.bin> <out.bin>: {Input, Pooling} with IDENTICAL quant info on both tensors, so that the reference keeps the op
// in int8 (CPUBackend.cpp:930-941 -> CPUPoolInt8).  x is fed as float (q - z)*s, y read back and re-quantised exactly.
static int cmdPool(const char* reqPath, const char* outPath) {
    auto buf = readFile(reqPath);
    PoolReq r; memcpy(&r, buf.data(), sizeof(r));
    const int8_t* x = (const int8_t*)(buf.data() + sizeof(r));
    std::unique_ptr<NetT> net(new NetT);
    net->tensorName = {"x", "y"}; net->outputName = {"y"}; net->sourceType = NetSource_CAFFE;
    {
        std::unique_ptr<OpT> in(new OpT);
        in->type = OpType_Input; in->name = "x"; in->outputIndexes = {0};
        in->main.type = OpParameter_Input; in->main.value = new InputT;
        auto ip = in->main.AsInput();
        ip->dims = {r.n, r.c, r.ih, r.iw}; ip->dtype = DataType_DT_FLOAT; ip->dformat = MNN_DATA_FORMAT_NC4HW4;
        net->oplists.emplace_back(std::move(in));
    }
    {
        std::unique_ptr<OpT> op(new OpT);
        op->type = OpType_Pooling; op->name = "y"; op->inputIndexes = {0}; op->outputIndexes = {1};
        op->main.type = OpParameter_Pool; op->main.value = new PoolT;
        auto p = op->main.AsPool();
        p->kernelX = r.kw; p->kernelY = r.kh; p->strideX = r.sw; p->strideY = r.sh; p->padX = r.pw; p->padY = r.ph;
        p->type = r.isAvg ? PoolType_AVEPOOL : PoolType_MAXPOOL; p->padType = PoolPadType_CAFFE; p->isGlobal = false;
        p->ceilModel = false;
        net->oplists.emplace_back(std::move(op));
    }
    for (int i = 0; i < 2; ++i) {
        std::unique_ptr<TensorDescribeT> d(new TensorDescribeT);
        d->index = i; d->quantInfo.reset(new TensorQuantInfoT);
        d->quantInfo->scale = r.scale; d->quantInfo->zero = (float)r.zero; d->quantInfo->min = -128.f; d->quantInfo->max = 127.f;
        d->quantInfo->type = DataType_DT_INT8;
        net->extraTensorDescribe.emplace_back(std::move(d));
    }
    flatbuffers::FlatBufferBuilder fb(1024);
    fb.Finish(Net::Pack(fb, net.get()));
    std::shared_ptr<Interpreter> itp(Interpreter::createFromBuffer(fb.GetBufferPointer(), fb.GetSize()), Interpreter::destroy);
    ScheduleConfig c; c.type = MNN_FORWARD_CPU; c.numThread = 1;
    BackendConfig bc; bc.precision = BackendConfig::Precision_High; c.backendConfig = &bc;
    auto s = itp->createSession(c);
    auto input = itp->getSessionInput(s, nullptr);
    {
        Tensor host(input, Tensor::CAFFE);
        auto p = host.host<float>();
        for (int i = 0; i < host.elementSize(); ++i) p[i] = ((float)x[i] - (float)r.zero) * r.scale;
        input->copyFromHostTensor(&host);
    }
    itp->runSession(s);
    auto output = itp->getSessionOutput(s, nullptr);
    Tensor hostOut(output, Tensor::CAFFE);
    output->copyToHostTensor(&hostOut);
    int32_t hdr[4] = {hostOut.length(0), hostOut.length(1), hostOut.length(2), hostOut.length(3)};
    std::vector<int8_t> q(hostOut.elementSize());
    auto po = hostOut.host<float>();
    for (size_t i = 0; i < q.size(); ++i) q[i] = (int8_t)std::lrintf(po[i] / r.scale + (float)r.zero);
    std::ofstream o(outPath, std::ios::binary);
    o.write((const char*)hdr, sizeof(hdr));
    o.write((const char*)q.data(), q.size());
    return 0;
}

struct PoolFReq { int32_t n, c, ih, iw, kh, kw, sh, sw, ph, pw, isAvg, padType, countType, ceilModel, isGlobal, npads; };
// poolf <req.bin> <out.bin>: {Input, Pooling} on float tensors (no quant info: CPUPool with the core's MNNPoolingAvg /
// MNNPoolingMax).  npads = -1: no Pool.pads vector, else npads int32 values follow the header, then x [n][c][ih][iw] fp32.
// Writes int32 dims[4] + y fp32 NCHW.
static int cmdPoolF(const char* reqPath, const char* outPath) {
    auto buf = readFile(reqPath);
    PoolFReq r; memcpy(&r, buf.data(), sizeof(r));
    const char* p = buf.data() + sizeof(r);
    std::vector<int32_t> pads(r.npads > 0 ? r.npads : 0);
    if (!pads.empty()) { memcpy(pads.data(), p, pads.size() * 4); p += pads.size() * 4; }
    const float* x = (const float*)p;
    std::unique_ptr<NetT> net(new NetT);
    net->tensorName = {"x", "y"}; net->outputName = {"y"}; net->sourceType = NetSource_CAFFE;
    {
        std::unique_ptr<OpT> in(new OpT);
        in->type = OpType_Input; in->name = "x"; in->outputIndexes = {0};
        in->main.type = OpParameter_Input; in->main.value = new InputT;
        auto ip = in->main.AsInput();
        ip->dims = {r.n, r.c, r.ih, r.iw}; ip->dtype = DataType_DT_FLOAT; ip->dformat = MNN_DATA_FORMAT_NC4HW4;
        net->oplists.emplace_back(std::move(in));
    }
    {
        std::unique_ptr<OpT> op(new OpT);
        op->type = OpType_Pooling; op->name = "y"; op->inputIndexes = {0}; op->outputIndexes = {1};
        op->main.type = OpParameter_Pool; op->main.value = new PoolT;
        auto pl = op->main.AsPool();
        pl->kernelX = r.kw; pl->kernelY = r.kh; pl->strideX = r.sw; pl->strideY = r.sh; pl->padX = r.pw; pl->padY = r.ph;
        pl->type = r.isAvg ? PoolType_AVEPOOL : PoolType_MAXPOOL; pl->padType = (PoolPadType)r.padType;
        pl->countType = (AvgPoolCountType)r.countType; pl->ceilModel = r.ceilModel != 0; pl->isGlobal = r.isGlobal != 0;
        if (r.npads >= 0) pl->pads = pads;
        net->oplists.emplace_back(std::move(op));
    }
    flatbuffers::FlatBufferBuilder fb(1024);
    fb.Finish(Net::Pack(fb, net.get()));
    std::shared_ptr<Interpreter> itp(Interpreter::createFromBuffer(fb.GetBufferPointer(), fb.GetSize()), Interpreter::destroy);
    ScheduleConfig c; c.type = MNN_FORWARD_CPU; c.numThread = 1;
    BackendConfig bc; bc.precision = BackendConfig::Precision_High; c.backendConfig = &bc;
    auto s = itp->createSession(c);
    if (!s) return 2;
    auto input = itp->getSessionInput(s, nullptr);
    {
        Tensor host(input, Tensor::CAFFE);
        memcpy(host.host<float>(), x, (size_t)host.elementSize() * 4);
        input->copyFromHostTensor(&host);
    }
    if (itp->runSession(s) != NO_ERROR) return 2;
    auto output = itp->getSessionOutput(s, nullptr);
    Tensor hostOut(output, Tensor::CAFFE);
    output->copyToHostTensor(&hostOut);
    int32_t hdr[4] = {hostOut.length(0), hostOut.length(1), hostOut.length(2), hostOut.length(3)};
    std::ofstream o(outPath, std::ios::binary);
    o.write((const char*)hdr, sizeof(hdr));
    o.write((const char*)hostOut.host<float>(), (size_t)hostOut.elementSize() * 4);
    return 0;
}

struct LinReq { int32_t tokens, ic, oc, asym, relu, relu6, hasBias, pad; };   // pad = number of K blocks of the weight scales (0 / 1: per channel)
// linear <req.bin> <out.bin>: weight-quantised Conv1x1 (what MNN-LLM lowers nn.Linear to,
// transformers/llm/export/utils/mnn_converter.py:767-787) run with Memory_Low => W8A8 dynamic quant.
// Op built exactly as test/CommonOpCreator.hpp:27-68 does (_HybridConv), with pre-quantised int8 weights.
static int cmdLinear(const char* reqPath, const char* outPath, int threads) {
    auto buf = readFile(reqPath);
    LinReq r; memcpy(&r, buf.data(), sizeof(r));
    const char* p = buf.data() + sizeof(r);
    std::vector<float> x((size_t)r.tokens * r.ic); memcpy(x.data(), p, x.size() * 4); p += x.size() * 4;
    std::vector<int8_t> wq((size_t)r.oc * r.ic); memcpy(wq.data(), p, wq.size()); p += wq.size();
    const int blocks = r.pad > 0 ? r.pad : 1;   // K-blocked weight scales: alpha holds oc * blocks entries ({min, scale} pairs when asymmetric)
    std::vector<float> alpha((size_t)r.oc * blocks * (r.asym ? 2 : 1)); memcpy(alpha.data(), p, alpha.size() * 4); p += alpha.size() * 4;
    std::vector<float> bias(r.oc, 0.f); if (r.hasBias) memcpy(bias.data(), p, 4 * r.oc);

    BackendConfig bc; bc.memory = BackendConfig::Memory_Low; bc.precision = BackendConfig::Precision_Normal;
    auto exe = Executor::newExecutor(forwardType(), bc, threads);
    ExecutorScope scope(exe);

    std::unique_ptr<OpT> convOp(new OpT);
    convOp->type = OpType_Convolution;
    convOp->main.type = OpParameter_Convolution2D;
    convOp->main.value = new Convolution2DT;
    auto conv2D = convOp->main.AsConvolution2D();
    conv2D->common.reset(new Convolution2DCommonT);
    conv2D->quanParameter = IDSTEncoder::encode(nullptr, alpha, r.ic, r.oc, r.asym != 0, wq.data(), -128, {8, false});
    conv2D->common->outputCount = r.oc; conv2D->common->inputCount = r.ic;
    conv2D->common->kernelX = 1; conv2D->common->kernelY = 1;
    conv2D->common->relu = r.relu != 0; conv2D->common->relu6 = r.relu6 != 0;
    conv2D->bias = bias;
    // activations [tokens, ic] -> NCHW [1, ic, tokens, 1] like the LLM export (Reshape -> ConvertTensor -> Conv1x1)
    VARP xin = _Input({1, r.ic, r.tokens, 1}, NCHW, halide_type_of<float>());
    auto xp = xin->writeMap<float>();
    for (int t = 0; t < r.tokens; ++t) for (int c = 0; c < r.ic; ++c) xp[(size_t)c * r.tokens + t] = x[(size_t)t * r.ic + c];
    auto xC4 = _Convert(xin, NC4HW4);
    auto y = Variable::create(Expr::create(convOp.get(), {xC4}));
    y = _Convert(y, NCHW);
    auto yp = y->readMap<float>();
    if (!yp) { fprintf(stderr, "refdump linear: run failed\n"); return 2; }
    if (getenv("REFDUMP_TIMING_ITERS")) {   // timed like test/speed/GemmSpeed.cpp / ConvInt8Test.cpp:618-629
        int iters = atoi(getenv("REFDUMP_TIMING_ITERS"));
        xC4.fix(VARP::INPUT);
        xC4->writeMap<float>(); y->readMap<float>();
        auto t0 = std::chrono::steady_clock::now();
        for (int i = 0; i < iters; ++i) { xC4->writeMap<float>(); y->readMap<float>(); }
        double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count() / iters;
        printf("{\"ms_per_iter\": %.4f, \"threads\": %d, \"tokens\": %d, \"ic\": %d, \"oc\": %d}\n", ms, threads, r.tokens, r.ic, r.oc);
        yp = y->readMap<float>();
    }
    std::vector<float> out((size_t)r.tokens * r.oc);
    for (int t = 0; t < r.tokens; ++t) for (int o = 0; o < r.oc; ++o) out[(size_t)t * r.oc + o] = yp[(size_t)o * r.tokens + t];
    writeFile(outPath, out.data(), out.size() * 4);
    pluginStats();
    return 0;
}

// revert <weightless.mnn> <out.mnn> <retune> <seed>
// retune=0: exactly what benchmark.out's testQuantizedModel=1 runs (Revert::initialize(0,1,false,true)),
//           serialised once because the tool seeds with time(NULL) (SURVEY F11).
// retune=1: same graph, but with seeded weights/biases and per-tensor scales / zero points chosen so
//           activations do NOT saturate -- the parity fixture (a saturated net hides epilogue errors).
static int cmdRevert(const char* in, const char* out, int retune, int seed) {
    Revert r(in);
    r.initialize(0, 1, false, true);
    if (!retune) { writeFile(out, r.getBuffer(), r.getBufferSize()); return 0; }
    std::unique_ptr<NetT> net(UnPackNet(r.getBuffer()));
    std::mt19937 rng(seed);
    std::uniform_real_distribution<float> uw(-1.f, 1.f);
    int nT = (int)net->extraTensorDescribe.size();
    for (int i = 0; i < nT; ++i) {
        auto& q = net->extraTensorDescribe[i]->quantInfo;
        if (!q) continue;
        int ti = net->extraTensorDescribe[i]->index;
        (void)ti;
        q->scale = 0.02f + 0.03f * (float)((i * 37) % 11) / 11.f;
        q->zero = (float)(((i * 13) % 9) - 4);
        q->min = -127; q->max = 127;
    }
    for (auto& op : net->oplists) {
        if (op->type != OpType_Convolution && op->type != OpType_ConvolutionDepthwise) continue;
        auto conv = op->main.AsConvolution2D();
        int oc = conv->common->outputCount;
        int ks = conv->common->kernelX * conv->common->kernelY * conv->common->inputCount / conv->common->group;
        if (op->type == OpType_ConvolutionDepthwise) ks = conv->common->kernelX * conv->common->kernelY;
        std::vector<float> wf((size_t)oc * ks), alpha(oc);
        std::vector<int8_t> wq((size_t)oc * ks);
        float mag = 1.2f / std::sqrt((float)ks);
        for (int o = 0; o < oc; ++o) {
            float amax = 1e-6f;
            for (int k = 0; k < ks; ++k) { wf[(size_t)o * ks + k] = uw(rng) * mag * (0.5f + (o % 5) * 0.25f); amax = std::max(amax, std::fabs(wf[(size_t)o * ks + k])); }
            alpha[o] = amax / 127.f;
            for (int k = 0; k < ks; ++k) wq[(size_t)o * ks + k] = (int8_t)std::max(-127.f, std::min(127.f, std::round(wf[(size_t)o * ks + k] / alpha[o])));
        }
        float sIn = conv->quanParameter->scaleIn, sOut = conv->quanParameter->scaleOut;
        conv->quanParameter = IDSTEncoder::encode(nullptr, alpha, ks, oc, false, wq.data(), -127);
        conv->quanParameter->scaleIn = sIn; conv->quanParameter->scaleOut = sOut;
        conv->bias.resize(oc);
        for (int o = 0; o < oc; ++o) conv->bias[o] = uw(rng) * 0.5f;
    }
    flatbuffers::FlatBufferBuilder b(1024);
    b.Finish(Net::Pack(b, net.get()));
    writeFile(out, b.GetBufferPointer(), b.GetSize());
    return 0;
}

static void fillInput(Tensor* input, int seed) {
    Tensor host(input, Tensor::CAFFE);
    std::mt19937 rng(seed);
    std::uniform_real_distribution<float> u(-1.f, 1.f);
    auto p = host.host<float>();
    for (int i = 0; i < host.elementSize(); ++i) p[i] = u(rng);
    input->copyFromHostTensor(&host);
}

// The model with its Input op's batch dimension rewritten, so that the session is built for `batch` directly and never resized
// a second time: CPUScaleInt8::onResize folds its float scale/bias into fixed point IN PLACE (CPUScaleInt8.cpp:60-90), a second
// resize re-reads the folded integers as floats and the op outputs nothing but the zero point from then on -- an upstream bug that
// has nothing to do with the arithmetic under test.
static std::vector<uint8_t> netWithBatch(const char* model, int batch) {
    auto buf = readFile(model);
    std::unique_ptr<NetT> net(UnPackNet(buf.data()));
    for (auto& op : net->oplists) {
        if (op->type != OpType_Input) continue;
        auto ip = op->main.AsInput();
        if (ip && !ip->dims.empty()) ip->dims[0] = batch;
    }
    flatbuffers::FlatBufferBuilder fb(1024);
    fb.Finish(Net::Pack(fb, net.get()));
    return std::vector<uint8_t>(fb.GetBufferPointer(), fb.GetBufferPointer() + fb.GetSize());
}
static std::shared_ptr<Interpreter> loadWithBatch(const char* model, int batch) {
    auto buf = netWithBatch(model, batch);
    return std::shared_ptr<Interpreter>(Interpreter::createFromBuffer(buf.data(), buf.size()), Interpreter::destroy);
}

// run <model.mnn> <batch> <seed> <outdir> <threads>: dump the input and every command's outputs
// (dequantised to float NCHW by the backend's own onCopyBuffer, the reference's comparison boundary, SURVEY F6).
static int cmdRun(const char* model, int batch, int seed, const std::string& dir, int threads) {
    std::shared_ptr<Interpreter> net = loadWithBatch(model, batch);
    ScheduleConfig c; c.type = forwardType(); c.numThread = threads; c.backupType = MNN_FORWARD_CPU;
    BackendConfig bc; bc.precision = BackendConfig::Precision_High; c.backendConfig = &bc;
    auto s = net->createSession(c);
    if (!s) { fprintf(stderr, "refdump run: createSession failed\n"); return 2; }
    auto input = net->getSessionInput(s, nullptr);
    auto shape = input->shape(); shape[0] = batch;
    net->resizeTensor(input, shape); net->resizeSession(s);
    fillInput(input, seed);
    { Tensor host(input, Tensor::CAFFE); input->copyToHostTensor(&host); writeFile(dir + "/input.f32", host.host<float>(), host.size()); }
    // REFDUMP_RUN_REPEATS=<n>: n plain runSession() calls first (a backend that captures/replays a graph goes eager -> capture ->
    // replay), the LAST one's output is written as output_plain.f32; the per-command dump below then runs with callbacks.
    if (const char* rp = getenv("REFDUMP_RUN_REPEATS")) {
        const int reps = atoi(rp);
        auto output = net->getSessionOutput(s, nullptr);
        Tensor host(output, Tensor::CAFFE);
        for (int i = 0; i < reps; ++i) {
            fillInput(input, seed);
            if (net->runSession(s) != NO_ERROR) { fprintf(stderr, "refdump run: plain runSession failed\n"); return 2; }
            output->copyToHostTensor(&host);
        }
        if (reps > 0) writeFile(dir + "/output_plain.f32", host.host<float>(), host.size());
        fillInput(input, seed);   // a session may reuse the input's memory for intermediates: every forward gets its input again
    }
    FILE* idx = fopen((dir + "/index.txt").c_str(), "w");
    int n = 0;
    const bool hashOnly = getenv("REFDUMP_HASH") && atoi(getenv("REFDUMP_HASH")) != 0;
    const int maxCommands = getenv("REFDUMP_MAX_COMMANDS") ? atoi(getenv("REFDUMP_MAX_COMMANDS")) : 0;
    TensorCallBackWithInfo before = [&](const std::vector<Tensor*>&, const OperatorInfo*) { return true; };
    TensorCallBackWithInfo after = [&](const std::vector<Tensor*>& ts, const OperatorInfo* info) {
        for (size_t i = 0; i < ts.size(); ++i) {
            auto t = ts[i];
            if (t->elementSize() <= 0 || t->getType().code != halide_type_float) continue;
            Tensor host(t, Tensor::CAFFE);
            t->copyToHostTensor(&host);
            auto des = TensorUtils::getDescribe(t);
            float qs = 0, qz = 0, qmin = 0, qmax = 0; int aq = des->applyQuant ? 1 : 0;
            if (des->quantAttr) { qs = des->quantAttr->scale; qz = des->quantAttr->zero; qmin = des->quantAttr->min; qmax = des->quantAttr->max; }
            char name[64]; snprintf(name, sizeof(name), "%04d_%zu.f32", n, i);
            if (hashOnly) {   // REFDUMP_HASH=1: full-size runs (batch 32) record a position-weighted 64-bit sum instead of GBs of floats
                const uint32_t* wv = (const uint32_t*)host.host<float>();
                const size_t cnt = (size_t)host.elementSize();
                uint64_t hsum = 0;
                for (size_t k = 0; k < cnt; ++k) hsum += (uint64_t)wv[k] * ((uint64_t)k * 0x9E3779B97F4A7C15ull + 1ull);
                snprintf(name, sizeof(name), "hash:%016llx", (unsigned long long)hsum);
            } else
            writeFile(dir + "/" + name, host.host<float>(), host.size());
            fprintf(idx, "%s|%s|%s|", name, info->name().c_str(), info->type().c_str());
            for (int d = 0; d < host.dimensions(); ++d) fprintf(idx, "%d%s", host.length(d), d + 1 < host.dimensions() ? "," : "");
            fprintf(idx, "|%.9g|%.9g|%g|%g|%d\n", qs, qz, qmin, qmax, aq);
        }
        ++n;
        return maxCommands <= 0 || n < maxCommands;      // REFDUMP_MAX_COMMANDS: stop the forward after that many commands
    };
    auto code = net->runSessionWithCallBackInfo(s, before, after, true);
    if (maxCommands > 0 && n >= maxCommands) code = NO_ERROR;
    fclose(idx);
    if (code != NO_ERROR) { fprintf(stderr, "refdump run: runSession -> %d\n", (int)code); return 2; }
    if (maxCommands <= 0) {   // the session output as the user reads it (copyToHostTensor through the backend's onCopyBuffer)
        auto output = net->getSessionOutput(s, nullptr);
        Tensor host(output, Tensor::CAFFE);
        output->copyToHostTensor(&host);
        writeFile(dir + "/output.f32", host.host<float>(), host.size());
    }
    pluginStats();
    return 0;
}

// clone <model.mnn> <batch> <outdir> [<tensor>]: the model as an Express Module (express/module: StaticModule over one Session) on
// the forward type, run once so that every execution is created, then copied with Module::clone, which goes StaticModule::clone ->
// Session::clone -> Execution::onClone for each cached execution (StaticModule.cpp:814-828, Session.cpp:612-625).  The original
// and the clone then run on the same seeded input (fillInput's values); their first outputs go to output.f32 and
// output_clone.f32, the original's first forward to output_first.f32.  A plugin's stats are printed after the first forward
// and at the end.  <tensor>: the module's output is that tensor instead of the model's outputs.
static int cmdClone(const char* model, int batch, const std::string& dir, const char* output) {
    const auto buf = netWithBatch(model, batch);   // outlives both modules
    ScheduleConfig c; c.type = forwardType(); c.numThread = 4; c.backupType = MNN_FORWARD_CPU;
    BackendConfig bc; bc.precision = BackendConfig::Precision_High; c.backendConfig = &bc;
    std::shared_ptr<Executor::RuntimeManager> rtm(Executor::RuntimeManager::createRuntimeManager(c));
    std::vector<std::string> outputs;
    if (output) outputs.push_back(output);
    std::shared_ptr<Module> net(Module::load({}, outputs, buf.data(), buf.size(), rtm));
    if (!net) { fprintf(stderr, "refdump clone: Module::load failed\n"); return 2; }
    const auto& in = net->getInfo()->inputs[0];
    VARP x = _Input(in.dim, NCHW, halide_type_of<float>());
    {
        std::mt19937 rng(3);
        std::uniform_real_distribution<float> u(-1.f, 1.f);
        auto p = x->writeMap<float>();
        const int n = x->getInfo()->size;
        for (int i = 0; i < n; ++i) p[i] = u(rng);
    }
    if (in.order == NC4HW4) x = _Convert(x, NC4HW4);
    x.fix(VARP::CONSTANT);
    auto forward = [&](Module* m, const char* name) {
        auto outs = m->onForward({x});
        if (outs.empty() || !outs[0]->getInfo()) return false;
        VARP y = outs[0];
        if (y->getInfo()->order == NC4HW4 && y->getInfo()->dim.size() > 1) y = _Convert(y, NCHW);
        auto p = y->readMap<float>();
        if (!p) return false;
        writeFile(dir + "/" + name, p, (size_t)y->getInfo()->size * 4);
        return true;
    };
    if (!forward(net.get(), "output_first.f32")) { fprintf(stderr, "refdump clone: first forward failed\n"); return 2; }
    pluginStats();   // the original's executions; the last line adds what the clone had to create instead of cloning
    std::shared_ptr<Module> copy(Module::clone(net.get()));
    if (!copy) { fprintf(stderr, "refdump clone: Module::clone failed\n"); return 2; }
    if (!forward(net.get(), "output.f32") || !forward(copy.get(), "output_clone.f32")) {
        fprintf(stderr, "refdump clone: forward failed\n");
        return 2;
    }
    pluginStats();
    return 0;
}

// bench <model.mnn> <batch> <threads> <warmup> <iters>: wall-clock like benchmark/benchmark.cpp:120-181
// (input copy + runSession + output copy per iteration).  Prints one JSON line.
static int cmdBench(const char* model, int batch, int threads, int warmup, int iters) {
    std::shared_ptr<Interpreter> net = loadWithBatch(model, batch);
    ScheduleConfig c; c.type = forwardType(); c.numThread = threads; c.backupType = MNN_FORWARD_CPU;
    BackendConfig bc; bc.precision = BackendConfig::Precision_High; c.backendConfig = &bc;
    auto s = net->createSession(c);
    if (!s) { fprintf(stderr, "refdump bench: createSession failed\n"); return 2; }
    auto input = net->getSessionInput(s, nullptr);
    auto shape = input->shape(); shape[0] = batch;
    net->resizeTensor(input, shape); net->resizeSession(s);
    Tensor hostIn(input, Tensor::CAFFE);
    { std::mt19937 rng(1000); std::uniform_real_distribution<float> u(-1.f, 1.f); auto p = hostIn.host<float>(); for (int i = 0; i < hostIn.elementSize(); ++i) p[i] = u(rng); }
    auto output = net->getSessionOutput(s, nullptr);
    Tensor hostOut(output, Tensor::CAFFE);
    for (int i = 0; i < warmup; ++i) { input->copyFromHostTensor(&hostIn); net->runSession(s); output->copyToHostTensor(&hostOut); }
    // REFDUMP_BENCH_WINDOWS=<n> (default 1): time n windows of <iters> iterations each and also report the median window
    int windows = 1;
    if (const char* w = getenv("REFDUMP_BENCH_WINDOWS")) windows = std::max(1, atoi(w));
    std::vector<double> win;
    double total = 0;
    for (int wdx = 0; wdx < windows; ++wdx) {
        auto t0 = std::chrono::steady_clock::now();
        for (int i = 0; i < iters; ++i) { input->copyFromHostTensor(&hostIn); net->runSession(s); output->copyToHostTensor(&hostOut); }
        auto t1 = std::chrono::steady_clock::now();
        double ms = std::chrono::duration<double, std::milli>(t1 - t0).count() / iters;
        win.push_back(ms); total += ms;
    }
    std::vector<double> sorted = win;
    std::sort(sorted.begin(), sorted.end());
    int created = -1, declined = -1;
    if (g_plugin) {
        typedef void (*Fn)(int*, int*);
        Fn fn = (Fn)dlsym(g_plugin, "mnnb200_plugin_stats");
        if (fn) fn(&created, &declined);
    }
    printf("{\"ms_per_iter\": %.6f, \"ms_median_window\": %.6f, \"ms_min_window\": %.6f, \"windows\": %d, \"batch\": %d, \"threads\": %d, \"iters\": %d, "
           "\"plugin_created\": %d, \"plugin_declined\": %d, \"h2d_bytes\": %zu, \"d2h_bytes\": %zu}\n",
           total / windows, sorted[sorted.size() / 2], sorted[0], windows, batch, threads, iters, created, declined,
           (size_t)hostIn.elementSize() * 4, (size_t)hostOut.elementSize() * 4);
    return 0;
}


// convbench <model.mnn> <shapes.txt> <batch> <threads> <warmup> <iters>
// Times the reference CPU backend on the DENSE CONV layers of a model, one 2-op net {Input, conv} per layer
// with the layer's own tensor quant info (so it takes the same static-int8 executor as inside the full net).
// shapes.txt: "<opIndex> <ih> <iw>" per line.  Input is fed as int8-representable floats once; the timed loop is
// runSession only (activations resident, like the GPU arm's device-timed number).  Prints one JSON line.
static int cmdConvBench(const char* model, const char* shapesPath, int batch, int threads, int warmup, int iters) {
    auto buf = readFile(model);
    std::ifstream sf(shapesPath);
    int opIndex, ih, iw;
    double totalMs = 0; int layers = 0;
    std::string per = "[";
    while (sf >> opIndex >> ih >> iw) {
        std::unique_ptr<NetT> src(UnPackNet(buf.data()));
        std::unique_ptr<NetT> net(new NetT);
        net->tensorName = {"x", "y"}; net->outputName = {"y"}; net->sourceType = NetSource_CAFFE;
        auto& sop = src->oplists[opIndex];
        int tin = sop->inputIndexes[0], tout = sop->outputIndexes[0];
        auto conv = sop->main.AsConvolution2D();
        {
            std::unique_ptr<OpT> in(new OpT);
            in->type = OpType_Input; in->name = "x"; in->outputIndexes = {0};
            in->main.type = OpParameter_Input; in->main.value = new InputT;
            auto ip = in->main.AsInput();
            ip->dims = {batch, conv->common->inputCount, ih, iw}; ip->dtype = DataType_DT_FLOAT; ip->dformat = MNN_DATA_FORMAT_NC4HW4;
            net->oplists.emplace_back(std::move(in));
        }
        for (auto& d : src->extraTensorDescribe) {
            if (!d->quantInfo) continue;
            if (d->index == tin || d->index == tout) {
                std::unique_ptr<TensorDescribeT> nd(new TensorDescribeT);
                nd->index = d->index == tin ? 0 : 1;
                nd->quantInfo.reset(new TensorQuantInfoT(*d->quantInfo));
                net->extraTensorDescribe.emplace_back(std::move(nd));
            }
        }
        sop->inputIndexes = {0}; sop->outputIndexes = {1}; sop->name = "y";
        net->oplists.emplace_back(std::move(sop));
        flatbuffers::FlatBufferBuilder fb(1024);
        fb.Finish(Net::Pack(fb, net.get()));
        std::shared_ptr<Interpreter> itp(Interpreter::createFromBuffer(fb.GetBufferPointer(), fb.GetSize()), Interpreter::destroy);
        ScheduleConfig c; c.type = MNN_FORWARD_CPU; c.numThread = threads;
        BackendConfig bc; bc.precision = BackendConfig::Precision_High; c.backendConfig = &bc;
        auto s = itp->createSession(c);
        fillInput(itp->getSessionInput(s, nullptr), 1000 + opIndex);
        for (int i = 0; i < warmup; ++i) itp->runSession(s);
        auto t0 = std::chrono::steady_clock::now();
        for (int i = 0; i < iters; ++i) itp->runSession(s);
        auto t1 = std::chrono::steady_clock::now();
        double ms = std::chrono::duration<double, std::milli>(t1 - t0).count() / iters;
        totalMs += ms; ++layers;
        char tmp[64]; snprintf(tmp, sizeof(tmp), "%s%.4f", layers > 1 ? "," : "", ms); per += tmp;
    }
    per += "]";
    printf("{\"ms_total\": %.6f, \"layers\": %d, \"batch\": %d, \"threads\": %d, \"iters\": %d, \"ms_per_layer\": %s}\n",
           totalMs, layers, batch, threads, iters, per.c_str());
    return 0;
}

// export <model.mnn> <outdir>: weights of every conv as decoded by the reference itself
// (ConvolutionCommon::load -> Int8Common{weight, alpha}), to cross-check our own .mnn/IDST reader (SURVEY a1).
static int cmdExport(const char* model, const std::string& dir) {
    auto buf = readFile(model);
    auto net = GetNet(buf.data());
    FILE* idx = fopen((dir + "/convs.txt").c_str(), "w");
    for (int i = 0; i < (int)net->oplists()->size(); ++i) {
        auto op = net->oplists()->GetAs<Op>(i);
        if (op->type() != OpType_Convolution && op->type() != OpType_ConvolutionDepthwise) continue;
        auto conv = op->main_as_Convolution2D();
        if (!conv->quanParameter()) continue;
        auto q = ConvolutionCommon::load(op, nullptr, false, true);
        char name[64]; snprintf(name, sizeof(name), "conv_%04d", i);
        writeFile(dir + "/" + name + ".w8", q->weight.get(), q->weight.size());
        writeFile(dir + "/" + name + ".alpha", q->alpha.get(), q->alpha.size() * 4);
        fprintf(idx, "%s|%s|%d|%d|%d\n", name, op->name() ? op->name()->c_str() : "", (int)q->weight.size(), (int)q->alpha.size(), q->asymmetric ? 1 : 0);
    }
    fclose(idx);
    return 0;
}

int main(int argc, char** argv) {
    if (argc < 2) { fprintf(stderr, "usage: refdump conv|linear|revert|run|clone|bench|convbench|export ...\n"); return 1; }
    std::string cmd = argv[1];
    if (cmd == "conv" && argc >= 4) return cmdConv(argv[2], argv[3]);
    if (cmd == "pool" && argc >= 4) return cmdPool(argv[2], argv[3]);
    if (cmd == "poolf" && argc >= 4) return cmdPoolF(argv[2], argv[3]);
    if (cmd == "matmul" && argc >= 4) return cmdMatMul(argv[2], argv[3]);
    if (cmd == "wino" && argc >= 4) return cmdWino(argv[2], argv[3]);
    if (cmd == "linear" && argc >= 4) return cmdLinear(argv[2], argv[3], argc > 4 ? atoi(argv[4]) : 1);
    if (cmd == "revert" && argc >= 6) return cmdRevert(argv[2], argv[3], atoi(argv[4]), atoi(argv[5]));
    if (cmd == "run" && argc >= 7) return cmdRun(argv[2], atoi(argv[3]), atoi(argv[4]), argv[5], atoi(argv[6]));
    if (cmd == "clone" && argc >= 5) return cmdClone(argv[2], atoi(argv[3]), argv[4], argc > 5 ? argv[5] : nullptr);
    if (cmd == "bench" && argc >= 7) return cmdBench(argv[2], atoi(argv[3]), atoi(argv[4]), atoi(argv[5]), atoi(argv[6]));
    if (cmd == "convbench" && argc >= 8) return cmdConvBench(argv[2], argv[3], atoi(argv[4]), atoi(argv[5]), atoi(argv[6]), atoi(argv[7]));
    if (cmd == "export" && argc >= 4) return cmdExport(argv[2], argv[3]);
    fprintf(stderr, "refdump: bad arguments\n");
    return 1;
}
