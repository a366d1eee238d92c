// refdump_w4: the reference's LLM linear layer with 4-bit weights, the request format of `refdump linear` (oracle/refdump.cpp,
// whose helpers -- file I/O, REFDUMP_PLUGIN loading, plugin statistics -- it reuses by inclusion).  TEST INFRASTRUCTURE ONLY.
//
//   refdump_w4 linear <req.bin> <out.bin> [threads]
//
// The request's weights are q in [-8, 7], one byte each.  They are encoded as a 4-bit IDST layer the way MNN-LLM's export writes
// one (--quant_bit 4: IDSTEncoder::encode(..., {4, false}), aMin = -8, transformers/llm/export/utils/mnn_converter.py:751-764),
// so ConvolutionCommon::load hands the backend packed nibbles (canUseInt4) and turns each wire min into min + 8 * scale.
// its headers first, so that renaming its main() below cannot reach the `main()` accessor of the generated schema types
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
#define main(...) refdump_main(__VA_ARGS__)
#include "refdump.cpp"
#undef main

static int cmdLinearW4(const char* reqPath, const char* outPath, int threads) {
    auto buf = readFile(reqPath);
    LinReq r; memcpy(&r, buf.data(), sizeof(r));
    const char* p = buf.data() + sizeof(r);
    std::vector<float> x((size_t)r.tokens * r.ic); memcpy(x.data(), p, x.size() * 4); p += x.size() * 4;
    std::vector<int8_t> wq((size_t)r.oc * r.ic); memcpy(wq.data(), p, wq.size()); p += wq.size();
    const int blocks = r.pad > 0 ? r.pad : 1;
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
    conv2D->quanParameter = IDSTEncoder::encode(nullptr, alpha, r.ic, r.oc, r.asym != 0, wq.data(), -8, {4, false});
    conv2D->common->outputCount = r.oc; conv2D->common->inputCount = r.ic;
    conv2D->common->kernelX = 1; conv2D->common->kernelY = 1;
    conv2D->common->relu = r.relu != 0; conv2D->common->relu6 = r.relu6 != 0;
    conv2D->bias = bias;
    VARP xin = _Input({1, r.ic, r.tokens, 1}, NCHW, halide_type_of<float>());
    auto xp = xin->writeMap<float>();
    for (int t = 0; t < r.tokens; ++t) for (int c = 0; c < r.ic; ++c) xp[(size_t)c * r.tokens + t] = x[(size_t)t * r.ic + c];
    auto y = Variable::create(Expr::create(convOp.get(), {_Convert(xin, NC4HW4)}));
    y = _Convert(y, NCHW);
    auto yp = y->readMap<float>();
    if (!yp) { fprintf(stderr, "refdump_w4 linear: run failed\n"); return 2; }
    std::vector<float> out((size_t)r.tokens * r.oc);
    for (int t = 0; t < r.tokens; ++t) for (int o = 0; o < r.oc; ++o) out[(size_t)t * r.oc + o] = yp[(size_t)o * r.tokens + t];
    writeFile(outPath, out.data(), out.size() * 4);
    pluginStats();
    return 0;
}

int main(int argc, char** argv) {
    if (argc >= 4 && std::string(argv[1]) == "linear") return cmdLinearW4(argv[2], argv[3], argc > 4 ? atoi(argv[4]) : 1);
    fprintf(stderr, "usage: refdump_w4 linear <req.bin> <out.bin> [threads]\n");
    return 1;
}
