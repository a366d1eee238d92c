// refdump_llm: one LayerNorm or one fused RoPE op as a one-op .mnn, written with the reference's FlatBuffers code (NetT / OpT, as
// `refdump pool` writes its model) and run by the reference's Interpreter on MNN_FORWARD_CPU, or on the plugin when REFDUMP_PLUGIN
// is set.  It reuses refdump.cpp's helpers (file I/O, REFDUMP_PLUGIN loading, plugin statistics) by inclusion.
// TEST INFRASTRUCTURE ONLY.  The RoPE op has a shape computer only in a core built with MNN_SUPPORT_TRANSFORMER_FUSE, so this
// harness links oracle/_ref/libMNN_fuse.so (oracle/build_ref_fuse.py).
//
//   refdump_llm <req.bin> <out.bin> [model.mnn]
//
// The request is an LlmReq, the op's tables, then `runs` sets of inputs; every run is one runSession of the same session with
// that run's inputs, so runs 2 and later go through the plugin's recorded CUDA graph.  out.bin holds every run's outputs in
// order: LayerNorm [sum,] y; RoPE q_out, k_out.  model.mnn, when given, receives the model.
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

struct LlmReq {
    int32_t kind, runs;
    // LayerNorm: form 0 = plain NCHW input, 1 = NC4HW4 1-in / 1-out, 2 = NC4HW4 residual (inputs x, r; outputs x + r, its norm).
    // axis = the number of trailing reduced axes written as axis [-axis, ..., -1] (0: no axis vector); gamma / beta of
    // `affine` values each when present
    int32_t form, rank, dims[4], axis, group, rms, hasGamma, hasBeta, affine;
    float eps;
    // RoPE: q [seq, heads * headDim, 1, 1] and k NC4HW4, cos / sin [seq, ropeDim]; q / k norm tables of headDim values
    int32_t seq, heads, kvHeads, headDim, ropeCut, qNorm, kNorm, normRms, normBeta;
    float normEps;
};

static std::unique_ptr<OpT> inputOp(const char* name, int index, std::vector<int> dims, MNN_DATA_FORMAT fmt) {
    std::unique_ptr<OpT> in(new OpT);
    in->type = OpType_Input; in->name = name; in->outputIndexes = {index};
    in->main.type = OpParameter_Input; in->main.value = new InputT;
    auto ip = in->main.AsInput();
    ip->dims = dims; ip->dtype = DataType_DT_FLOAT; ip->dformat = fmt;
    return in;
}

static LayerNormT* normTable(const float*& p, int size, bool rms, bool beta, float eps) {
    auto t = new LayerNormT;
    t->gamma.assign(p, p + size); p += size;
    if (beta) { t->beta.assign(p, p + size); p += size; }
    t->epsilon = eps; t->useRMSNorm = rms; t->axis = {-1};
    return t;
}

static int cmdLlm(const char* reqPath, const char* outPath, const char* modelPath) {
    auto buf = readFile(reqPath);
    LlmReq r; memcpy(&r, buf.data(), sizeof(r));
    const float* p = (const float*)(buf.data() + sizeof(r));
    std::unique_ptr<NetT> net(new NetT);
    net->sourceType = NetSource_TORCH;
    std::unique_ptr<OpT> op(new OpT);
    std::vector<std::pair<std::string, size_t>> ins;   // input name, elements
    std::vector<std::string> outs;
    if (r.kind == 0) {
        const bool c4 = r.form != 0, residual = r.form == 2;
        std::vector<int> dims(r.dims, r.dims + r.rank);
        size_t n = 1;
        for (int d : dims) n *= d;
        const MNN_DATA_FORMAT fmt = c4 ? MNN_DATA_FORMAT_NC4HW4 : MNN_DATA_FORMAT_NCHW;
        net->oplists.emplace_back(inputOp("x", 0, dims, fmt));
        ins.push_back({"x", n});
        if (residual) { net->oplists.emplace_back(inputOp("r", 1, dims, fmt)); ins.push_back({"r", n}); }
        op->type = OpType_LayerNorm; op->name = "norm";
        op->defaultDimentionFormat = fmt;
        op->main.type = OpParameter_LayerNorm; op->main.value = new LayerNormT;
        auto ln = op->main.AsLayerNorm();
        for (int a = r.axis; a > 0; --a) ln->axis.push_back(-a);
        ln->epsilon = r.eps; ln->group = r.group; ln->useRMSNorm = r.rms != 0;
        if (r.hasGamma) { ln->gamma.assign(p, p + r.affine); p += r.affine; }
        if (r.hasBeta) { ln->beta.assign(p, p + r.affine); p += r.affine; }
        if (residual) {
            op->inputIndexes = {0, 1}; op->outputIndexes = {2, 3};
            net->tensorName = {"x", "r", "sum", "y"}; outs = {"sum", "y"};
        } else {
            op->inputIndexes = {0}; op->outputIndexes = {1};
            net->tensorName = {"x", "y"}; outs = {"y"};
        }
    } else {
        const int hd = r.headDim;
        const int ropeDim = (r.ropeCut <= 0 || r.ropeCut > hd ? hd : r.ropeCut) / 2 * 2;
        net->oplists.emplace_back(inputOp("q", 0, {r.seq, r.heads * hd, 1, 1}, MNN_DATA_FORMAT_NC4HW4));
        net->oplists.emplace_back(inputOp("k", 1, {r.seq, r.kvHeads * hd, 1, 1}, MNN_DATA_FORMAT_NC4HW4));
        net->oplists.emplace_back(inputOp("cos", 2, {r.seq, ropeDim}, MNN_DATA_FORMAT_NCHW));
        net->oplists.emplace_back(inputOp("sin", 3, {r.seq, ropeDim}, MNN_DATA_FORMAT_NCHW));
        ins = {{"q", (size_t)r.seq * r.heads * hd}, {"k", (size_t)r.seq * r.kvHeads * hd}, {"cos", (size_t)r.seq * ropeDim},
               {"sin", (size_t)r.seq * ropeDim}};
        op->type = OpType_RoPE; op->name = "rope";
        op->main.type = OpParameter_RoPEParam; op->main.value = new RoPEParamT;
        auto rp = op->main.AsRoPEParam();
        rp->num_head = r.heads; rp->kv_num_head = r.kvHeads; rp->head_dim = hd; rp->rope_cut_head_dim = r.ropeCut;
        if (r.qNorm) rp->q_norm.reset(normTable(p, hd, r.normRms != 0, r.normBeta != 0, r.normEps));
        if (r.kNorm) rp->k_norm.reset(normTable(p, hd, r.normRms != 0, r.normBeta != 0, r.normEps));
        op->inputIndexes = {0, 1, 2, 3}; op->outputIndexes = {4, 5};
        net->tensorName = {"q", "k", "cos", "sin", "q_out", "k_out"}; outs = {"q_out", "k_out"};
    }
    net->oplists.emplace_back(std::move(op));
    net->outputName = outs;
    flatbuffers::FlatBufferBuilder fb(1024);
    fb.Finish(Net::Pack(fb, net.get()));
    if (modelPath) writeFile(modelPath, fb.GetBufferPointer(), fb.GetSize());

    std::shared_ptr<Interpreter> itp(Interpreter::createFromBuffer(fb.GetBufferPointer(), fb.GetSize()), Interpreter::destroy);
    ScheduleConfig c; c.type = forwardType(); c.numThread = 1;
    BackendConfig bc; bc.precision = BackendConfig::Precision_High; c.backendConfig = &bc;
    auto s = itp->createSession(c);
    if (!s) { fprintf(stderr, "refdump_llm: createSession failed\n"); return 2; }
    std::ofstream o(outPath, std::ios::binary);
    for (int run = 0; run < r.runs; ++run) {
        for (auto& in : ins) {
            auto t = itp->getSessionInput(s, in.first.c_str());
            Tensor host(t, Tensor::CAFFE);
            if ((size_t)host.elementSize() != in.second) { fprintf(stderr, "refdump_llm: input %s size\n", in.first.c_str()); return 2; }
            memcpy(host.host<float>(), p, in.second * 4); p += in.second;
            t->copyFromHostTensor(&host);
        }
        if (itp->runSession(s) != NO_ERROR) { fprintf(stderr, "refdump_llm: runSession failed\n"); return 2; }
        for (auto& name : outs) {
            auto t = itp->getSessionOutput(s, name.c_str());
            // NC4HW4 outputs read back as NCHW ([tokens][C]); RoPE's NHWC outputs as they are ([seq][heads][head_dim])
            auto dt = t->getDimensionType() == Tensor::CAFFE_C4 ? Tensor::CAFFE : t->getDimensionType();
            Tensor host(t, dt);
            t->copyToHostTensor(&host);
            o.write((const char*)host.host<float>(), (size_t)host.elementSize() * 4);
        }
    }
    pluginStats();
    return 0;
}

int main(int argc, char** argv) {
    if (argc >= 3) return cmdLlm(argv[1], argv[2], argc > 3 ? argv[3] : nullptr);
    fprintf(stderr, "usage: refdump_llm <req.bin> <out.bin> [model.mnn]\n");
    return 1;
}
