// refdump_ops -- the reference's fp32 neighbour ops one op at a time (BinaryOp, Eltwise, ReLU, UnaryOp, Pooling, Reduction,
// Softmax, ArgMax / ArgMin, Scale, and the Raster producers: Transpose, Concat, Slice, StridedSlice, Pad, Tile, BroadcastTo,
// Reshape, ConvertTensor), for the tests of the plugin's float executions.
//
//   refdump_ops <request> <out>   every case of the request, in order, each built with the Express API (or as an OpT where
//                                 Express leaves a field out) and run through the Express executor on MNN_FORWARD_CPU
//                                 (REFDUMP_PLUGIN: on the plugin), once per run listed, on one executor.  A run may give its
//                                 inputs new shapes: the variables are resized before the values are written.
//
// Every word of both files is 32-bit little-endian.
//   request: int32 cases, then per case
//              int32 kind, int32 ni, int32 ip[ni], int32 nf, float fp[nf],
//              int32 inputs, per input int32 type (0 float, 1 int32), int32 format (0 NCHW, 1 NHWC),
//              int32 runs, per run and per input: int32 ndim, int32 dims[ndim], then the input's values
//   out:     per case int32 ok (0: a run failed, no outputs follow), int32 created, int32 declined (the plugin's counts for the
//            case, 0 on the CPU), int32 runs, per run int32 type (0 float, 1 int32), int32 ndim, int32 dims[ndim], values
#include <MNN/expr/Expr.hpp>
#include <MNN/expr/ExprCreator.hpp>
#include <MNN/expr/Executor.hpp>
#include <MNN/expr/ExecutorScope.hpp>
#include <dlfcn.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <string>
#include <vector>
#include "MNN_generated.h"

using namespace MNN;
using namespace MNN::Express;

enum Kind {
    K_BINARY = 0, K_ELTWISE, K_RELU, K_UNARY, K_POOL, K_REDUCE, K_SOFTMAX, K_ARGMAX, K_SCALE, K_TRANSPOSE, K_CONCAT,
    K_STRIDED_SLICE, K_SLICE, K_PAD, K_TILE, K_BROADCAST_TO, K_RESHAPE, K_CONVERT
};

static void* g_plugin = nullptr;
static MNNForwardType forwardType() {
    const char* p = getenv("REFDUMP_PLUGIN");
    if (!p || !*p) return MNN_FORWARD_CPU;
    g_plugin = dlopen(p, RTLD_NOW | RTLD_GLOBAL);
    if (!g_plugin) { fprintf(stderr, "refdump_ops: dlopen(%s): %s\n", p, dlerror()); exit(3); }
    return MNN_FORWARD_CUDA;
}
static void pluginStats(int* created, int* declined) {
    *created = *declined = 0;
    if (!g_plugin) return;
    typedef void (*Fn)(int*, int*);
    Fn fn = (Fn)dlsym(g_plugin, "mnnb200_plugin_stats");
    if (fn) fn(created, declined);
}

struct Reader {
    std::vector<char> buf;
    size_t at = 0;
    int32_t i() { int32_t v; memcpy(&v, buf.data() + at, 4); at += 4; return v; }
    float f() { float v; memcpy(&v, buf.data() + at, 4); at += 4; return v; }
    const char* take(size_t bytes) { const char* p = buf.data() + at; at += bytes; return p; }
};

static VARP intConst(const std::vector<int>& v) { return _Const(v.data(), {(int)v.size()}, NCHW, halide_type_of<int>()); }
static VARP opVar(OpT* op, const std::vector<VARP>& in) {
    std::unique_ptr<OpT> own(op);
    return Variable::create(Expr::create(own.get(), in));
}

// the case's op on its input variables
static VARP build(int kind, const std::vector<int>& ip, const std::vector<float>& fp, const std::vector<VARP>& x) {
    switch (kind) {
        case K_BINARY: {   // ip: opType, activationType (Express's _Add & co. leave activationType 0)
            auto op = new OpT;
            op->type = OpType_BinaryOp;
            op->main.type = OpParameter_BinaryOp;
            auto p = new BinaryOpT;
            p->opType = (BinaryOpOperation)ip[0];
            p->T = DataType_DT_FLOAT;
            p->activationType = ip[1];
            op->main.value = p;
            return opVar(op, {x[0], x[1]});
        }
        case K_ELTWISE: {   // ip: type; fp: coeff (none for the plain fold)
            auto op = new OpT;
            op->type = OpType_Eltwise;
            op->main.type = OpParameter_Eltwise;
            auto p = new EltwiseT;
            p->type = (EltwiseType)ip[0];
            p->coeff = fp;
            op->main.value = p;
            return opVar(op, x);
        }
        case K_RELU:
            return _Relu(x[0], fp[0]);
        case K_UNARY: {
            auto op = new OpT;
            op->type = OpType_UnaryOp;
            op->main.type = OpParameter_UnaryOp;
            auto p = new UnaryOpT;
            p->opType = (UnaryOpOperation)ip[0];
            p->T = DataType_DT_FLOAT;
            op->main.value = p;
            return opVar(op, {x[0]});
        }
        case K_POOL: {   // ip: type, kh, kw, sh, sw, padType, padY, padX, isGlobal, ceilModel, countType, npads, pads...
            auto op = new OpT;
            op->type = OpType_Pooling;
            op->main.type = OpParameter_Pool;
            auto p = new PoolT;
            p->type = (PoolType)ip[0];
            p->kernelY = ip[1]; p->kernelX = ip[2]; p->strideY = ip[3]; p->strideX = ip[4];
            p->padType = (PoolPadType)ip[5];
            p->padY = ip[6]; p->padX = ip[7];
            p->isGlobal = ip[8] != 0;
            p->ceilModel = ip[9] != 0;
            p->countType = (AvgPoolCountType)ip[10];
            p->pads.assign(ip.begin() + 12, ip.begin() + 12 + ip[11]);
            op->main.value = p;
            return opVar(op, {x[0]});
        }
        case K_REDUCE: {   // ip: operation, keepDims, axes...
            auto op = new OpT;
            op->type = OpType_Reduction;
            op->main.type = OpParameter_ReductionParam;
            auto p = new ReductionParamT;
            p->operation = (ReductionType)ip[0];
            p->keepDims = ip[1] != 0;
            p->dim.assign(ip.begin() + 2, ip.end());
            p->dType = DataType_DT_FLOAT;
            op->main.value = p;
            return opVar(op, {x[0]});
        }
        case K_SOFTMAX:
            return _Softmax(x[0], ip[0]);
        case K_ARGMAX: {   // ip: isMin, axis, topK, outMaxVal (Express's _ArgMax leaves topK 0; the converters write 1)
            auto op = new OpT;
            op->type = ip[0] ? OpType_ArgMin : OpType_ArgMax;
            op->main.type = OpParameter_ArgMax;
            auto p = new ArgMaxT;
            p->axis = ip[1];
            p->topK = ip[2];
            p->outMaxVal = ip[3];
            op->main.value = p;
            return opVar(op, {x[0]});
        }
        case K_SCALE: {   // ip: channels, hasBias; fp: scale[channels], then bias[channels] when hasBias
            auto op = new OpT;
            op->type = OpType_Scale;
            op->main.type = OpParameter_Scale;
            auto p = new ScaleT;
            p->channels = ip[0];
            p->scaleData.assign(fp.begin(), fp.begin() + ip[0]);
            if (ip[1]) p->biasData.assign(fp.begin() + ip[0], fp.begin() + 2 * ip[0]);
            op->main.value = p;
            // CPUScale reads and writes NC4HW4, as a Scale behind a convolution has it
            return _Convert(opVar(op, {_Convert(x[0], NC4HW4)}), NCHW);
        }
        case K_TRANSPOSE:
            return _Transpose(x[0], ip);
        case K_CONCAT:
            return _Concat(x, ip[0]);
        case K_STRIDED_SLICE: {   // ip: n, begin[n], end[n], strides[n], beginMask, endMask
            const int n = ip[0];
            std::vector<int> b(ip.begin() + 1, ip.begin() + 1 + n), e(ip.begin() + 1 + n, ip.begin() + 1 + 2 * n),
                s(ip.begin() + 1 + 2 * n, ip.begin() + 1 + 3 * n);
            return _StridedSlice(x[0], intConst(b), intConst(e), intConst(s), ip[1 + 3 * n], ip[2 + 3 * n], 0, 0, 0);
        }
        case K_SLICE: {   // ip: n, starts[n], sizes[n]
            const int n = ip[0];
            return _Slice(x[0], intConst(std::vector<int>(ip.begin() + 1, ip.begin() + 1 + n)),
                          intConst(std::vector<int>(ip.begin() + 1 + n, ip.begin() + 1 + 2 * n)));
        }
        case K_PAD:   // ip: (before, after) per dimension
            return _Pad(x[0], intConst(ip), CONSTANT);
        case K_TILE:
            return _Tile(x[0], intConst(ip));
        case K_BROADCAST_TO:
            return _BroadcastTo(x[0], intConst(ip));
        case K_RESHAPE:   // ip: original format (0 NCHW, 1 NHWC), shape...
            return _Reshape(x[0], std::vector<int>(ip.begin() + 1, ip.end()), ip[0] ? NHWC : NCHW);
        case K_CONVERT:   // ip: format (0 NCHW, 1 NHWC)
            return _Convert(x[0], ip[0] ? NHWC : NCHW);
        default:
            return nullptr;
    }
}

int main(int argc, char** argv) {
    if (argc < 3) {
        fprintf(stderr, "usage: refdump_ops <request> <out>\n");
        return 1;
    }
    Reader r;
    {
        std::ifstream f(argv[1], std::ios::binary);
        r.buf.assign(std::istreambuf_iterator<char>(f), std::istreambuf_iterator<char>());
    }
    BackendConfig bc;
    bc.precision = BackendConfig::Precision_High;
    ExecutorScope scope(Executor::newExecutor(forwardType(), bc, 1));
    std::ofstream o(argv[2], std::ios::binary);
    auto put = [&](int32_t v) { o.write((const char*)&v, 4); };
    const int cases = r.i();
    for (int c = 0; c < cases; ++c) {
        const int kind = r.i();
        std::vector<int> ip(r.i());
        for (auto& v : ip) v = r.i();
        std::vector<float> fp(r.i());
        for (auto& v : fp) v = r.f();
        const int nin = r.i();
        std::vector<int> types(nin), fmts(nin);
        for (int k = 0; k < nin; ++k) { types[k] = r.i(); fmts[k] = r.i(); }
        const int runs = r.i();
        int c0, d0, c1, d1;
        pluginStats(&c0, &d0);
        std::vector<VARP> x(nin);
        VARP y;
        std::vector<char> outs;   // the case's runs, written after its counts
        auto out32 = [&](int32_t v) { outs.insert(outs.end(), (const char*)&v, (const char*)&v + 4); };
        bool ok = true;
        for (int run = 0; run < runs; ++run) {
            for (int k = 0; k < nin; ++k) {
                std::vector<int> dims(r.i());
                size_t count = 1;
                for (auto& d : dims) { d = r.i(); count *= (size_t)d; }
                const char* data = r.take(count * 4);
                if (run == 0) {
                    x[k] = _Input(dims, fmts[k] ? NHWC : NCHW, types[k] ? halide_type_of<int>() : halide_type_of<float>());
                } else if (x[k]->getInfo()->dim != dims) {
                    x[k]->resize(dims);
                }
                if (!ok) continue;
                void* w = types[k] ? (void*)x[k]->writeMap<int>() : (void*)x[k]->writeMap<float>();
                if (!w) { ok = false; continue; }
                memcpy(w, data, count * 4);
            }
            if (!ok) continue;
            if (run == 0) {
                y = build(kind, ip, fp, x);
                auto info = y.get() ? y->getInfo() : nullptr;
                if (info && info->order == NC4HW4) y = _Convert(y, NCHW);
            }
            auto info = y.get() ? y->getInfo() : nullptr;
            const void* py = info ? y->readMap<void>() : nullptr;
            if (!py) { ok = false; continue; }
            out32(info->type.code == halide_type_float ? 0 : 1);
            out32((int32_t)info->dim.size());
            for (auto d : info->dim) out32(d);
            outs.insert(outs.end(), (const char*)py, (const char*)py + (size_t)info->size * 4);
        }
        y = nullptr;
        x.clear();
        pluginStats(&c1, &d1);
        put(ok ? 1 : 0);
        put(c1 - c0);
        put(d1 - d0);
        put(ok ? runs : 0);
        if (ok) o.write(outs.data(), outs.size());
    }
    return 0;
}
