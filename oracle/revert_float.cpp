// revert_float -- seeded fp32 weights for the reference's weight-less benchmark graphs.
//
// TEST INFRASTRUCTURE ONLY (built by oracle/float_models.py against the reference headers and oracle/_ref/libMNN.so).
// The reference's Revert tool (tools/cpp/revertMNNModel.cpp:143-231) sizes every conv's weight and bias but leaves them at
// zero unless it quantises the model; a float model needs real weights to be a test of anything.
//
// revert_float <weightless.mnn> <out.mnn> <seed>
//   Convolution / ConvolutionDepthwise: weights U(-1, 1) * 1.2 / sqrt(ks) (ks = weights per output channel, the magnitude
//   refdump's retuned int8 revert uses, so activations stay O(1)), biases U(-0.1, 0.1).
//   Scale: scale U(0.9, 1.1), bias U(-0.05, 0.05).
//   Everything else, relu6 included, is left as Revert leaves it in float mode.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <memory>
#include <random>
#include <vector>
#include "MNN_generated.h"
#include "revertMNNModel.hpp"

using namespace MNN;

int main(int argc, char** argv) {
    if (argc < 4) { fprintf(stderr, "usage: revert_float <weightless.mnn> <out.mnn> <seed>\n"); return 1; }
    Revert r(argv[1]);
    r.initialize(0.f, 1, false, false);
    std::unique_ptr<NetT> net(UnPackNet(r.getBuffer()));
    std::mt19937 rng(atoi(argv[3]));
    std::uniform_real_distribution<float> u(-1.f, 1.f);
    int convs = 0;
    for (auto& op : net->oplists) {
        if (op->type == OpType_Convolution || op->type == OpType_ConvolutionDepthwise) {
            auto conv = op->main.AsConvolution2D();
            const int oc = conv->common->outputCount;
            if (oc <= 0 || conv->weight.empty()) continue;
            const size_t ks = conv->weight.size() / oc;
            const float mag = 1.2f / std::sqrt((float)ks);
            for (auto& w : conv->weight) w = u(rng) * mag;
            conv->bias.resize(oc);
            for (auto& b : conv->bias) b = u(rng) * 0.1f;
            ++convs;
        } else if (op->type == OpType_Scale) {
            auto sc = op->main.AsScale();
            for (auto& s : sc->scaleData) s = 1.f + 0.1f * u(rng);
            for (auto& b : sc->biasData) b = 0.05f * u(rng);
        }
    }
    flatbuffers::FlatBufferBuilder b(1024);
    b.Finish(Net::Pack(b, net.get()));
    std::ofstream o(argv[2], std::ios::binary);
    o.write((const char*)b.GetBufferPointer(), b.GetSize());
    printf("revert_float: %d convolutions seeded\n", convs);
    return o.good() ? 0 : 2;
}
