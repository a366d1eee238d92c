// activations.cuh -- the fp32 sigmoid and tanh the float kernels share: UnaryOp's SIGMOID / TANH / SILU / GELU (elementwise.cu)
// and the LSTM / RNN gates (rnn.cu) compute them with the same expressions, so a gate equals the UnaryOp of its argument bit
// for bit.
#pragma once
#include <cuda_runtime.h>

namespace mnnb200 {

// x * sigmoid(t) = x / (1 + e^-t) for t >= 0, x e^t / (1 + e^t) for t < 0: e^-|t| never overflows, so the result keeps its
// magnitude where 1 / (1 + e^-t) would be 1 / inf (t < -88.7).  Below t = -64 (1 + e^t is then 1) the exponential is taken at
// t + 32 (exact for |t| < 256, beyond which the result is 0 anyway) and the product scaled by e^-32, so that a subnormal e^t
// does not lose the digits the product still has.
__device__ __forceinline__ float times_sigmoid(float x, float t) {
    if (t >= 0.f) return __fdiv_rn(x, __fadd_rn(1.f, expf(-t)));
    if (t >= -64.f) {
        const float e = expf(t);
        return __fdiv_rn(__fmul_rn(x, e), __fadd_rn(1.f, e));
    }
    return __fmul_rn(__fmul_rn(x, expf(__fadd_rn(t, 32.f))), 1.26641655e-14f);   // e^-32
}
__device__ __forceinline__ float sigmoid_f32(float x) { return x >= -64.f ? times_sigmoid(1.f, x) : expf(x); }   // 1 + e^x is 1 below -64
__device__ __forceinline__ float tanh_f32(float x) { return tanhf(x); }

}  // namespace mnnb200
