// conv_int8_stem.cu -- the network's first convolution: <= 4 input channels (an RGB image), any kernel / stride / pad.
//
// In the NHWC16 device layout such a layer has K = taps x 16 with 75-81 % structural zeros; the implicit-GEMM kernel spends
// 36 us on MobileNet-v2's 3x3/s2 stem at batch 32 for 6 us worth of HBM traffic.  Here one thread owns one output pixel and
// all (<= 64) output channels: per tap it reads the pixel's 4 real channels as one 32-bit word and issues one dp4a per output
// channel against a tap-major weight table in shared memory (16-byte broadcast loads).  Same accumulator (incl. the x86
// +128 storage offset added as 128*sum(w)) and the same exact fp32 requantisation as every other conv kernel (common.cuh).
#include "common.cuh"
#include "kernels.h"

namespace mnnb200 {

namespace {

template <int OCP>
__global__ void __launch_bounds__(128) conv_int8_stem_kernel(const ConvParams p) {
    extern __shared__ uint32_t w_s[];                 // [taps][OCP] words = 4 input channels of one (tap, oc)
    __shared__ float s_scale[OCP], s_bias[OCP];
    __shared__ int s_wsum[OCP];
    const int taps = p.KH * p.KW;
    if (threadIdx.x < OCP) {
        const bool v = threadIdx.x < p.OC;
        s_scale[threadIdx.x] = v ? p.wscale[threadIdx.x] : 0.f;
        s_bias[threadIdx.x] = v ? p.bias[threadIdx.x] : 0.f;
        s_wsum[threadIdx.x] = v ? p.wsum128[threadIdx.x] : 0;
    }
    for (int i = threadIdx.x; i < taps * OCP; i += blockDim.x) {
        const int t = i / OCP, oc = i - t * OCP;
        w_s[i] = *reinterpret_cast<const uint32_t*>(p.w + ((size_t)oc * taps + t) * p.Cp);
    }
    __syncthreads();
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= p.M) return;
    const int ox = m % p.OW, oy = (m / p.OW) % p.OH, b = m / (p.OW * p.OH);
    int acc[OCP];
#pragma unroll
    for (int o = 0; o < OCP; ++o) acc[o] = 0;
    const int iy0 = oy * p.sh - p.ph, ix0 = ox * p.sw - p.pw;
    for (int ky = 0; ky < p.KH; ++ky) {
        const int iy = iy0 + ky * p.dh;
        for (int kx = 0; kx < p.KW; ++kx) {
            const int ix = ix0 + kx * p.dw;
            int xw = p.zin_splat;                     // padded taps hold the input zero point (ConvInt8TiledExecutor.cpp:2269-2271)
            if (iy >= 0 && iy < p.IH && ix >= 0 && ix < p.IW)
                xw = *reinterpret_cast<const int*>(p.x + (((size_t)b * p.IH + iy) * p.IW + ix) * p.Cp);
            const uint4* wt = reinterpret_cast<const uint4*>(w_s + (ky * p.KW + kx) * OCP);
#pragma unroll
            for (int o4 = 0; o4 < OCP / 4; ++o4) {
                const uint4 wv = wt[o4];
                acc[o4 * 4 + 0] = __dp4a(xw, (int)wv.x, acc[o4 * 4 + 0]);
                acc[o4 * 4 + 1] = __dp4a(xw, (int)wv.y, acc[o4 * 4 + 1]);
                acc[o4 * 4 + 2] = __dp4a(xw, (int)wv.z, acc[o4 * 4 + 2]);
                acc[o4 * 4 + 3] = __dp4a(xw, (int)wv.w, acc[o4 * 4 + 3]);
            }
        }
    }
    int8_t* yrow = p.y + (size_t)m * p.OCp;
#pragma unroll
    for (int g = 0; g < OCP / 16; ++g) {
        int8_t q[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            const int o = g * 16 + k;
            int v = requant_cpu_exact(acc[o] + s_wsum[o], s_scale[o], p.scale_x, s_bias[o], p.minv, p.maxv);
            q[k] = o < p.OC ? (int8_t)v : (int8_t)0;
        }
        *reinterpret_cast<int4*>(yrow + g * 16) = *reinterpret_cast<const int4*>(q);
    }
}

}  // namespace

bool conv_int8_stem_supported(const ConvParams& p, int ic) {
    return ic <= 4 && p.Cp == 16 && (p.OCp == 16 || p.OCp == 32 || p.OCp == 64);
}

cudaError_t launch_conv_int8_stem(const ConvParams& p, cudaStream_t stream) {
    const int grid = (p.M + 127) / 128;
    const int smem = p.KH * p.KW * p.OCp * 4;
    ++g_launch_count;
    if (p.OCp == 16) conv_int8_stem_kernel<16><<<grid, 128, smem, stream>>>(p);
    else if (p.OCp == 32) conv_int8_stem_kernel<32><<<grid, 128, smem, stream>>>(p);
    else conv_int8_stem_kernel<64><<<grid, 128, smem, stream>>>(p);
    return cudaGetLastError();
}

}  // namespace mnnb200
