// deconv_ops.h -- host-callable launchers of libmnn_b200_deconv.so's kernels (deconv_f32_wgmma.cu), enqueue-only on the given
// stream.
#pragma once
#include <cuda_runtime.h>
#include "kernels.h"   // DwF32Params

namespace mnnb200 {

// fp32 Deconvolution (transposed conv, group 1) on split-TF32 wgmma (deconv_f32_wgmma.cu), NCHW-linear fp32 in and out.
// y[n][oc][oy][ox] = bias + sum x[n][ic][iy][ix] w[ic][oc][ky][kx] over oy + pad_h = iy * sh + ky * dh (and the same in x).  Output
// pixels with the same (oy + pad_h) % sh and (ox + pad_w) % sw -- one phase -- share their taps, so each of the sh * sw phases is a
// stride-1 implicit GEMM over the input: M = the phase's output pixels, N = oc, K = the phase's taps * cp8.
constexpr int kDeconvMaxStride = 16;
// The taps of one axis whose outputs u = o + pad have u % s == r: k = k0 + t * kstep for t < nk, reading input
// u / s - (off0 + t * istep).  kstep = s / gcd(s, d), istep = d / gcd(s, d); phase r = 0 always has tap 0.
struct DeconvAxisTaps {
    int k0, nk, off0, kstep, istep;
};
__host__ __device__ inline DeconvAxisTaps deconv_axis_taps(int r, int s, int d, int K) {
    int g = s, b = d;
    while (b) { const int t = g % b; g = b; b = t; }
    DeconvAxisTaps a{0, 0, 0, s / g, d / g};
    for (int k = 0; k < K && k < a.kstep; ++k)
        if ((k * d) % s == r) {
            a.k0 = k;
            a.nk = (K - 1 - k) / a.kstep + 1;
            a.off0 = (k * d - r) / s;
            break;
        }
    return a;
}
// One phase residue of one output axis: outputs o0, o0 + s, ... (len of them), the first reading input q0 - off0 (tap 0 of the
// phase), nk taps, istep input rows apart
struct DeconvAxis {
    int o0, len, q0, nk, off0;
};
struct DeconvF32Params {
    const float* x;       // [N][IC][IH][IW]
    float* y;             // [N][OC][OH][OW]
    const float* bias;    // [OC]
    int N, IC, IH, IW, OC, OH, OW;
    int sh, sw, istep_h, istep_w;
    int Cp8, ocp, n_chunks, items;
    int act;              // 0 none, 1 ReLU, 2 ReLU6
    DeconvAxis ay[kDeconvMaxStride], ax[kDeconvMaxStride];   // by (oy + pad_h) % sh and (ox + pad_w) % sw
    int item_end[kDeconvMaxStride * kDeconvMaxStride];    // work items of phases 0..ph (ph = ry * sw + rx), m tile-major
};
// w [ic][oc][kh][kw] -> hi / lo [sh * sw][ocp][kp], per phase k = (ty * nkx + tx) * cp8 + c, zero padded; w = hi + lo
cudaError_t launch_pack_deconv_w_f32(const float* w, int ic, int oc, int kh, int kw, int sh, int sw, int dh, int dw, int cp8,
                                     int kp, int ocp, float* hi, float* lo, cudaStream_t s);
// tmap_hi / tmap_lo: 2D maps over the [sh * sw * ocp][kp * 4 bytes] weight arrays with {128 bytes, bn rows} boxes, 128B swizzle
cudaError_t launch_deconv_f32_wgmma(const DeconvF32Params& p, const void* tmap_hi, const void* tmap_lo, int bn, cudaStream_t s,
                                    int sm_count);
int deconv_f32_stages(int bn);

// transposed depthwise conv (CPUDeconvolutionDepthwise): w [C][KH*KW], ph / pw the begin pads; one thread per output
cudaError_t launch_dwdeconv_f32(const DwF32Params& p, cudaStream_t s);

}  // namespace mnnb200
