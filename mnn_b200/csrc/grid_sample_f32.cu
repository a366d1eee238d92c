// grid_sample_f32.cu -- fp32 GridSample (CPUGridSample, source/backend/cpu/CPUGridSample.cpp) over NCHW-linear tensors: 2-D
// (4-D tensors) and 3-D (5-D tensors), nearest and bilinear / trilinear, zeros and clamp padding (reflection is clamp, as on the
// CPU).
//
// grid_sample_f32_kernel<D3, NEAREST, ZEROS> restates, per output pixel, what the x86 CPU backend computes there on an AVX-512
// host, as its disassembly shows:
//   2-D coordinate  c = 0.5 * fma(1 + g, in - a, -b)         (_AVX512_MNNGridSampleComputeCord, contracted by GCC under -mfma)
//   3-D coordinate  c = k * g + k0, product and sum rounded   (_AVX_MNNGridSampleComputeCord3D, built without -mfma)
//   nearest         tap (int)floor(c + 0.5f)
//   bilinear        taps (int)floor(c), (int)ceil(c), f0 = (float)tap1 - c, f1 = 1 - f0, and per axis from W outwards
//                   v = fma(v1, f1, v0 * f0)                  (GridSampler.hpp's i00 * f0 + i01 * f1 in the avx512 table)
// where (int) is x86's cvttss2si: NaN, +-Inf and |v| >= 2^31 give INT_MIN (cvt_x86).  An out-of-range tap reads +0 under ZEROS
// (still multiplied by its weight) and is clamped otherwise.  The file is built with --fmad=false and every float operation is
// an explicit __fadd_rn / __fmul_rn / __fmaf_rn, so nothing is contracted but what the CPU contracts.
//
// A thread owns one output pixel of one batch and one group of channels: it reads the pixel's grid entry once (one float2 for
// 2-D when the grid is 8-byte aligned), computes the taps and weights once, then loops over the group's channels, gathering 1,
// 4 or 8 taps and storing one value per channel.  Consecutive threads take consecutive pixels, so the stores are coalesced
// along W and the taps of neighbouring pixels share L1 / L2 lines.  The channel groups (GridSampleF32Params::cgroups) are
// chosen at resize so that few-pixel, many-channel shapes still fill the card.  A grid-stride loop over (batch, group, pixel)
// holds any size: the C ABI bounds every index of x, grid and y to 31 bits.
#include <climits>
#include "common.cuh"
#include "grid_sample_ops.h"

namespace mnnb200 {
namespace {

// x86's cvttss2si of an integral float v: the int, or INT_MIN for NaN, +-Inf and values outside the int range
__device__ __forceinline__ int cvt_x86(float v) {
    return (v >= -2147483648.f && v < 2147483648.f) ? __float2int_rz(v) : INT_MIN;
}

// one axis of a bilinear sample: taps t0 <= t1 (unclamped, as the CPU computes them) and weights f0 (of t0), f1 (of t1)
struct Axis {
    int t0, t1;
    float f0, f1;
};
__device__ __forceinline__ Axis bilinear_axis(float c) {
    Axis a;
    a.t0 = cvt_x86(floorf(c));
    a.t1 = cvt_x86(ceilf(c));
    a.f0 = __fsub_rn((float)a.t1, c);
    a.f1 = __fsub_rn(1.0f, a.f0);
    return a;
}
__device__ __forceinline__ int clampi(int v, int n) { return v < 0 ? 0 : (v > n - 1 ? n - 1 : v); }
__device__ __forceinline__ bool inside(int v, int n) { return v >= 0 && v < n; }
// v0 * f0 + v1 * f1 as the AVX-512 table computes it: the second product fused into the sum of the first
__device__ __forceinline__ float lerp(float v0, float v1, float f0, float f1) { return __fmaf_rn(v1, f1, __fmul_rn(v0, f0)); }

template <bool D3, bool NEAREST, bool ZEROS>
__global__ void __launch_bounds__(kGridSampleThreads) grid_sample_f32_kernel(const GridSampleF32Params p, const bool vec2) {
    constexpr int AX = D3 ? 3 : 2;              // grid entries per pixel, axes x (W), y (H)[, z (D)]
    constexpr int TAPS = NEAREST ? 1 : (D3 ? 8 : 4);
    const unsigned pixels = (unsigned)p.pixels;
    const unsigned items = (unsigned)p.n * (unsigned)p.cgroups * pixels;
    const unsigned stride = gridDim.x * blockDim.x;
    const int dims[3] = {p.iw, p.ih, p.id};
    for (unsigned g = blockIdx.x * blockDim.x + threadIdx.x; g < items; g += stride) {
        const unsigned r = g / pixels;               // batch * cgroups + group
        const unsigned pix = g - r * pixels;
        const unsigned b = r / (unsigned)p.cgroups, grp = r - b * (unsigned)p.cgroups;
        // the pixel's coordinates in the CPU's sequence
        float gv[AX];
        const float* gp = p.grid + ((size_t)b * pixels + pix) * AX;
        if (!D3 && vec2) {
            const float2 t = __ldg(reinterpret_cast<const float2*>(gp));
            gv[0] = t.x; gv[AX > 1 ? 1 : 0] = t.y;
        } else {
#pragma unroll
            for (int a = 0; a < AX; ++a) gv[a] = __ldg(gp + a);
        }
        float cord[AX];
#pragma unroll
        for (int a = 0; a < AX; ++a)
            cord[a] = D3 ? __fadd_rn(__fmul_rn(p.k[a], gv[a]), p.k0[a])
                         : __fmul_rn(0.5f, __fmaf_rn(__fadd_rn(1.0f, gv[a]), p.in_a[a], -p.b));
        // tap offsets within one channel's plane, -1 for a tap that reads zero, and the weights
        int off[TAPS];
        float w[AX][2];
        if constexpr (NEAREST) {
            int t[AX];
            bool ok = true;
#pragma unroll
            for (int a = 0; a < AX; ++a) {
                t[a] = cvt_x86(floorf(__fadd_rn(cord[a], 0.5f)));
                if (ZEROS) ok = ok && inside(t[a], dims[a]);
                else t[a] = clampi(t[a], dims[a]);
            }
            off[0] = ok ? ((D3 ? t[D3 ? 2 : 0] * p.ih : 0) + t[1]) * p.iw + t[0] : -1;
        } else {
            int t[AX][2];
            bool ok[AX][2];
#pragma unroll
            for (int a = 0; a < AX; ++a) {
                const Axis ax = bilinear_axis(cord[a]);
                t[a][0] = ax.t0; t[a][1] = ax.t1; w[a][0] = ax.f0; w[a][1] = ax.f1;
#pragma unroll
                for (int s = 0; s < 2; ++s) {
                    ok[a][s] = !ZEROS || inside(t[a][s], dims[a]);
                    if (!ZEROS) t[a][s] = clampi(t[a][s], dims[a]);
                }
            }
            // tap i = (dz, dy, dx) in bit order z y x, as the CPU's s000 .. s111
#pragma unroll
            for (int i = 0; i < TAPS; ++i) {
                const int sx = i & 1, sy = (i >> 1) & 1, sz = (i >> 2) & 1;
                const bool v = ok[0][sx] && ok[1][sy] && (!D3 || ok[D3 ? 2 : 0][sz]);
                off[i] = v ? ((D3 ? t[D3 ? 2 : 0][sz] * p.ih : 0) + t[1][sy]) * p.iw + t[0][sx] : -1;
            }
        }
        const size_t in_plane = (size_t)p.id * p.ih * p.iw;
        const int c0 = (int)grp * p.cper, c1 = min(p.c, c0 + p.cper);
        const float* xp = p.x + ((size_t)b * p.c + c0) * in_plane;
        float* yp = p.y + ((size_t)b * p.c + c0) * pixels + pix;
#pragma unroll 4
        for (int ch = c0; ch < c1; ++ch, xp += in_plane, yp += pixels) {
            float v[TAPS];
#pragma unroll
            for (int i = 0; i < TAPS; ++i) v[i] = (!ZEROS || off[i] >= 0) ? __ldg(xp + off[i]) : 0.0f;
            if constexpr (NEAREST) {
                *yp = v[0];
            } else {
                const float i0 = lerp(lerp(v[0], v[1], w[0][0], w[0][1]), lerp(v[2], v[3], w[0][0], w[0][1]), w[1][0], w[1][1]);
                if constexpr (D3) {
                    const float i1 = lerp(lerp(v[4], v[5], w[0][0], w[0][1]), lerp(v[6], v[7], w[0][0], w[0][1]), w[1][0], w[1][1]);
                    *yp = lerp(i0, i1, w[2][0], w[2][1]);
                } else {
                    *yp = i0;
                }
            }
        }
    }
}

template <bool D3, bool NEAREST>
cudaError_t launch_mode(const GridSampleF32Params& p, bool zeros, bool vec2, int grid, cudaStream_t s) {
    if (zeros)
        grid_sample_f32_kernel<D3, NEAREST, true><<<grid, kGridSampleThreads, 0, s>>>(p, vec2);
    else
        grid_sample_f32_kernel<D3, NEAREST, false><<<grid, kGridSampleThreads, 0, s>>>(p, vec2);
    return cudaGetLastError();
}

}  // namespace

// one thread per work item up to 16 CTAs of 256 threads per SM (two full waves); beyond that the grid-stride loop
int grid_sample_f32_grid(const GridSampleF32Params& p, int sm_count) {
    const long long items = (long long)p.n * p.cgroups * p.pixels;
    const long long cap = 16LL * (sm_count > 0 ? sm_count : 1);
    return (int)std::min(cap, (items + kGridSampleThreads - 1) / kGridSampleThreads);
}

cudaError_t launch_grid_sample_f32(const GridSampleF32Params& p, int rank, bool nearest, bool zeros, bool vec2, int sm_count,
                                   cudaStream_t s) {
    const int grid = grid_sample_f32_grid(p, sm_count);
    if (grid <= 0 || (rank != 4 && rank != 5)) return cudaErrorInvalidValue;
    cudaError_t e;
    if (rank == 4)
        e = nearest ? launch_mode<false, true>(p, zeros, vec2, grid, s) : launch_mode<false, false>(p, zeros, vec2, grid, s);
    else
        e = nearest ? launch_mode<true, true>(p, zeros, false, grid, s) : launch_mode<true, false>(p, zeros, false, grid, s);
    ++g_launch_count;
    return e;
}

}  // namespace mnnb200
