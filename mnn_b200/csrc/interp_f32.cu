// interp_f32.cu -- fp32 Interp (CPUInterp, source/backend/cpu/CPUInterp.cpp) over NCHW-linear planes: nearest (resize type 1),
// bilinear (2), cubic (3) and nearest-round (4).
//
// interp_f32_kernel<TAPS, VEC>: every per-column and per-row index and weight comes from the tables resize built on the host in
// the CPU's expressions (interp_capi.cu), so the kernel only gathers and, for TAPS > 1, multiplies and adds in the CPU's order:
// horizontal first, ((x0 * w0 + x1 * w1) + x2 * w2) + x3 * w3 per input row, then the same over the rows.  Every product and sum
// is a separately rounded __fmul_rn / __fadd_rn (the file is also built with --fmad=false), as the reference's SSE Vec4 without
// -mfma computes them: all four types are bit-identical to the CPU.
//
// The op is bound by its output stores (up to 64x its input).  A thread owns a group of output columns of one row: 4 with a
// 16-byte store when ow % 4 == 0 and y is 16-byte aligned (VEC), else 1 with a scalar store; consecutive threads take
// consecutive groups of a row, so the stores are coalesced along W.  The input rows the CTA's threads share are read through
// the read-only path and hit L1 / L2 after their first read.  A grid-stride loop over (plane, row, group) holds any number of
// planes and rows: the C ABI bounds every index of x and y to 31 bits.
#include "common.cuh"
#include "interp_ops.h"

namespace mnnb200 {
namespace {

// x0 * w0 + x1 * w1 (+ x2 * w2 + x3 * w3), summed left to right, every operation rounded on its own
template <int TAPS>
__device__ __forceinline__ float taps_sum(const float (&v)[TAPS], const float (&w)[TAPS]) {
    float s = __fadd_rn(__fmul_rn(v[0], w[0]), __fmul_rn(v[1], w[1]));
#pragma unroll
    for (int i = 2; i < TAPS; ++i) s = __fadd_rn(s, __fmul_rn(v[i], w[i]));
    return s;
}

template <int TAPS, bool VEC>
__global__ void __launch_bounds__(kInterpThreads) interp_f32_kernel(const InterpF32Params p) {
    constexpr int W = VEC ? 4 : 1;
    const unsigned row_groups = (unsigned)(p.ow / W);
    const unsigned groups = (unsigned)p.planes * (unsigned)p.oh * row_groups;
    const unsigned stride = gridDim.x * blockDim.x;
    for (unsigned g = blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += stride) {
        const unsigned r = g / row_groups;            // output row of all planes: plane * oh + oy
        const int ox0 = (int)(g - r * row_groups) * W;
        const int plane = (int)(r / (unsigned)p.oh), oy = (int)(r - (unsigned)plane * p.oh);
        const float* __restrict__ base = p.x + (size_t)plane * p.ih * p.iw;
        const float* __restrict__ rows[TAPS];
        float wy[TAPS];
#pragma unroll
        for (int j = 0; j < TAPS; ++j) {
            rows[j] = base + __ldg(p.yi + oy * TAPS + j) * p.iw;
            if (TAPS > 1) wy[j] = __ldg(p.yw + oy * TAPS + j);
        }
        float out[W];
#pragma unroll
        for (int k = 0; k < W; ++k) {
            const int c = ox0 + k;
            int cx[TAPS];
#pragma unroll
            for (int i = 0; i < TAPS; ++i) cx[i] = __ldg(p.xi + c * TAPS + i);
            if (TAPS == 1) {
                out[k] = __ldg(rows[0] + cx[0]);
            } else {
                float wx[TAPS], h[TAPS];
#pragma unroll
                for (int i = 0; i < TAPS; ++i) wx[i] = __ldg(p.xw + c * TAPS + i);
#pragma unroll
                for (int j = 0; j < TAPS; ++j) {
                    float v[TAPS];
#pragma unroll
                    for (int i = 0; i < TAPS; ++i) v[i] = __ldg(rows[j] + cx[i]);
                    h[j] = taps_sum<TAPS>(v, wx);
                }
                out[k] = taps_sum<TAPS>(h, wy);
            }
        }
        float* dst = p.y + (size_t)r * p.ow + ox0;
        if (VEC)
            *reinterpret_cast<float4*>(dst) = make_float4(out[0], out[W > 1 ? 1 : 0], out[W > 2 ? 2 : 0], out[W > 3 ? 3 : 0]);
        else
            dst[0] = out[0];
    }
}

template <int TAPS>
cudaError_t launch_taps(const InterpF32Params& p, bool vec, int grid, cudaStream_t s) {
    if (vec)
        interp_f32_kernel<TAPS, true><<<grid, kInterpThreads, 0, s>>>(p);
    else
        interp_f32_kernel<TAPS, false><<<grid, kInterpThreads, 0, s>>>(p);
    return cudaGetLastError();
}

}  // namespace

bool interp_f32_vec(const InterpF32Params& p) { return p.ow % 4 == 0 && ((uintptr_t)p.y & 15) == 0; }

// one thread per column group up to 16 CTAs of 256 threads per SM (two full waves); beyond that the grid-stride loop
void interp_f32_grid(const InterpF32Params& p, bool vec, int sm_count, int* grid, int* row_groups) {
    *row_groups = vec ? p.ow / 4 : p.ow;
    const long long groups = (long long)p.planes * p.oh * *row_groups;
    const long long cap = 16LL * (sm_count > 0 ? sm_count : 1);
    *grid = (int)std::min(cap, (groups + kInterpThreads - 1) / kInterpThreads);
}

cudaError_t launch_interp_f32(const InterpF32Params& p, int sm_count, cudaStream_t s) {
    const bool vec = interp_f32_vec(p);
    int grid = 0, row_groups = 0;
    interp_f32_grid(p, vec, sm_count, &grid, &row_groups);
    if (grid <= 0) return cudaErrorInvalidValue;
    cudaError_t e;
    switch (p.taps) {
        case 1: e = launch_taps<1>(p, vec, grid, s); break;
        case 2: e = launch_taps<2>(p, vec, grid, s); break;
        case 4: e = launch_taps<4>(p, vec, grid, s); break;
        default: return cudaErrorInvalidValue;
    }
    ++g_launch_count;
    return e;
}

}  // namespace mnnb200
