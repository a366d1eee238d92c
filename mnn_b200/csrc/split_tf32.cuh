// split_tf32.cuh -- what the split-TF32 wgmma kernels (conv_f32_wgmma.cu, deconv_f32_wgmma.cu, gemm_f16_wgmma.cu) share: the
// 128-row tile and its stage layout, the TF32 rounding and split, the 4-byte cp.async gather of the activation tile and the
// register-A wgmma m64nNk8 tf32.
#pragma once
#include <cuda.h>
#include "common.cuh"
#include "hopper_common.cuh"

namespace mnnb200 {
namespace hop {

constexpr int kBM = 128, kBK = 32 /* floats = 128 bytes */, kLdA = kBM + 8 /* conflict-free fragment reads */, kMaxStages = 8;
constexpr int kLoaderThreads = 128;
constexpr int kConvThreads = kConsumerThreads + kLoaderThreads;

template <int BN>
struct Layout {
    static constexpr int b_bytes = BN * kBK * 4;                         // one weight tile (hi or lo), 128B-swizzled rows
    static constexpr int a_bytes = kBK * kLdA * 4;
    static constexpr int stage_bytes = (2 * b_bytes + a_bytes + 1023) & ~1023;
    static constexpr int stages_fit = (227 * 1024 - 1024 - 256) / stage_bytes;
    static constexpr int stages = stages_fit > kMaxStages ? kMaxStages : stages_fit;
    static constexpr int smem = stages * stage_bytes + 1024 + 256;
};

__device__ __forceinline__ uint32_t tf32_rna(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(r) : "f"(x));
    return r;
}
// x = hi + lo, both TF32, for a_hi*b_hi + a_hi*b_lo + a_lo*b_hi: hi = tf32_rna(x), lo = tf32_rna(x - hi), |x - hi - lo| <=
// 2^-22 |x|.  A finite x that rounds past FLT_MAX (|x| >= (2 - 2^-11) 2^127) truncates instead, so both parts stay finite.
// A non-finite x goes whole into lo, with hi = 0 (tf32_rna(x - hi) would be NaN for an infinity): of the three products only
// x_lo * partner_hi then sees it, and partner_hi is 0 only when the partner is 0 and has the partner's sign, so Inf * b is what
// fp32 makes of it for every finite b (Inf * Inf is NaN: each infinity meets the other's hi part, 0).  A NaN keeps its sign
// with every mantissa bit set: its payload may lie only in the 13 bits TF32 drops, which would read as an infinity.  (The
// MatMul's operand pack; the convolutions split their own way.)
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
    if (!isfinite(x)) {
        hi = 0.f;
        lo = isnan(x) ? __int_as_float(__float_as_int(x) | 0x7fffffff) : x;
        return;
    }
    uint32_t h = tf32_rna(x);
    if ((h & 0x7f800000u) == 0x7f800000u) h = __float_as_uint(x) & 0xffffe000u;
    hi = __uint_as_float(h);
    lo = __uint_as_float(tf32_rna(x - hi));
}
__device__ __forceinline__ void cp_async4(uint32_t dst, const void* src, int src_bytes) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;\n" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
// arrives on bar once every cp.async this thread issued before has landed (counts as one of the barrier's expected arrivals)
__device__ __forceinline__ void cp_async_arrive_noinc(uint32_t bar) {
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];\n" ::"r"(bar) : "memory");
}

// wgmma m64nNk8 tf32 with A from registers: a[0..3] = A[r][q], A[r + 8][q], A[r][q + 4], A[r + 8][q + 4] with r = 16 * (warp % 4) +
// lane / 4, q = lane % 4 (the per-warp layout of mma.m16n8k8.tf32); B K-major in shared memory.
template <int N>
__device__ __forceinline__ void wgmma_rs(float* d, const uint32_t (&a)[4], uint64_t b, int scale_d);
template <> __device__ __forceinline__ void wgmma_rs<32>(float* d, const uint32_t (&a)[4], uint64_t b, int scale_d) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %21, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_rs<64>(float* d, const uint32_t (&a)[4], uint64_t b, int scale_d) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_rs<128>(float* d, const uint32_t (&a)[4], uint64_t b, int scale_d) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %69, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(scale_d));
}

}  // namespace hop
}  // namespace mnnb200
