// common.cuh -- small device helpers shared by the sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <atomic>

namespace mnnb200 {

constexpr int kPack = 16;  // INT8_PACK_NUMBER: channel padding of the device NHWC16 layout
__host__ __device__ inline int up16(int c) { return (c + 15) & ~15; }

// ---------------------------------------------------------------------------------------------
// The reference CPU epilogue, bit for bit (x86_x64/avx512/GemmInt8_VNNI.cpp:27-39 POSTTREAT and the
// scale/bias sequence :262-392): int32 -> fp32 (rn), * wscale, * scaleX, + biasFloat, min, max,
// +-0.5, truncate.  Every step is an explicitly-rounded intrinsic so ptxas cannot contract into FMA.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int requant_cpu_exact(int acc_u, float wscale, float scale_x, float bias_float,
                                                 float minv, float maxv) {
    float f = __fmul_rn(__int2float_rn(acc_u), wscale);
    f = __fmul_rn(f, scale_x);
    f = __fadd_rn(f, bias_float);
    f = fminf(f, maxv);
    f = fmaxf(f, minv);
    f = __fadd_rn(f, f < 0.0f ? -0.5f : 0.5f);
    return __float2int_rz(f);
}

// FloatToInt8 as the AVX512 build of the reference executes it (x86_x64/avx512/GemmInt8.cpp:234-283, _AVX512_MNNFloat2Int8):
// the source says mul then add, but that directory is compiled with -mfma (x86_x64/CMakeLists.txt:59,69) and GCC's default
// -ffp-contract=fast fuses the pair: the shipped kernel is vfmadd132ps (checked in the disassembly of the reference library built by the test recipe and
// on a 1-in-4.8M input of the batch-32 MobileNet run).  fma(x, inv_scale, zero), clamp, +-0.5, truncate.
__device__ __forceinline__ int quant_avx512_exact(float x, float inv_scale, float zero, float minv, float maxv) {
    float f = __fmaf_rn(x, inv_scale, zero);
    f = fminf(f, maxv);
    f = fmaxf(f, minv);
    f = __fadd_rn(f, f < 0.0f ? -0.5f : 0.5f);
    return __float2int_rz(f);
}

// The same cast WITHOUT fusion: the AVX2 kernels (x86_x64/avx/, compiled without -mfma) that the int8 Winograd oracle build uses:
// x*inv_scale + zero (two roundings), clamp, +-0.5, truncate
__device__ __forceinline__ int quant_cpu_exact(float x, float inv_scale, float zero, float minv, float maxv) {
    float f = __fmul_rn(x, inv_scale);
    f = __fadd_rn(f, zero);
    f = fminf(f, maxv);
    f = fmaxf(f, minv);
    f = __fadd_rn(f, f < 0.0f ? -0.5f : 0.5f);
    return __float2int_rz(f);
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
    int sz = valid ? 16 : 0;  // src-size 0 => 16 bytes of zero fill
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(dst), "l"(src), "r"(sz));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

__device__ __forceinline__ void ldmatrix_x4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
                 : "r"(addr));
}

// D(16x8,s32) += A(16x32,s8,row) * B(32x8,s8,col)
__device__ __forceinline__ void mma_s8_16832(int (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ int4 ld_nc_16(const void* p) {
    int4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}

extern __attribute__((visibility("default"))) std::atomic<unsigned long long> g_launch_count;  // host-side counter (capi.cu); any thread may launch

}  // namespace mnnb200
