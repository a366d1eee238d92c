// exec.h -- what the C ABI's execution entry points share across libmnn_b200.so and libmnn_b200_llm.so: the runtime and
// execution structs behind the opaque handles of include/mnn_b200.h, the execution type tags, the device-buffer owner and the
// error reporting of mnnb200_last_error.  A handle made by either library is destroyed by mnnb200_exec_destroy (virtual
// destructor) and refused by the other library's entry points (its type tag).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <memory>
#include <string>
#include <vector>

#include "../../include/mnn_b200.h"

// the few internal symbols libmnn_b200.so exports to libmnn_b200_llm.so (everything else stays hidden)
#define MNNB200_INTERNAL __attribute__((visibility("default")))

// Sets the message mnnb200_last_error returns and passes the status through (capi.cu)
namespace mnnb200 {
MNNB200_INTERNAL mnnb200_status fail(mnnb200_status s, const std::string& m);
// row-major int8 matrix [rows][k] -> 2D tensor map with a {128 bytes, box_rows} box, 128B swizzle, zero OOB fill (capi.cu)
MNNB200_INTERNAL mnnb200_status make_tmap_i8(CUtensorMap* m, const void* ptr, int rows, int k, int box_rows);
}
#define CK(call)                                                                                   \
    do {                                                                                           \
        cudaError_t _e = (call);                                                                   \
        if (_e != cudaSuccess) {                                                                   \
            cudaGetLastError(); /* do not leave it for an unrelated cudaGetLastError() to report */ \
            return mnnb200::fail(MNNB200_CUDA_ERROR, std::string(#call) + ": " + cudaGetErrorString(_e)); \
        }                                                                                          \
    } while (0)

struct mnnb200_runtime {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    cudaDeviceProp prop;
    cudaEvent_t ev_begin = nullptr, ev_end = nullptr;   // onGetLastGpuTimeMs
    bool ev_valid = false;
};

// One device allocation, owned by the execution (or conv group) that holds it and freed with it.  Zero elements allocate 16
// bytes, so every buffer has an address.  It converts to T* where a kernel's parameter block takes the pointer.
template <class T>
class DevBuf {
  public:
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { reset(); }
    operator T*() const { return p_; }
    // grow-only: a new allocation only when n elements do not fit.  The old one is released then (cudaFree waits for the
    // device, so kernels still reading it have finished): repeated resizes do not accumulate device memory.
    mnnb200_status reserve(size_t n) {
        if (p_ && n <= cap_) return MNNB200_OK;
        void* q = nullptr;
        CK(cudaMalloc(&q, n ? n * sizeof(T) : 16));
        reset();
        p_ = static_cast<T*>(q);
        cap_ = n;
        return MNNB200_OK;
    }
    // reserve(h.size()), then copy h to the front of the buffer and wait for the copy: h may be a temporary
    mnnb200_status upload(const std::vector<T>& h, cudaStream_t s) {
        if (mnnb200_status st = reserve(h.size())) return st;
        if (!h.empty()) CK(cudaMemcpyAsync(p_, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice, s));
        CK(cudaStreamSynchronize(s));
        return MNNB200_OK;
    }
    void reset() {
        if (p_) cudaFree(p_);
        p_ = nullptr;
        cap_ = 0;
    }

  private:
    T* p_ = nullptr;
    size_t cap_ = 0;
};

// The execution types, one bit each: a handle is tested against the types an entry point takes before it is cast (exec_as).
enum ExecType : unsigned {
    kConvInt8 = 1u << 0, kDwConvInt8 = 1u << 1, kLinearW8 = 1u << 2, kWinoInt8 = 1u << 3, kMatMul = 1u << 4,
    kConvGroup = 1u << 5, kScaleInt8 = 1u << 6, kConvF32 = 1u << 7, kDwConvF32 = 1u << 8, kScaleF32 = 1u << 9,
    kLayerNormF32 = 1u << 10, kRoPEF32 = 1u << 11, kDeconvF32 = 1u << 12, kDwDeconvF32 = 1u << 13,
    kInterpF32 = 1u << 14, kGather = 1u << 15, kScatter = 1u << 16, kRnn = 1u << 17,
    kGridSampleF32 = 1u << 18, kGru = 1u << 19,
};
struct mnnb200_exec {
    unsigned type = 0;  // the ExecType of the struct new_exec made
    mnnb200_runtime* rt = nullptr;
    int variant = 0;  // mnnb200_conv_int8_set_variant: 0 auto, 1 mma.sync implicit GEMM (conv), 2 wgmma, 3 CTA pair, 4 GEMV (linear)
    bool resized = false;
    double cost_bytes = 0, cost_macs = 0;
    virtual ~mnnb200_exec() = default;
};
// An execution struct derives from Tagged<its ExecType, its base>.
template <unsigned Type, class Base = mnnb200_exec>
struct Tagged : Base {
    static constexpr unsigned kTypes = Type;
};
template <class T>
inline std::unique_ptr<T> new_exec(mnnb200_runtime* rt) {
    auto e = std::make_unique<T>();
    e->type = T::kTypes;
    e->rt = rt;
    return e;
}
// The handle as a T, or null for a NULL handle or a handle of a type outside `types`.  A tag compare rather than
// dynamic_cast: nothing depends on RTTI across the library's hidden symbols.
template <class T>
inline T* exec_as(mnnb200_exec* ex, unsigned types = T::kTypes) {
    return ex && (ex->type & types) ? static_cast<T*>(ex) : nullptr;
}

// The convolutions: the descriptor that set_pad edits.
struct ConvExec : mnnb200_exec {
    mnnb200_conv_desc d;
};
inline bool conv_desc_valid(const mnnb200_conv_desc* d) {
    return d->ic > 0 && d->oc > 0 && d->kh > 0 && d->kw > 0 && d->stride_h > 0 && d->stride_w > 0 && d->dilate_h > 0 &&
           d->dilate_w > 0 && d->pad_h >= 0 && d->pad_w >= 0;
}
// the activation code of the float convolutions' epilogues: 0 none, 1 ReLU, 2 ReLU6
inline int float_act(const mnnb200_conv_desc* d, int relu6) { return relu6 ? 2 : (d->relu ? 1 : 0); }
// a plan query: the first `count` (at most N) of the plan's fields go to `fields`
template <size_t N>
inline mnnb200_status copy_fields(const int (&v)[N], int* fields, int count) {
    for (int i = 0; i < count && i < (int)N; ++i) fields[i] = v[i];
    return MNNB200_OK;
}
