// b200_plugin.cpp -- the drop-in: an MNN RuntimeCreator / Runtime / Backend / Execution set registered under
// MNN_FORWARD_CUDA, written against the reference's UNCHANGED plugin surface (source/core/Backend.hpp:89-457,
// source/core/Execution.hpp:24-135) and calling only the C ABI of libmnn_b200.so (include/mnn_b200.h).
//
// It plays the roles of source/backend/cuda/Register.cpp (registration), core/runtime/CUDARuntime.cpp (device, stream),
// core/CUDABackend.cpp (creator map, onAcquire, onCopyBuffer) and the execution/int8/*Execution.cu host classes, but it is
// not a translation of them: device tensors use the layouts of mnn_b200.h (int8 = NHWC16, everything else = the tensor's
// linear NCHW/NHWC layout, so Raster regions apply directly), memory is a per-backend free-list over cudaMalloc, and every
// kernel is the sm_90a code behind the C ABI.  Built here (needs the reference headers) by build_plugin.py; the GPU box
// runs the prebuilt .so next to the reference's libMNN.so.
//
// An op this file has no execution for returns nullptr from onCreate, which is the reference's documented way to say "not
// here" (Backend.hpp:163-167): MNN's pipeline then places that op on its backup backend.  For the models of BASELINE.json
// (int8 MobileNet-v2 / ResNet-50) every command is created here -- tests/test_plugin.py asserts the backup backend ran nothing.
#include <MNN/ErrorCode.hpp>
#include <MNN/MNNForwardType.h>
#define MNN_USER_SET_DEVICE
#include <MNN/MNNSharedContext.h>
#include <MNN/Tensor.hpp>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <mutex>
#include <set>
#include <thread>
#include <vector>

#include "MNN_generated.h"
#include "core/Backend.hpp"
#include "core/ConvolutionCommon.hpp"
#include "core/Execution.hpp"
#include "core/Macro.h"
#include "core/OpCommonUtils.hpp"
#include "core/TensorUtils.hpp"

#include "../../../include/mnn_b200_deconv.h"
#include "../../../include/mnn_b200_gather.h"
#include "../../../include/mnn_b200_scatter.h"
#include "../../../include/mnn_b200_rnn.h"
#include "../../../include/mnn_b200_interp.h"
#include "../../../include/mnn_b200_grid_sample.h"
#include "../../../include/mnn_b200_llm.h"

namespace MNN {
namespace {

int g_created = 0, g_declined = 0;   // commands placed here / handed back to the pipeline (read by the test harness)

inline int up16(int c) { return (c + 15) / 16 * 16; }

struct Dims4 { int n = 1, c = 1, h = 1, w = 1; };
// logical (N, C, H, W) of a tensor; extra trailing dims fold into W
Dims4 dims4(const Tensor* t) {
    Dims4 d;
    const int nd = t->dimensions();
    if (nd == 0) return d;
    auto fmt = TensorUtils::getDescribe(t)->dimensionFormat;
    d.n = t->length(0);
    if (fmt == MNN_DATA_FORMAT_NHWC && nd > 2) {
        d.c = t->length(nd - 1);
        d.h = t->length(1);
        for (int i = 2; i < nd - 1; ++i) d.w *= t->length(i);
    } else {
        if (nd > 1) d.c = t->length(1);
        if (nd > 2) d.h = t->length(2);
        for (int i = 3; i < nd; ++i) d.w *= t->length(i);
    }
    return d;
}
inline bool isInt8(const Tensor* t) {
    auto des = TensorUtils::getDescribe(t);
    return (des->quantAttr.get() != nullptr && des->applyQuant) || t->getType().bytes() == 1;
}
inline size_t elemCount(const Tensor* t) {
    size_t n = 1;
    for (int i = 0; i < t->dimensions(); ++i) n *= (size_t)t->length(i);
    return n;
}
// bytes of the DEVICE copy of a tensor (the role of CUDABackend::realSize * getBytes, core/CUDABackend.cpp:188-263)
size_t deviceBytes(const Tensor* t) {
    if (isInt8(t)) {
        auto d = dims4(t);
        return mnnb200_nhwc16_bytes(d.n, d.c, d.h, d.w);
    }
    return elemCount(t) * (size_t)t->getType().bytes();
}
inline void* dev(const Tensor* t) { return (void*)(uintptr_t)t->deviceId(); }

// The one owner of a C ABI execution: destroyed exactly once, with the execution that holds it
struct ExecDeleter { void operator()(mnnb200_exec* h) const { mnnb200_exec_destroy(h); } };
typedef std::unique_ptr<mnnb200_exec, ExecDeleter> ExecHandle;

// A grow-only scratch allocation (device or pinned host, by Alloc / Free): reallocated only when a request does not fit, the
// old allocation freed after a sync because the device may still read it; a failed allocation leaves it empty
template <mnnb200_status (*Alloc)(mnnb200_runtime*, size_t, void**), mnnb200_status (*Free)(mnnb200_runtime*, void*)>
class Scratch {
public:
    explicit Scratch(mnnb200_runtime* h) : mH(h) {}
    Scratch(const Scratch&) = delete;
    Scratch& operator=(const Scratch&) = delete;
    ~Scratch() { release(); }
    void* get(size_t bytes) {
        if (bytes > mBytes) {
            release();
            if (Alloc(mH, bytes, &mP) != MNNB200_OK) { mP = nullptr; return nullptr; }
            mBytes = bytes;
        }
        return mP;
    }
    void* data() const { return mP; }
private:
    void release() {
        if (mP) { mnnb200_runtime_sync(mH); Free(mH, mP); mP = nullptr; mBytes = 0; }
    }
    mnnb200_runtime* mH;
    void* mP = nullptr;
    size_t mBytes = 0;
};
typedef Scratch<mnnb200_alloc, mnnb200_free> DeviceScratch;
typedef Scratch<mnnb200_alloc_host, mnnb200_free_host> PinnedScratch;

class B200Runtime;

// ------------------------------------------------------------------------------------------------ Backend
class B200Exec;

class B200Backend : public Backend {
public:
    B200Backend(const B200Runtime* rt, mnnb200_runtime* h, bool memoryLow)
        : Backend(MNN_FORWARD_CUDA), mRuntime(rt), mH(h), mMemoryLow(memoryLow), mStageDev(h), mStageHost(h) {
        if (const char* v = getenv("MNNB200_PLUGIN_GRAPH")) mGraphEnabled = atoi(v) != 0;
        if (const char* v = getenv("MNNB200_PLUGIN_HOSTREG")) mHostRegEnabled = atoi(v) != 0;
    }
    bool memoryLow() const { return mMemoryLow; }
    ~B200Backend() override {
        mnnb200_runtime_sync(mH);
        dropGraph();
        for (auto& kv : mRegistered) mnnb200_host_unregister(mH, kv.first);
        freePool();
    }
    mnnb200_runtime* handle() const { return mH; }

    Execution* onCreate(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs, const MNN::Op* op) override;
    void onResizeBegin() override { dropGraph(); }
    ErrorCode onResizeEnd() override { dropGraph(); return NO_ERROR; }
    const Runtime* getRuntime() override;

    // ---- one forward = onExecuteBegin, Execution::onExecute x N, onExecuteEnd (Pipeline::execute, source/core/Pipeline.cpp:1167-1230).
    //      Run 1 after a resize executes eagerly (module load, descriptor creation).  From run 2 on the executions only LOG
    //      their call (DEFER); onExecuteEnd then
    //        - first time: captures the logged calls, each with its own kernel launches, into a CUDA graph;
    //        - afterwards: checks that the logged forward is the captured one and launches the graph (one host call per forward).
    //      Anything that needs the device mid-run (Tensor::copyToHostTensor from a callback, a command on the CPU backup backend
    //      reading a device tensor) calls interrupt(): the deferred calls are flushed eagerly and the run goes on eagerly.
    enum Mode { EAGER = 0, DEFER = 1 };
    struct Call { B200Exec* exec; const std::vector<Tensor*>* in; const std::vector<Tensor*>* out; uint64_t sig; };
    void onExecuteBegin() const override;
    void onExecuteEnd() const override;
    bool deferring() const { return mInRun && mMode == DEFER; }
    void log(B200Exec* e, const std::vector<Tensor*>& in, const std::vector<Tensor*>& out) const {
        uint64_t sig = (uint64_t)(uintptr_t)e * 1000003ull;
        for (auto t : in) sig = sig * 1099511628211ull + t->deviceId();
        for (auto t : out) sig = sig * 1099511628211ull + t->deviceId();
        mPending.push_back({e, &in, &out, sig});
    }
    void interrupt() const;
    bool buildAndCapture() const;
    void dropGraph() const {
        if (mGraph) { mnnb200_runtime_sync(mH); mnnb200_graph_destroy(mGraph); mGraph = nullptr; }
        mRuns = 0; mGraphBroken = false; mTrace.clear(); mPending.clear();
    }

    // ---- memory: STATIC = own cudaMalloc, freed with the MemObj; DYNAMIC = free-list reuse inside one resize plan,
    //      everything returned to the driver at onClearBuffer (Backend.hpp StorageType contract)
    struct Chunk { void* ptr; size_t bytes; bool free; };
    struct PoolState { std::vector<Chunk> chunks; int epoch = 0; };   // outlives the backend if a MemObj does
    class StaticMem : public Backend::MemObj {
    public:
        StaticMem(mnnb200_runtime* h, void* p) : mH(h), mP(p) {}
        ~StaticMem() override { mnnb200_runtime_sync(mH); mnnb200_free(mH, mP); }
    private:
        mnnb200_runtime* mH; void* mP;
    };
    class DynamicMem : public Backend::MemObj {
    public:
        DynamicMem(std::shared_ptr<PoolState> s, int idx, int epoch) : mS(s), mIdx(idx), mEpoch(epoch) {}
        ~DynamicMem() override { if (mEpoch == mS->epoch) mS->chunks[mIdx].free = true; }
    private:
        std::shared_ptr<PoolState> mS; int mIdx; int mEpoch;
    };
    MemObj* onAcquire(const Tensor* tensor, StorageType storageType) override {
        size_t bytes = deviceBytes(tensor);
        bytes = (bytes + 255) & ~(size_t)255;
        if (bytes == 0) bytes = 256;
        void* p = nullptr;
        if (storageType == STATIC) {
            if (mnnb200_alloc(mH, bytes, &p) != MNNB200_OK) return nullptr;
            const_cast<Tensor*>(tensor)->buffer().device = (uint64_t)(uintptr_t)p;
            return new StaticMem(mH, p);
        }
        auto& ch = mPool->chunks;
        int best = -1;
        if (storageType == DYNAMIC) {
            for (int i = 0; i < (int)ch.size(); ++i)
                if (ch[i].free && ch[i].bytes >= bytes && (best < 0 || ch[i].bytes < ch[best].bytes)) best = i;
        }
        if (best < 0) {
            if (mnnb200_alloc(mH, bytes, &p) != MNNB200_OK) return nullptr;
            ch.push_back({p, bytes, false});
            best = (int)ch.size() - 1;
        }
        ch[best].free = false;
        const_cast<Tensor*>(tensor)->buffer().device = (uint64_t)(uintptr_t)ch[best].ptr;
        if (storageType != DYNAMIC) return new DynamicMem(mPool, best, -1);   // never reused before onClearBuffer
        return new DynamicMem(mPool, best, mPool->epoch);
    }
    bool onClearBuffer() override {
        dropGraph();
        mnnb200_runtime_sync(mH);
        freePool();
        return true;
    }
    // every dynamic chunk back to the driver; a DynamicMem that outlives this sees the new epoch and leaves the list alone
    void freePool() {
        for (auto& c : mPool->chunks) mnnb200_free(mH, c.ptr);
        mPool->chunks.clear();
        ++mPool->epoch;
    }
    void onCopyBuffer(const Tensor* src, const Tensor* dst) const override;
    int onSync(Tensor::MapType, bool toCpu, const Tensor*) override {
        interrupt();
        if (toCpu) mnnb200_runtime_sync(mH);
        return 0;
    }

    // ---- staging for onCopyBuffer: one grow-only device scratch + one grow-only pinned host scratch per backend (no
    //      malloc/free per copy), and the user's own host tensors pinned in place on first sight (cudaHostRegister) so that
    //      the H2D/D2H DMA runs at PCIe speed instead of through the driver's pageable-memory bounce buffers
    void* stageDev(size_t bytes) const {
        void* p = mStageDev.get(bytes);
        if (!p) MNN_ERROR("mnn_b200: staging alloc of %zu bytes failed: %s\n", bytes, mnnb200_last_error());
        return p;
    }
    void* stageHost(size_t bytes) const {
        void* p = mStageHost.get(bytes);
        if (!p) MNN_ERROR("mnn_b200: pinned staging alloc failed: %s\n", mnnb200_last_error());
        return p;
    }
    // true when [p, p+bytes) is pinned (registered now or before); copies below 1 MiB are not worth a registration.
    // OFF by default (MNNB200_PLUGIN_HOSTREG=1 opts in): the backend cannot see a user tensor die.  A host tensor that is freed
    // and re-allocated at the same address leaves a stale registration behind; usually the next cudaMemcpyAsync on it fails with
    // "invalid argument" (h2d()/d2h() then drop the entry and redo the copy unpinned), but one batch-32 run with hundreds of
    // short-lived host tensors returned a wrong tensor instead -- so only an application that keeps its input / output host
    // tensors alive for the session's lifetime should turn it on (1.0 ms instead of 1.6 ms per batch-32 runSession).
    bool pinned(void* p, size_t bytes) const {
        if (!mHostRegEnabled || bytes < (1u << 20)) return false;
        auto it = mRegistered.find(p);
        if (it != mRegistered.end()) {
            if (it->second >= bytes) return true;
            mnnb200_host_unregister(mH, p);
            mRegistered.erase(it);
        }
        if (mRegistered.size() >= 16) {   // bounded: forget the oldest entries rather than pin without limit
            for (auto& kv : mRegistered) mnnb200_host_unregister(mH, kv.first);
            mRegistered.clear();
        }
        if (mnnb200_host_register(mH, p, bytes) != MNNB200_OK) return false;
        mRegistered[p] = bytes;
        return true;
    }
    // host -> device, returns after the host memory has been read (the caller may reuse it).  A pinned (registered) user tensor
    // is read by DMA at PCIe speed; anything else goes through the driver's pageable path (measured for the 19 MB batch-32 input:
    // 0.45 ms registered vs 1.3 ms pageable; a pool of host threads copying into a pinned staging buffer was slower than both).
    bool h2d(void* devDst, const void* hostSrc, size_t bytes) const {
        if (pinned(const_cast<void*>(hostSrc), bytes)) {
            if (mnnb200_memcpy_h2d(mH, devDst, hostSrc, bytes) == MNNB200_OK) return mnnb200_runtime_sync(mH) == MNNB200_OK;
            unpin(const_cast<void*>(hostSrc));
        }
        if (mnnb200_memcpy_h2d(mH, devDst, hostSrc, bytes) != MNNB200_OK) return false;
        return mnnb200_runtime_sync(mH) == MNNB200_OK;
    }
    bool d2h(void* hostDst, const void* devSrc, size_t bytes) const {
        if (pinned(hostDst, bytes)) {
            if (mnnb200_memcpy_d2h(mH, hostDst, devSrc, bytes) == MNNB200_OK) return mnnb200_runtime_sync(mH) == MNNB200_OK;
            unpin(hostDst);
        }
        void* st = stageHost(bytes);
        if (!st) return false;
        if (mnnb200_memcpy_d2h(mH, st, devSrc, bytes) != MNNB200_OK || mnnb200_runtime_sync(mH) != MNNB200_OK) return false;
        ::memcpy(hostDst, st, bytes);
        return true;
    }
    // a pinned copy that failed: the registration is stale (the tensor was freed and its address reused), the copy failed
    // cleanly, and the caller redoes it unpinned
    void unpin(void* p) const {
        mnnb200_host_unregister(mH, p);
        mRegistered.erase(p);
    }
    float lastGpuMs() const { return mnnb200_runtime_last_gpu_ms(mH); }

private:
    const B200Runtime* mRuntime;
    mnnb200_runtime* mH;
    bool mMemoryLow;
    std::shared_ptr<PoolState> mPool{new PoolState};
    bool mGraphEnabled = true, mHostRegEnabled = false;   // MNNB200_PLUGIN_HOSTREG=1: pin user tensors in place (see pinned())
    mutable bool mInRun = false, mGraphBroken = false;
    mutable Mode mMode = EAGER;
    mutable int mRuns = 0;
    mutable mnnb200_graph* mGraph = nullptr;
    mutable std::vector<Call> mPending;
    mutable std::vector<uint64_t> mTrace;   // signature of the captured forward
    mutable DeviceScratch mStageDev;
    mutable PinnedScratch mStageHost;
    mutable std::map<void*, size_t> mRegistered;
};

// Every execution of this plugin: onExecute either launches (eager) or only logs the call (deferred: plan / graph replay)
class B200Exec : public Execution {
public:
    explicit B200Exec(Backend* bn) : Execution(bn) {}
    ErrorCode onExecute(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) final {
        if (owner()->deferring()) { owner()->log(this, inputs, outputs); return NO_ERROR; }
        return launch(inputs, outputs);
    }
    virtual ErrorCode launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) = 0;
protected:
    B200Backend* owner() const { return static_cast<B200Backend*>(backend()); }
    mnnb200_runtime* rt() const { return owner()->handle(); }
};

// Execution::onClone (source/core/Execution.hpp:63) for an execution that T::create(backend, op) makes from the op alone.  A clone
// makes its weights again from the op: the C ABI keeps the launch plan and epilogue constants per execution and has no way to
// share its device weights.  dst == nullptr asks whether the execution can be cloned.
template <class T>
class ClonedFromOp : public B200Exec {
public:
    explicit ClonedFromOp(Backend* bn) : B200Exec(bn) {}
    bool onClone(Backend* bn, const Op* op, Execution** dst) override {
        if (dst == nullptr) return true;
        *dst = T::create(static_cast<B200Backend*>(bn), op);
        return *dst != nullptr;
    }
};

void B200Backend::onExecuteBegin() const {
    mnnb200_runtime_mark_begin(mH);
    mInRun = true;
    mMode = EAGER;
    mPending.clear();
    if (mGraphEnabled && !mGraphBroken && mRuns >= 1) mMode = DEFER;
}
void B200Backend::interrupt() const {
    if (!mInRun || mMode == EAGER) return;
    mMode = EAGER;   // run the deferred calls now, the rest of this forward goes eagerly (a captured graph stays valid)
    for (auto& c : mPending) c.exec->launch(*c.in, *c.out);
    mPending.clear();
}
// Capture the logged forward: every pending call launches its own kernels into one CUDA graph.
bool B200Backend::buildAndCapture() const {
    if (mnnb200_graph_begin_capture(mH) != MNNB200_OK) return false;
    bool ok = true;
    for (auto& c : mPending) ok = ok && c.exec->launch(*c.in, *c.out) == NO_ERROR;
    mnnb200_graph* g = nullptr;
    if (mnnb200_graph_end_capture(mH, &g) != MNNB200_OK || !ok) {
        if (g) mnnb200_graph_destroy(g);
        return false;
    }
    mGraph = g;
    mTrace.clear();
    for (auto& c : mPending) mTrace.push_back(c.sig);
    return true;
}
void B200Backend::onExecuteEnd() const {
    if (mInRun && mMode == DEFER) {
        mMode = EAGER;
        bool launched = false;
        if (!mGraph) {
            if (buildAndCapture()) {
                launched = mnnb200_graph_launch(mH, mGraph) == MNNB200_OK;
            } else {
                MNN_ERROR("mnn_b200: graph capture failed (%s); this session runs eagerly\n", mnnb200_last_error());
                mGraphBroken = true;
            }
        } else {
            bool same = mPending.size() == mTrace.size();
            for (size_t i = 0; same && i < mPending.size(); ++i) same = mPending[i].sig == mTrace[i];
            if (same) {
                launched = mnnb200_graph_launch(mH, mGraph) == MNNB200_OK;
            } else {   // a different command list / different tensors than the captured forward: run eagerly, drop the graph
                mGraphBroken = true;
            }
        }
        if (!launched) {
            for (auto& c : mPending) c.exec->launch(*c.in, *c.out);
            if (mGraphBroken && mGraph) { mnnb200_runtime_sync(mH); mnnb200_graph_destroy(mGraph); mGraph = nullptr; }
        }
        mPending.clear();
    }
    mInRun = false;
    ++mRuns;
    mnnb200_runtime_mark_end(mH);
}

// host tensor <-> linear fp32/int32 device layout.  User host tensors are NCHW (Tensor::CAFFE), NHWC (TENSORFLOW) or
// NC4HW4 with pack 4 (CAFFE_C4); the device keeps NCHW-linear for NCHW/NC4HW4-format tensors and NHWC-linear for NHWC.
// Calls copy(host tensor's byte offset, linear layout's byte offset, element bytes) for every element.
template <class F>
static void forEachElement(const Tensor* host, MNN_DATA_FORMAT devFmt, F copy) {
    auto hfmt = TensorUtils::getDescribe(host)->dimensionFormat;
    const size_t bytes = host->getType().bytes();
    auto d = dims4(host);
    const size_t area = (size_t)d.h * d.w;
    auto devIndex = [&](int n, int c, size_t a) -> size_t {
        return devFmt == MNN_DATA_FORMAT_NHWC ? ((size_t)n * area + a) * d.c + c : ((size_t)n * d.c + c) * area + a;
    };
    auto hostIndex = [&](int n, int c, size_t a) -> size_t {
        if (hfmt == MNN_DATA_FORMAT_NHWC) return ((size_t)n * area + a) * d.c + c;
        if (hfmt == MNN_DATA_FORMAT_NC4HW4) return (((size_t)n * ((d.c + 3) / 4) + c / 4) * area + a) * 4 + c % 4;
        return ((size_t)n * d.c + c) * area + a;
    };
    for (int n = 0; n < d.n; ++n)
        for (int c = 0; c < d.c; ++c)
            for (size_t a = 0; a < area; ++a) copy(hostIndex(n, c, a) * bytes, devIndex(n, c, a) * bytes, bytes);
}
static MNN_DATA_FORMAT linearFormat(const Tensor* t) {
    auto f = TensorUtils::getDescribe(t)->dimensionFormat;
    return f == MNN_DATA_FORMAT_NHWC ? MNN_DATA_FORMAT_NHWC : MNN_DATA_FORMAT_NCHW;
}

static inline bool hostIsLinear(const Tensor* host, MNN_DATA_FORMAT devFmt) {
    auto hfmt = TensorUtils::getDescribe(host)->dimensionFormat;
    if (host->dimensions() <= 1) return true;
    if (hfmt == MNN_DATA_FORMAT_NC4HW4) return false;
    return hfmt == devFmt;
}

void B200Backend::onCopyBuffer(const Tensor* src, const Tensor* dst) const {
    interrupt();   // a copy in the middle of a forward needs the device state as of now
    // host side = a tensor with host memory and no device address (CUDABackend.cpp:431-432 uses deviceId() the same way)
    const bool srcDev = src->deviceId() != 0 && src->host<void>() == nullptr;
    const bool dstDev = dst->deviceId() != 0 && dst->host<void>() == nullptr;
    auto rt = mH;
    mnnb200_status st = MNNB200_OK;
    if (srcDev && dstDev) {
        if (isInt8(src) == isInt8(dst) && linearFormat(src) == linearFormat(dst)) {
            st = mnnb200_memcpy_d2d(rt, dev(dst), dev(src), deviceBytes(src));
        } else if (isInt8(src) && !isInt8(dst) && (linearFormat(dst) == MNN_DATA_FORMAT_NCHW || dst->dimensions() <= 2)) {
            auto d = dims4(src); auto q = TensorUtils::getQuantInfo(src);
            st = mnnb200_int8_to_float(rt, (const int8_t*)dev(src), d.n, d.c, d.h, d.w, q[0], q[1], (float*)dev(dst));
        } else if (!isInt8(src) && isInt8(dst) && (linearFormat(src) == MNN_DATA_FORMAT_NCHW || src->dimensions() <= 2)) {
            auto d = dims4(dst); auto q = TensorUtils::getQuantInfo(dst);
            st = mnnb200_float_to_int8(rt, (const float*)dev(src), d.n, d.c, d.h, d.w, q[0], q[1], (int)q[2], (int)q[3], (int8_t*)dev(dst));
        } else {
            // the cast kernels read/write NCHW-linear fp32: an NHWC-format float tensor of > 2 dims would be filled in the wrong layout
            MNN_ERROR("mnn_b200: device->device copy between NHWC and NCHW layouts (or a cast on an NHWC float tensor) is not supported\n");
        }
        if (st != MNNB200_OK) MNN_ERROR("mnn_b200 onCopyBuffer d2d: %s\n", mnnb200_last_error());
        return;
    }
    if (!srcDev && dstDev) {   // host -> device
        const void* from = src->host<void>();
        const size_t bytes = elemCount(src) * (size_t)src->getType().bytes();
        const auto devFmt = isInt8(dst) ? MNN_DATA_FORMAT_NCHW : linearFormat(dst);
        std::vector<uint8_t> lin;
        if (!hostIsLinear(src, devFmt)) {
            lin.assign(bytes, 0);
            forEachElement(src, devFmt, [&](size_t h, size_t l, size_t n) { ::memcpy(&lin[l], src->host<uint8_t>() + h, n); });
            from = lin.data();
        }
        if (isInt8(dst)) {
            auto d = dims4(dst);
            void* stage = stageDev(bytes);
            if (!stage || !h2d(stage, from, bytes)) { MNN_ERROR("mnn_b200 onCopyBuffer h2d failed: %s\n", mnnb200_last_error()); return; }
            if (src->getType().bytes() == 1) {   // int8 host, logical NCHW -> NHWC16
                st = mnnb200_pack_nchw_int8(rt, (const int8_t*)stage, d.n, d.c, d.h, d.w, (int8_t*)dev(dst));
            } else {                              // float host -> int8 device: the FloatToInt8 cast inside the copy
                auto q = TensorUtils::getQuantInfo(dst);
                st = mnnb200_float_to_int8(rt, (const float*)stage, d.n, d.c, d.h, d.w, q[0], q[1], (int)q[2], (int)q[3], (int8_t*)dev(dst));
            }
            // no sync here: the cast is stream-ordered before everything that follows, and the staging buffer is only rewritten
            // by a later copy on the same stream
            if (st != MNNB200_OK) MNN_ERROR("mnn_b200 onCopyBuffer cast: %s\n", mnnb200_last_error());
            return;
        }
        if (!h2d(dev(dst), from, bytes)) MNN_ERROR("mnn_b200 onCopyBuffer h2d failed: %s\n", mnnb200_last_error());
        return;
    }
    if (srcDev && !dstDev) {   // device -> host
        const void* from = dev(src);
        auto d = dims4(src);
        size_t bytes = elemCount(src) * (size_t)dst->getType().bytes();
        if (isInt8(src)) {
            void* stage = stageDev(bytes);
            if (!stage) return;
            if (dst->getType().bytes() == 1) {
                st = mnnb200_unpack_nchw_int8(rt, (const int8_t*)dev(src), d.n, d.c, d.h, d.w, (int8_t*)stage);
            } else {                              // dequantise inside the copy (core/CUDABackend.cpp:537-589)
                auto q = TensorUtils::getQuantInfo(src);
                st = mnnb200_int8_to_float(rt, (const int8_t*)dev(src), d.n, d.c, d.h, d.w, q[0], q[1], (float*)stage);
            }
            if (st != MNNB200_OK) { MNN_ERROR("mnn_b200 onCopyBuffer cast: %s\n", mnnb200_last_error()); return; }
            from = stage;
        }
        auto devFmt = isInt8(src) ? MNN_DATA_FORMAT_NCHW : linearFormat(src);
        if (hostIsLinear(dst, devFmt)) {
            if (!d2h(dst->host<void>(), from, bytes)) MNN_ERROR("mnn_b200 onCopyBuffer d2h failed: %s\n", mnnb200_last_error());
        } else {
            std::vector<uint8_t> lin(bytes);
            if (!d2h(lin.data(), from, bytes)) { MNN_ERROR("mnn_b200 onCopyBuffer d2h failed: %s\n", mnnb200_last_error()); return; }
            forEachElement(dst, devFmt, [&](size_t h, size_t l, size_t n) { ::memcpy(dst->host<uint8_t>() + h, &lin[l], n); });
        }
        return;
    }
    MNN_ERROR("mnn_b200: onCopyBuffer between two host tensors\n");
}

// ------------------------------------------------------------------------------------------------ Executions
static ErrorCode toErr(mnnb200_status s, const char* what) {
    if (s == MNNB200_OK) return NO_ERROR;
    MNN_ERROR("mnn_b200 %s: status %d: %s\n", what, s, mnnb200_last_error());
    return s == MNNB200_OUT_OF_MEMORY ? OUT_OF_MEMORY : (s == MNNB200_NOT_SUPPORT ? NOT_SUPPORT : (s == MNNB200_COMPUTE_SIZE_ERROR ? COMPUTE_SIZE_ERROR : INVALID_VALUE));
}

// Convolution / ConvolutionDepthwise / ConvInt8 / DepthwiseConvInt8 with int8 tensors (ConvInt8CutlassExecution's role)
class ConvInt8Exec : public ClonedFromOp<ConvInt8Exec> {
public:
    ConvInt8Exec(Backend* bn, const Op* op, mnnb200_exec* h, bool dw, bool wino)
        : ClonedFromOp(bn), mOp(op), mH(h), mDepthwise(dw), mWino(wino) {}
    static Execution* create(B200Backend* bn, const Op* op) {
        const bool depthwise = op->type() == OpType_ConvolutionDepthwise || op->type() == OpType_DepthwiseConvInt8;
        auto conv = op->main_as_Convolution2D();
        if (!conv || !conv->common()) return nullptr;
        auto cm = conv->common();
        const int oc = cm->outputCount(), kh = cm->kernelY(), kw = cm->kernelX();
        const int ocUp = up16(oc);
        std::vector<float> scale(2 * ocUp, 0.f);
        std::vector<int32_t> bias(ocUp, 0);
        std::shared_ptr<ConvolutionCommon::Int8Common> quanCommon;
        const int8_t* w = nullptr;
        int wsize = 0;
        // SURVEY a1: the reference's own decoder, reused through its exported symbol
        if (!ConvolutionCommon::getConvInt8Parameters(op, quanCommon, bn, w, wsize, scale.data(), bias.data(), ocUp)) return nullptr;
        if (quanCommon && quanCommon->asymmetric) return nullptr;          // asymmetric static weights: not on this path
        const bool legacy = conv->symmetricQuan() && conv->symmetricQuan()->bias() && conv->symmetricQuan()->scale();
        int ic = depthwise ? oc : cm->inputCount();
        if (!depthwise && ic <= 0) ic = wsize / (oc * kh * kw);
        mnnb200_conv_desc d;
        d.ic = ic; d.oc = oc; d.kh = kh; d.kw = kw; d.stride_h = cm->strideY(); d.stride_w = cm->strideX();
        d.pad_h = cm->padY(); d.pad_w = cm->padX(); d.dilate_h = cm->dilateY(); d.dilate_w = cm->dilateX();
        d.group = depthwise ? oc : 1; d.relu = (cm->relu() || cm->relu6()) ? 1 : 0;
        if (!depthwise && cm->group() != 1) return nullptr;
        const bool wino = !depthwise && conv->symmetricQuan() && conv->symmetricQuan()->winogradAttr();
        mnnb200_exec* h = nullptr;
        mnnb200_status st;
        if (wino) {
            auto a = conv->symmetricQuan()->winogradAttr();
            st = mnnb200_conv_int8_wino_create(bn->handle(), &d, w, scale.data(), (const float*)bias.data(), a->data(), (int)a->size(), &h);
        } else if (depthwise) {
            if (legacy) return nullptr;
            st = mnnb200_dwconv_int8_create(bn->handle(), &d, w, scale.data(), (const float*)bias.data(), &h);
        } else if (legacy) {
            st = mnnb200_conv_int8_create_legacy(bn->handle(), &d, w, scale.data(), bias.data(), &h);
        } else {
            st = mnnb200_conv_int8_create(bn->handle(), &d, w, scale.data(), (const float*)bias.data(), &h);
        }
        if (st != MNNB200_OK) {
            if (st != MNNB200_NOT_SUPPORT) MNN_ERROR("mnn_b200 conv create: %s\n", mnnb200_last_error());
            return nullptr;
        }
        return new ConvInt8Exec(bn, op, h, depthwise, wino);
    }
    ErrorCode onResize(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        auto in = inputs[0], out = outputs[0];
        auto conv = mOp->main_as_Convolution2D();
        auto pad = ConvolutionCommon::convolutionPad(in, out, conv->common());   // (padX, padY), resolves SAME/VALID
        auto qi = TensorUtils::getQuantInfo(in), qo = TensorUtils::getQuantInfo(out);
        float si = qi[0], so = qo[0];
        int zi = (int)qi[1], zo = (int)qo[1], cmin = (int)qo[2], cmax = (int)qo[3];
        if (TensorUtils::getDescribe(in)->quantAttr.get() == nullptr && conv->quanParameter()) {
            // op-carried quant info (Express-built ConvInt8, ConvInt8Winograd.cpp:316-330 / ConvInt8TiledExecutor.cpp:55-84)
            si = conv->quanParameter()->scaleIn(); so = conv->quanParameter()->scaleOut();
            if (conv->symmetricQuan()) {
                zi = conv->symmetricQuan()->zeroPoint(); zo = conv->symmetricQuan()->outputZeroPoint();
                cmin = conv->symmetricQuan()->clampMin(); cmax = conv->symmetricQuan()->clampMax();
            }
        }
        int oh = out->height(), ow = out->width();
        mnnb200_status st = mnnb200_conv_int8_set_pad(mH.get(), pad.second, pad.first);
        if (st == MNNB200_OK) {
            if (mWino) st = mnnb200_conv_int8_wino_resize(mH.get(), in->batch(), in->height(), in->width(), si, zi, so, zo, cmin, cmax, &oh, &ow);
            else if (mDepthwise) st = mnnb200_dwconv_int8_resize(mH.get(), in->batch(), in->height(), in->width(), si, zi, so, zo, cmin, cmax, &oh, &ow);
            else st = mnnb200_conv_int8_resize(mH.get(), in->batch(), in->height(), in->width(), si, zi, so, zo, cmin, cmax, &oh, &ow);
        }
        return toErr(st, "conv resize");
    }
    ErrorCode launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        auto x = (const int8_t*)dev(inputs[0]);
        auto y = (int8_t*)dev(outputs[0]);
        mnnb200_status st = mWino ? mnnb200_conv_int8_wino_execute(mH.get(), x, y)
                                  : (mDepthwise ? mnnb200_dwconv_int8_execute(mH.get(), x, y) : mnnb200_conv_int8_execute(mH.get(), x, y));
        return toErr(st, "conv execute");
    }
private:
    const Op* mOp;
    ExecHandle mH;
    bool mDepthwise, mWino;
};

// Convolution 1x1 with IDST int8 weights on FLOAT tensors under BackendConfig::Memory_Low = the MNN-LLM linear layer:
// DenseConvInt8TiledExecutor's dynamic-quant branch (compute/ConvolutionFloatFactory.cpp:139-150,
// compute/ConvInt8TiledExecutor.cpp:1990-2096) -> W8A8 on wgmma.  Tensors are [N][C][H][W] (stored NCHW-linear), the GEMM
// wants token-major rows: transposed in and out unless H*W == 1.
class LinearW8Exec : public B200Exec {
public:
    LinearW8Exec(B200Backend* bn, mnnb200_exec* h, int ic, int oc)
        : B200Exec(bn), mH(h), mIc(ic), mOc(oc), mX(bn->handle()), mY(bn->handle()) {}
    static Execution* create(B200Backend* bn, const Op* op) {
        auto conv = op->main_as_Convolution2D();
        auto cm = conv->common();
        if (cm->kernelX() != 1 || cm->kernelY() != 1 || cm->strideX() != 1 || cm->strideY() != 1 || cm->group() != 1 ||
            cm->padX() != 0 || cm->padY() != 0 || (cm->pads() && cm->pads()->size() > 0))
            return nullptr;
        auto q = ConvolutionCommon::load(op, bn, false, true);     // reference's own IDST decoder, int8 weights kept
        if (!q || q->weight.get() == nullptr) return nullptr;
        // 4-bit layers come back packed, two weights per byte (canUseInt4, ConvolutionCommon.cpp:279-307, :357-371), so the input
        // width is the op's inputCount, never weight.size() / oc; 2- and 3-bit layers stay on the CPU
        if (q->canUseInt2 || q->canUseInt3) return nullptr;
        const int oc = cm->outputCount(), ic = cm->inputCount();
        const size_t wbytes = q->canUseInt4 ? (size_t)oc * ic / 2 : (size_t)oc * ic;
        if (oc <= 0 || ic <= 0 || q->weight.size() != wbytes) return nullptr;
        const float* al = q->getAlphaFloat();
        const int per = q->asymmetric ? 2 : 1;
        // per-channel scales, or K-blocked ones (quant_block): [oc][blocks], blocks = alphaSize / (per * oc)
        if (q->alphaSize <= 0 || q->alphaSize % (per * oc) != 0) return nullptr;
        const int blocks = q->alphaSize / (per * oc);
        const size_t n = (size_t)oc * blocks;
        std::vector<float> alpha(n), wzero(n, 0.f), bias(oc, 0.f);
        for (size_t i = 0; i < n; ++i) {
            if (q->asymmetric) {   // {offset, scale}: load() has already turned the wire "min" into the offset of SIGNED int8
                                   // weights, min - clampMin * scale (ConvolutionCommon.cpp:757-766), so w = q * scale + offset
                alpha[i] = al[2 * i + 1];
                wzero[i] = al[2 * i];
            } else {
                alpha[i] = al[i];
            }
        }
        const bool hasBias = conv->bias() && (int)conv->bias()->size() == oc;
        if (hasBias) ::memcpy(bias.data(), conv->bias()->data(), sizeof(float) * oc);
        mnnb200_exec* h = nullptr;
        const mnnb200_status st =
            q->canUseInt4 ? mnnb200_linear_w4_create_blocked(bn->handle(), ic, oc, blocks, (const uint8_t*)q->weight.get(), alpha.data(),
                                                             q->asymmetric ? wzero.data() : nullptr, hasBias ? bias.data() : nullptr,
                                                             cm->relu() ? 1 : 0, cm->relu6() ? 1 : 0, &h)
                          : mnnb200_linear_w8_create_blocked(bn->handle(), ic, oc, blocks, q->weight.get(), alpha.data(),
                                                             q->asymmetric ? wzero.data() : nullptr, hasBias ? bias.data() : nullptr,
                                                             cm->relu() ? 1 : 0, cm->relu6() ? 1 : 0, &h);
        if (st != MNNB200_OK) {
            MNN_ERROR("mnn_b200 linear create: %s\n", mnnb200_last_error());
            return nullptr;
        }
        return new LinearW8Exec(bn, h, ic, oc);
    }
    ErrorCode onResize(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>&) override {
        auto d = dims4(inputs[0]);
        if (d.c != mIc) return COMPUTE_SIZE_ERROR;      // the weights were made for mIc input channels
        mN = d.n; mArea = d.h * d.w;
        const int tokens = mN * mArea;
        if (mArea > 1 && (!mX.get((size_t)tokens * mIc * 4) || !mY.get((size_t)tokens * mOc * 4))) return OUT_OF_MEMORY;
        return toErr(mnnb200_linear_w8_resize(mH.get(), tokens), "linear resize");
    }
    ErrorCode launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        if (mArea == 1) return toErr(mnnb200_linear_w8_execute(mH.get(), (const float*)dev(inputs[0]), (float*)dev(outputs[0])), "linear");
        mnnb200_status st = mnnb200_transpose_b32(rt(), dev(inputs[0]), mN, mIc, mArea, mX.data());            // [n][ic][hw] -> [n][hw][ic]
        if (st == MNNB200_OK) st = mnnb200_linear_w8_execute(mH.get(), (const float*)mX.data(), (float*)mY.data());
        if (st == MNNB200_OK) st = mnnb200_transpose_b32(rt(), mY.data(), mN, mArea, mOc, dev(outputs[0]));    // [n][hw][oc] -> [n][oc][hw]
        return toErr(st, "linear execute");
    }
private:
    ExecHandle mH;
    int mIc, mOc, mN = 0, mArea = 0;
    DeviceScratch mX, mY;   // token-major input and output when H*W > 1
};

// MatMul and BatchMatMul on float tensors (MatMulExecution.cu's role): C = op(A) op(B) (+ bias input), over the batch dims
// ShapeMatMul broadcasts (right-aligned, a dim of 1 against any) and with its squeeze of a 1-D operand: A of [l] is one row
// (transposeA ignored), B of [l] one column (transposeB ignored).  Under Compiler_Geometry the geometry stage hands every
// MatMul / BatchMatMul over unlowered (GeometryBatchMatMul is registered for Compiler_Loop only).
class MatMulExec : public B200Exec {
public:
    MatMulExec(Backend* bn, bool ta, bool tb) : B200Exec(bn), mTa(ta), mTb(tb) {}
    ErrorCode onResize(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        auto a = inputs[0], b = inputs[1];
        const int na = a->dimensions(), nb = b->dimensions();
        if (na < 1 || nb < 1) return NOT_SUPPORT;
        const bool ta = na > 1 && mTa, tb = nb == 1 || mTb;   // B of [l] is K-major [h = 1][l]
        const int e = na == 1 ? 1 : (ta ? a->length(na - 1) : a->length(na - 2));
        const int l = na == 1 ? a->length(0) : (ta ? a->length(na - 2) : a->length(na - 1));
        const int h = nb == 1 ? 1 : (tb ? b->length(nb - 2) : b->length(nb - 1));
        const int l2 = nb == 1 ? b->length(0) : (tb ? b->length(nb - 1) : b->length(nb - 2));
        if (l != l2) return COMPUTE_SIZE_ERROR;
        const int ba = std::max(na - 2, 0), bb = std::max(nb - 2, 0), nd = std::max(ba, bb);
        if (nd > 8) return NOT_SUPPORT;
        int cd[8], ad[8], bd[8];
        size_t batch = 1;
        for (int i = 0; i < nd; ++i) {
            const int ia = i - (nd - ba), ib = i - (nd - bb);
            ad[i] = ia >= 0 ? a->length(ia) : 1;
            bd[i] = ib >= 0 ? b->length(ib) : 1;
            if (ad[i] != bd[i] && ad[i] != 1 && bd[i] != 1) return NOT_SUPPORT;
            cd[i] = ad[i] == 1 ? bd[i] : ad[i];
            batch *= (size_t)cd[i];
        }
        if (batch * (size_t)e * (size_t)h != elemCount(outputs[0])) return NOT_SUPPORT;
        mH.reset();
        mnnb200_exec* m = nullptr;
        const mnnb200_status st = mnnb200_matmul_create_broadcast(rt(), nd, cd, ad, bd, e, l, h, ta, tb, &m);
        mH.reset(m);
        return toErr(st, "matmul create");
    }
    ErrorCode launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        const float* bias = inputs.size() > 2 ? (const float*)dev(inputs[2]) : nullptr;
        return toErr(mnnb200_matmul_execute(mH.get(), dev(inputs[0]), dev(inputs[1]), bias, (float*)dev(outputs[0])), "matmul");
    }
private:
    bool mTa, mTb;
    ExecHandle mH;
};

class FloatToInt8Exec : public B200Exec {
public:
    FloatToInt8Exec(Backend* bn) : B200Exec(bn) {}
    ErrorCode launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        auto d = dims4(inputs[0]);
        auto q = TensorUtils::getQuantInfo(outputs[0]);   // CPUCast.cpp:17-60: scale = 1/quant.scale, zero, min, max
        return toErr(mnnb200_float_to_int8(rt(), (const float*)dev(inputs[0]), d.n, d.c, d.h, d.w,
                                           q[0], q[1], (int)q[2], (int)q[3], (int8_t*)dev(outputs[0])), "FloatToInt8");
    }
};
class Int8ToFloatExec : public B200Exec {
public:
    Int8ToFloatExec(Backend* bn) : B200Exec(bn) {}
    ErrorCode launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        auto d = dims4(inputs[0]);
        auto q = TensorUtils::getQuantInfo(inputs[0]);
        return toErr(mnnb200_int8_to_float(rt(), (const int8_t*)dev(inputs[0]), d.n, d.c, d.h, d.w,
                                           q[0], q[1], (float*)dev(outputs[0])), "Int8ToFloat");
    }
};
class BinaryAddInt8Exec : public B200Exec {
public:
    BinaryAddInt8Exec(Backend* bn) : B200Exec(bn) {}
    ErrorCode launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        auto d = dims4(outputs[0]);
        auto q0 = TensorUtils::getQuantInfo(inputs[0]), q1 = TensorUtils::getQuantInfo(inputs[1]), qo = TensorUtils::getQuantInfo(outputs[0]);
        return toErr(mnnb200_binary_add_int8(rt(), (const int8_t*)dev(inputs[0]), q0[0], (int)q0[1],
                                             (const int8_t*)dev(inputs[1]), q1[0], (int)q1[1], (int8_t*)dev(outputs[0]), qo[0], (int)qo[1],
                                             (int)qo[2], (int)qo[3], d.n, d.c, d.h, d.w), "BinaryOp add int8");
    }
};
// kernel, stride and begin pads of a pooling window: global, SAME and VALID pooling (CPUPool.cpp:45-66, CPUPoolInt8.cpp:180-215)
struct PoolWindow { int kh, kw, sh, sw, ph, pw; };
static PoolWindow poolWindow(const Pool* p, const Tensor* in, const Tensor* out) {
    PoolWindow w = {p->kernelY(), p->kernelX(), p->strideY(), p->strideX(), p->padY(), p->padX()};
    if (p->isGlobal()) { w.kw = in->width(); w.kh = in->height(); w.sw = w.kw; w.sh = w.kh; w.pw = w.ph = 0; }
    if (p->padType() == PoolPadType_SAME) {
        int nw = (out->width() - 1) * w.sw + w.kw - in->width(), nh = (out->height() - 1) * w.sh + w.kh - in->height();
        w.pw = nw > 0 ? nw / 2 : 0; w.ph = nh > 0 ? nh / 2 : 0;
    } else if (p->padType() == PoolPadType_VALID) {
        w.pw = w.ph = 0;
    }
    return w;
}
class PoolF32Exec : public B200Exec {
public:
    PoolF32Exec(Backend* bn, const Pool* p) : B200Exec(bn), mP(p) {}
    ErrorCode launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        auto in = inputs[0], out = outputs[0];
        auto w = poolWindow(mP, in, out);
        int padType = (int)mP->padType();
        if (!mP->isGlobal() && mP->pads() != nullptr && mP->padType() == PoolPadType_CAFFE) {   // CPUPool.cpp:67-73
            if (mP->pads()->size() == 4) { w.ph = mP->pads()->data()[0]; w.pw = mP->pads()->data()[1]; }
            padType = (int)PoolPadType_VALID;   // any pads vector: DEFAULT counting then excludes the padding
        }
        return toErr(mnnb200_pool_f32(rt(), (const float*)dev(in), in->batch(), in->channel(),
                                      in->height(), in->width(), w.kh, w.kw, w.sh, w.sw, w.ph, w.pw, padType, (int)mP->countType(),
                                      mP->type() == PoolType_AVEPOOL ? 1 : 0, (float*)dev(out), out->height(), out->width()), "Pooling");
    }
private:
    const Pool* mP;
};
// int8 Scale (CPUScaleInt8's role): per-channel fixed-point scale + bias between int8 tensors
class ScaleInt8Exec : public ClonedFromOp<ScaleInt8Exec> {
public:
    ScaleInt8Exec(Backend* bn, mnnb200_exec* h) : ClonedFromOp(bn), mH(h) {}
    static Execution* create(B200Backend* bn, const Op* op) {
        auto sc = op->main_as_Scale();
        if (!sc || !sc->scaleData()) return nullptr;
        const int c = (int)sc->scaleData()->size();
        const float* bias = (sc->biasData() && (int)sc->biasData()->size() == c) ? sc->biasData()->data() : nullptr;
        mnnb200_exec* h = nullptr;
        if (mnnb200_scale_int8_create(bn->handle(), c, sc->scaleData()->data(), bias, &h) != MNNB200_OK) return nullptr;
        return new ScaleInt8Exec(bn, h);
    }
    ErrorCode onResize(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        auto qi = TensorUtils::getQuantInfo(inputs[0]), qo = TensorUtils::getQuantInfo(outputs[0]);
        return toErr(mnnb200_scale_int8_resize(mH.get(), qi[0], (int)qi[1], qo[0], (int)qo[1], (int)qo[2], (int)qo[3]), "Scale resize");
    }
    ErrorCode launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        auto d = dims4(inputs[0]);
        return toErr(mnnb200_scale_int8_execute(mH.get(), (const int8_t*)dev(inputs[0]), d.n, d.h, d.w, (int8_t*)dev(outputs[0])), "Scale int8");
    }
private:
    ExecHandle mH;
};
// int8 Pooling between tensors with equal quant attrs (CPUPoolInt8's role, x86 semantics)
class PoolInt8Exec : public B200Exec {
public:
    PoolInt8Exec(Backend* bn, const Pool* p) : B200Exec(bn), mP(p) {}
    ErrorCode launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        auto in = inputs[0], out = outputs[0];
        auto w = poolWindow(mP, in, out);
        return toErr(mnnb200_pool_int8(rt(), (const int8_t*)dev(in), in->batch(), in->channel(),
                                       in->height(), in->width(), w.kh, w.kw, w.sh, w.sw, w.ph, w.pw, mP->type() == PoolType_AVEPOOL ? 1 : 0,
                                       (int8_t*)dev(out), out->height(), out->width()), "Pooling int8");
    }
private:
    const Pool* mP;
};
class ReluF32Exec : public B200Exec {
public:
    ReluF32Exec(Backend* bn, float slope) : B200Exec(bn), mSlope(slope) {}
    ErrorCode launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        return toErr(mnnb200_relu_f32(rt(), (const float*)dev(inputs[0]), elemCount(inputs[0]), mSlope,
                                      (float*)dev(outputs[0])), "ReLU");
    }
private:
    float mSlope;
};
// Reduction over the op's one axis (ReductionParam.dim, keepDims): GeometryReduce hands a backend either the op itself when it
// reduces one axis of a non-NC4HW4 tensor, or [outside, axis, inside] views reduced over axis 1 (geometry/GeometryReduce.cpp:118-170)
class ReduceF32Exec : public B200Exec {
public:
    ReduceF32Exec(Backend* bn, int op, int axis) : B200Exec(bn), mOp(op), mAxis(axis) {}
    ErrorCode launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override;
private:
    int mOp, mAxis;
};
class SoftmaxInt8Exec : public B200Exec {
public:
    SoftmaxInt8Exec(Backend* bn) : B200Exec(bn) {}
    ErrorCode launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        auto d = dims4(inputs[0]);
        auto qi = TensorUtils::getQuantInfo(inputs[0]), qo = TensorUtils::getQuantInfo(outputs[0]);
        return toErr(mnnb200_softmax_int8(rt(), (const int8_t*)dev(inputs[0]), d.n, d.c, qi[0], qi[1],
                                          qo[0], qo[1], (int)qo[2], (int)qo[3], (int8_t*)dev(outputs[0])), "Softmax int8");
    }
};
class RasterExec : public B200Exec {
public:
    RasterExec(Backend* bn) : B200Exec(bn) {}
    ErrorCode onResize(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        // the pipeline may have replaced inputs by cast / wrapped tensors: re-point the regions (every reference backend's
        // Raster does this first, e.g. backend/cpu/CPURaster.cpp:400, backend/cuda/execution/RasterExecution.cpp:107)
        OpCommonUtils::rasterInputReset(inputs, outputs[0]);
        auto des = TensorUtils::getDescribe(outputs[0]);
        size_t covered = 0;
        for (auto& r : des->regions) covered += (size_t)r.size[0] * r.size[1] * r.size[2];
        mZero = covered < elemCount(outputs[0]);
        return NO_ERROR;
    }
    ErrorCode launch(const std::vector<Tensor*>&, const std::vector<Tensor*>& outputs) override {
        auto out = outputs[0];
        auto des = TensorUtils::getDescribe(out);
        std::vector<mnnb200_region> regs;
        for (auto& r : des->regions) {
            mnnb200_region g;
            g.src = dev(r.origin);
            g.src_offset = r.src.offset; g.dst_offset = r.dst.offset;
            for (int k = 0; k < 3; ++k) { g.src_stride[k] = r.src.stride[k]; g.dst_stride[k] = r.dst.stride[k]; g.size[k] = r.size[k]; }
            regs.push_back(g);
        }
        return toErr(mnnb200_raster_b32(rt(), regs.data(), (int)regs.size(), dev(out),
                                        elemCount(out) * 4, mZero ? 1 : 0), "Raster");
    }
private:
    bool mZero = false;
};

// ---- fp32 models: the CPU backend's float path on NCHW-linear device tensors
static bool isF32Nchw(const Tensor* t) {
    return t->getType().code == halide_type_float && t->getType().bytes() == 4 && linearFormat(t) == MNN_DATA_FORMAT_NCHW;
}
// Convolution (any group, split-TF32 wgmma) and ConvolutionDepthwise (also a Convolution whose group == ic == oc) on float
// tensors.  The group follows ConvolutionFloatFactory: common->group(), unless inputCount > 0 differs from the input's channel
// count `in_c`, when it is in_c / inputCount; group i then convolves input channels [i icg, (i+1) icg) with the weights
// [oc][icg][kh][kw], icg = wsize / (oc kh kw) = in_c / group.  A clone is made again from the op with the same input channel count.
class ConvF32Exec : public B200Exec {
public:
    ConvF32Exec(Backend* bn, const Op* op, mnnb200_exec* h, bool dw, int ic, int inC)
        : B200Exec(bn), mOp(op), mH(h), mDepthwise(dw), mIc(ic), mInC(inC) {}
    static Execution* create(B200Backend* bn, const Op* op, int inC) {
        auto conv = op->main_as_Convolution2D();
        if (!conv || !conv->common()) return nullptr;
        auto cm = conv->common();
        const int oc = cm->outputCount(), kh = cm->kernelY(), kw = cm->kernelX();
        std::shared_ptr<ConvolutionCommon::Int8Common> quanCommon;
        const float* w = nullptr;
        int wsize = 0;
        // plain float weights and IDST-coded ones, decoded as the CPU's float path does
        ConvolutionCommon::getConvParameters(&quanCommon, bn, op, &w, &wsize);
        if (!w || oc <= 0 || kh <= 0 || kw <= 0 || wsize <= 0) return nullptr;
        const bool dwOp = op->type() == OpType_ConvolutionDepthwise;
        int group = cm->group(), ic = oc;
        if (!dwOp && cm->inputCount() > 0 && cm->inputCount() != inC) group = inC / cm->inputCount();
        const bool dw = dwOp || (group > 1 && group == oc && wsize == oc * kh * kw);
        if (!dw) {
            if (group <= 0 || wsize % (oc * kh * kw)) return nullptr;
            const int icg = wsize / (oc * kh * kw);
            ic = icg * group;
            if (icg <= 0 || (group > 1 && ic != inC) || oc % group) return nullptr;
        }
        if ((size_t)wsize != (size_t)oc * (dw ? 1 : ic / group) * kh * kw) return nullptr;
        mnnb200_conv_desc d;
        d.ic = ic; d.oc = oc; d.kh = kh; d.kw = kw; d.stride_h = cm->strideY(); d.stride_w = cm->strideX();
        d.pad_h = 0; d.pad_w = 0; d.dilate_h = cm->dilateY(); d.dilate_w = cm->dilateX();   // pads: set at resize
        d.group = dw ? oc : group; d.relu = cm->relu() ? 1 : 0;
        const float* bias = (conv->bias() && (int)conv->bias()->size() == oc) ? conv->bias()->data() : nullptr;
        mnnb200_exec* h = nullptr;
        mnnb200_status st = dw          ? mnnb200_dwconv_f32_create(bn->handle(), &d, w, bias, cm->relu6() ? 1 : 0, &h)
                            : group > 1 ? mnnb200_conv_f32_create_grouped(bn->handle(), &d, w, bias, cm->relu6() ? 1 : 0, &h)
                                        : mnnb200_conv_f32_create(bn->handle(), &d, w, bias, cm->relu6() ? 1 : 0, &h);
        if (st != MNNB200_OK) {
            if (st != MNNB200_NOT_SUPPORT) MNN_ERROR("mnn_b200 float conv create: %s\n", mnnb200_last_error());
            return nullptr;
        }
        return new ConvF32Exec(bn, op, h, dw, ic, inC);
    }
    bool onClone(Backend* bn, const Op* op, Execution** dst) override {
        if (dst == nullptr) return true;
        *dst = create(static_cast<B200Backend*>(bn), op, mInC);
        return *dst != nullptr;
    }
    ErrorCode onResize(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        auto in = inputs[0], out = outputs[0];
        if (in->dimensions() != 4 || in->channel() != mIc) {   // the kernels index the input by the weights' channel count
            MNN_ERROR("mnn_b200 float conv: input has %d channels, the weights %d\n", in->channel(), mIc);
            return NOT_SUPPORT;
        }
        auto pad = ConvolutionCommon::convolutionPad(in, out, mOp->main_as_Convolution2D()->common());   // (padX, padY)
        int oh = out->height(), ow = out->width();
        mnnb200_status st = mnnb200_conv_f32_set_pad(mH.get(), pad.second, pad.first);
        if (st == MNNB200_OK)
            st = mDepthwise ? mnnb200_dwconv_f32_resize(mH.get(), in->batch(), in->height(), in->width(), &oh, &ow)
                            : mnnb200_conv_f32_resize(mH.get(), in->batch(), in->height(), in->width(), &oh, &ow);
        return toErr(st, "float conv resize");
    }
    ErrorCode launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        auto x = (const float*)dev(inputs[0]);
        auto y = (float*)dev(outputs[0]);
        return toErr(mDepthwise ? mnnb200_dwconv_f32_execute(mH.get(), x, y) : mnnb200_conv_f32_execute(mH.get(), x, y), "float conv");
    }
private:
    const Op* mOp;
    ExecHandle mH;
    bool mDepthwise;
    int mIc, mInC;
};
// Deconvolution (group 1, split-TF32 wgmma over the stride phases) and DeconvolutionDepthwise on float tensors: CPUDeconvolution /
// CPUDeconvolutionDepthwise with the weights in the op.  The input channel count is the input's (CPUDeconvolution ignores group);
// dynamic weights (a second input without an output shape) are declined.  A clone is made again from the op with the same input
// channel count.
class DeconvF32Exec : public B200Exec {
public:
    DeconvF32Exec(Backend* bn, const Op* op, mnnb200_exec* h, bool dw, int ic) : B200Exec(bn), mOp(op), mH(h), mDepthwise(dw), mIc(ic) {}
    static bool takes(const Op* op, const std::vector<Tensor*>& inputs) {
        auto conv = op->main_as_Convolution2D();
        return conv && conv->common() && !inputs.empty() && isF32Nchw(inputs[0]) &&
               (inputs.size() == 1 || (inputs.size() == 2 && conv->common()->hasOutputShape()));
    }
    static Execution* create(B200Backend* bn, const Op* op, int ic) {
        auto conv = op->main_as_Convolution2D();
        if (!conv || !conv->common()) return nullptr;
        auto cm = conv->common();
        const bool dw = op->type() == OpType_DeconvolutionDepthwise;
        const int oc = cm->outputCount(), kh = cm->kernelY(), kw = cm->kernelX();
        if (!dw && cm->group() != 1) return nullptr;
        if (dw && (ic != oc || (cm->group() != 1 && cm->group() != oc))) return nullptr;
        std::shared_ptr<ConvolutionCommon::Int8Common> quanCommon;
        const float* w = nullptr;
        int wsize = 0;
        ConvolutionCommon::getConvParameters(&quanCommon, bn, op, &w, &wsize);
        if (!w || oc <= 0 || kh <= 0 || kw <= 0 || ic <= 0 || (size_t)wsize != (size_t)(dw ? 1 : ic) * oc * kh * kw) return nullptr;
        mnnb200_conv_desc d;
        d.ic = ic; d.oc = oc; d.kh = kh; d.kw = kw; d.stride_h = cm->strideY(); d.stride_w = cm->strideX();
        d.pad_h = 0; d.pad_w = 0; d.dilate_h = cm->dilateY(); d.dilate_w = cm->dilateX();   // pads: set at resize
        d.group = dw ? oc : 1; d.relu = cm->relu() ? 1 : 0;
        const float* bias = (conv->bias() && (int)conv->bias()->size() == oc) ? conv->bias()->data() : nullptr;
        mnnb200_exec* h = nullptr;
        mnnb200_status st = dw ? mnnb200_dwdeconv_f32_create(bn->handle(), &d, w, bias, cm->relu6() ? 1 : 0, &h)
                               : mnnb200_deconv_f32_create(bn->handle(), &d, w, bias, cm->relu6() ? 1 : 0, &h);
        if (st != MNNB200_OK) {
            if (st != MNNB200_NOT_SUPPORT) MNN_ERROR("mnn_b200 float deconv create: %s\n", mnnb200_last_error());
            return nullptr;
        }
        return new DeconvF32Exec(bn, op, h, dw, ic);
    }
    bool onClone(Backend* bn, const Op* op, Execution** dst) override {
        if (dst == nullptr) return true;
        *dst = create(static_cast<B200Backend*>(bn), op, mIc);
        return *dst != nullptr;
    }
    ErrorCode onResize(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        auto in = inputs[0], out = outputs[0];
        if (in->dimensions() != 4 || in->channel() != mIc) {   // the kernels index the input by the weights' channel count
            MNN_ERROR("mnn_b200 float deconv: input has %d channels, the weights %d\n", in->channel(), mIc);
            return NOT_SUPPORT;
        }
        auto pad = ConvolutionCommon::convolutionTransposePad(in, out, mOp->main_as_Convolution2D()->common());   // (padX, padY)
        int oh = out->height(), ow = out->width();
        mnnb200_status st = mnnb200_deconv_f32_set_pad(mH.get(), pad.second, pad.first);
        if (st == MNNB200_OK)
            st = mDepthwise ? mnnb200_dwdeconv_f32_resize(mH.get(), in->batch(), in->height(), in->width(), &oh, &ow)
                            : mnnb200_deconv_f32_resize(mH.get(), in->batch(), in->height(), in->width(), &oh, &ow);
        return toErr(st, "float deconv resize");
    }
    ErrorCode launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        auto x = (const float*)dev(inputs[0]);
        auto y = (float*)dev(outputs[0]);
        return toErr(mDepthwise ? mnnb200_dwdeconv_f32_execute(mH.get(), x, y) : mnnb200_deconv_f32_execute(mH.get(), x, y),
                     "float deconv");
    }
private:
    const Op* mOp;
    ExecHandle mH;
    bool mDepthwise;
    int mIc;
};
static bool isF32(const Tensor* t) { return t->getType().code == halide_type_float && t->getType().bytes() == 4; }
// a full-size operand has the output's bytes: the same linear layout, or both of <= 2 dims (NCHW and NHWC are then the same)
static bool sameLinear(const Tensor* t, const Tensor* out) {
    return linearFormat(t) == linearFormat(out) || (t->dimensions() <= 2 && out->dimensions() <= 2);
}
// BinaryOp on float tensors (CPUBinary): with GEOMETRY_COMPUTE_MASK 0 every broadcast but a one-element side has been turned into
// a Raster before the op (GeometryBinary.cpp), so each input is either the output's size or one element
class BinaryF32Exec : public B200Exec {
public:
    BinaryF32Exec(Backend* bn, int op, int relu) : B200Exec(bn), mOp(op), mRelu(relu) {}
    static bool supports(int op) {
        switch (op) {
            case BinaryOpOperation_ADD: case BinaryOpOperation_SUB: case BinaryOpOperation_MUL: case BinaryOpOperation_REALDIV:
            case BinaryOpOperation_MINIMUM: case BinaryOpOperation_MAXIMUM: case BinaryOpOperation_SquaredDifference:
                return true;
            default:
                return false;
        }
    }
    static bool takes(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) {
        if (inputs.size() != 2 || outputs.size() != 1 || !isF32(outputs[0])) return false;
        const size_t n = elemCount(outputs[0]);
        int full = 0;
        for (auto t : inputs) {
            if (!isF32(t)) return false;
            const size_t c = elemCount(t);
            if (c == n && sameLinear(t, outputs[0])) ++full;
            else if (c != 1) return false;
        }
        return full >= 1 || n == 1;
    }
    ErrorCode launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        return toErr(mnnb200_binary_f32(rt(), mOp, (const float*)dev(inputs[0]), elemCount(inputs[0]),
                                        (const float*)dev(inputs[1]), elemCount(inputs[1]), (float*)dev(outputs[0]), elemCount(outputs[0]),
                                        mRelu), "BinaryOp fp32");
    }
private:
    int mOp, mRelu;
};
// Eltwise SUM / PROD / MAXIMUM / SUB (CPUEltwise.cpp:46-85): inputs 0 and 1, then every further input folded into the output
class EltwiseF32Exec : public B200Exec {
public:
    EltwiseF32Exec(Backend* bn, int op) : B200Exec(bn), mOp(op) {}
    static int binaryOp(EltwiseType t) {
        switch (t) {
            case EltwiseType_PROD: return BinaryOpOperation_MUL;
            case EltwiseType_SUM: return BinaryOpOperation_ADD;
            case EltwiseType_MAXIMUM: return BinaryOpOperation_MAXIMUM;
            case EltwiseType_SUB: return BinaryOpOperation_SUB;
            default: return -1;
        }
    }
    ErrorCode launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        const size_t n = elemCount(outputs[0]);
        auto y = (float*)dev(outputs[0]);
        mnnb200_status st = mnnb200_binary_f32(rt(), mOp, (const float*)dev(inputs[0]), n, (const float*)dev(inputs[1]), n, y, n, 0);
        for (size_t i = 2; st == MNNB200_OK && i < inputs.size(); ++i)
            st = mnnb200_binary_f32(rt(), mOp, y, n, (const float*)dev(inputs[i]), n, y, n, 0);
        return toErr(st, "Eltwise fp32");
    }
private:
    int mOp;
};
class UnaryF32Exec : public B200Exec {
public:
    UnaryF32Exec(Backend* bn, int op) : B200Exec(bn), mOp(op) {}
    static bool supports(int op) {
        switch (op) {
            case UnaryOpOperation_ABS: case UnaryOpOperation_NEG: case UnaryOpOperation_SQUARE: case UnaryOpOperation_SQRT:
            case UnaryOpOperation_RSQRT: case UnaryOpOperation_EXP: case UnaryOpOperation_LOG: case UnaryOpOperation_RECIPROCAL:
            case UnaryOpOperation_SIGMOID: case UnaryOpOperation_TANH: case UnaryOpOperation_HARDSWISH: case UnaryOpOperation_GELU:
            case UnaryOpOperation_GELU_STANDARD: case UnaryOpOperation_SILU:
                return true;
            default:
                return false;
        }
    }
    ErrorCode launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        return toErr(mnnb200_unary_f32(rt(), mOp, (const float*)dev(inputs[0]),
                                       (float*)dev(outputs[0]), elemCount(outputs[0])), "UnaryOp fp32");
    }
private:
    int mOp;
};
// a tensor as [outside][axis][inside] around one of its dimensions
struct AxisSplit { int outside, axis, inside; };
static AxisSplit splitAt(const Tensor* t, int axis) {
    AxisSplit s = {1, t->length(axis), 1};
    for (int i = 0; i < axis; ++i) s.outside *= t->length(i);
    for (int i = axis + 1; i < t->dimensions(); ++i) s.inside *= t->length(i);
    return s;
}
ErrorCode ReduceF32Exec::launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) {
    auto s = splitAt(inputs[0], mAxis);
    return toErr(mnnb200_reduce_f32(rt(), (const float*)dev(inputs[0]), s.outside, s.axis, s.inside, mOp, (float*)dev(outputs[0])),
                 "Reduction");
}
// ArgMax / ArgMin with one index per position and no values (CPUArgMax's non-NC4HW4 branch): int32 output
class ArgMaxExec : public B200Exec {
public:
    ArgMaxExec(Backend* bn, int axis, bool isMin) : B200Exec(bn), mAxis(axis), mIsMin(isMin) {}
    ErrorCode launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        auto s = splitAt(inputs[0], mAxis);
        return toErr(mnnb200_argmax_f32(rt(), (const float*)dev(inputs[0]), s.outside, s.axis, s.inside, mIsMin ? 1 : 0,
                                        (int32_t*)dev(outputs[0])), "ArgMax");
    }
private:
    int mAxis;
    bool mIsMin;
};
class ScaleF32Exec : public ClonedFromOp<ScaleF32Exec> {
public:
    ScaleF32Exec(Backend* bn, mnnb200_exec* h) : ClonedFromOp(bn), mH(h) {}
    static Execution* create(B200Backend* bn, const Op* op) {
        auto sc = op->main_as_Scale();
        if (!sc || !sc->scaleData()) return nullptr;
        const int c = (int)sc->scaleData()->size();
        const float* bias = (sc->biasData() && (int)sc->biasData()->size() == c) ? sc->biasData()->data() : nullptr;
        mnnb200_exec* h = nullptr;
        if (mnnb200_scale_f32_create(bn->handle(), c, sc->scaleData()->data(), bias, &h) != MNNB200_OK) return nullptr;
        return new ScaleF32Exec(bn, h);
    }
    ErrorCode onResize(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>&) override {
        auto d = dims4(inputs[0]);
        return toErr(mnnb200_scale_f32_resize(mH.get(), d.n, d.h, d.w), "Scale fp32 resize");
    }
    ErrorCode launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        return toErr(mnnb200_scale_f32_execute(mH.get(), (const float*)dev(inputs[0]), (float*)dev(outputs[0])), "Scale fp32");
    }
private:
    ExecHandle mH;
};
// Softmax over one axis of an [outside][axis][inside] view (CPUSoftmax.cpp)
class SoftmaxF32Exec : public B200Exec {
public:
    SoftmaxF32Exec(Backend* bn, int axis) : B200Exec(bn), mAxis(axis) {}
    ErrorCode launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        auto s = splitAt(inputs[0], mAxis);
        return toErr(mnnb200_softmax_f32(rt(), (const float*)dev(inputs[0]), s.outside, s.axis, s.inside, (float*)dev(outputs[0])),
                     "Softmax fp32");
    }
private:
    int mAxis;
};

// LayerNorm / RMSNorm fp32 (CPULayerNorm.cpp).  The [rows][inner] view comes from the input's shape, so the C ABI execution is made
// at the first resize and again when inner changes; gamma / beta are read from the op as CPULayerNorm::makeResource reads them.
class LayerNormF32Exec : public ClonedFromOp<LayerNormF32Exec> {
public:
    LayerNormF32Exec(Backend* bn, const Op* op) : ClonedFromOp(bn), mOp(op) {}
    static Execution* create(B200Backend* bn, const Op* op) {
        auto ln = op->main_as_LayerNorm();
        if (!ln) return nullptr;
        // gamma / beta held outside the op (LayerNorm.external, the useCachedMmap path) are not read here
        const bool external = ln->external() && ln->external()->size() > 1 && ln->external()->data()[1] > 0;
        if ((external && !(ln->gamma() && ln->beta())) || bn->getRuntime()->hint().useCachedMmap > 1) return nullptr;
        return new LayerNormF32Exec(bn, op);
    }
    // rows x inner of the CPU's onResize (CPULayerNorm.cpp:228-256): the NC4HW4 forms normalise channels of [tokens, C, 1, 1];
    // group > 1: length(0) * group rows; otherwise the last axis().size() dims.  false: a shape the execution does not take
    static bool view(const Op* op, const Tensor* x, int* rows, int* inner) {
        auto ln = op->main_as_LayerNorm();
        const int rank = x->dimensions();
        long long r = 1, n = 1;
        if (TensorUtils::getDescribe(x)->dimensionFormat == MNN_DATA_FORMAT_NC4HW4) {
            if (rank < 2) return false;
            r = x->length(0); n = x->length(1);
            if ((long long)elemCount(x) != r * n) return false;   // H * W > 1: the CPU's NC4HW4 branch ignores the spatial dims
        } else if (ln->group() > 1) {
            if (rank < 1) return false;
            r = (long long)x->length(0) * ln->group();
            for (int i = 1; i < rank; ++i) n *= x->length(i);
            if (n % ln->group()) return false;
            n /= ln->group();
        } else {
            const int axis = ln->axis() ? (int)ln->axis()->size() : 0;
            if (axis > rank) return false;
            for (int i = 0; i < rank - axis; ++i) r *= x->length(i);
            for (int i = rank - axis; i < rank; ++i) n *= x->length(i);
        }
        if (r <= 0 || n <= 0 || r > 0x7fffffffLL || n > 0x7fffffffLL) return false;
        *rows = (int)r; *inner = (int)n;
        return true;
    }
    // the 1-in / 1-out form, or the NC4HW4 residual form (2-in / 2-out, CPULayerNorm.cpp:93-153); fp32 tensors only
    static bool takes(const Op* op, const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) {
        if (inputs.empty() || inputs.size() != outputs.size() || inputs.size() > 2) return false;
        for (auto t : inputs) if (!isF32(t) || isInt8(t) || elemCount(t) != elemCount(inputs[0])) return false;
        for (auto t : outputs) if (!isF32(t) || isInt8(t) || elemCount(t) != elemCount(inputs[0])) return false;
        if (inputs.size() == 2) {
            for (auto t : inputs) if (TensorUtils::getDescribe(t)->dimensionFormat != MNN_DATA_FORMAT_NC4HW4) return false;
        }
        int rows, inner;
        if (!view(op, inputs[0], &rows, &inner)) return false;
        auto ln = op->main_as_LayerNorm();
        if (ln->gamma() && ln->beta() && ((int)ln->gamma()->size() != inner || (int)ln->beta()->size() != inner)) return false;
        return true;
    }
    ErrorCode onResize(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        int rows, inner;
        if (!takes(mOp, inputs, outputs) || !view(mOp, inputs[0], &rows, &inner)) return NOT_SUPPORT;
        if (!mH || inner != mInner) {
            auto ln = mOp->main_as_LayerNorm();
            const bool affine = ln->gamma() && ln->beta();
            mnnb200_exec* h = nullptr;
            ErrorCode ec = toErr(mnnb200_layernorm_f32_create(rt(), inner, ln->epsilon(), ln->useRMSNorm() ? 1 : 0,
                                                              affine ? ln->gamma()->data() : nullptr,
                                                              affine ? ln->beta()->data() : nullptr, affine ? inner : 0, &h),
                                 "LayerNorm fp32 create");
            if (ec != NO_ERROR) return ec;
            mH.reset(h);
            mInner = inner;
        }
        return toErr(mnnb200_layernorm_f32_resize(mH.get(), rows), "LayerNorm fp32 resize");
    }
    ErrorCode launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        if (inputs.size() == 2)   // outputs: the sum x + r, then its norm
            return toErr(mnnb200_layernorm_f32_execute(mH.get(), (const float*)dev(inputs[0]), (const float*)dev(inputs[1]),
                                                       (float*)dev(outputs[0]), (float*)dev(outputs[1])), "LayerNorm fp32");
        return toErr(mnnb200_layernorm_f32_execute(mH.get(), (const float*)dev(inputs[0]), nullptr, nullptr, (float*)dev(outputs[0])),
                     "LayerNorm fp32");
    }
private:
    const Op* mOp;
    ExecHandle mH;
    int mInner = 0;
};
// Fused RoPE fp32 (CPURoPE.cpp): q / k NC4HW4 [seq, C, 1, 1] (stored [seq][C] here), cos / sin [seq][ropeDim], outputs NHWC
// [1, seq, heads, head_dim]; the q / k norm tables read from RoPEParam as makeRopeNormResource reads them (CPURoPE.cpp:20-49)
class RoPEF32Exec : public ClonedFromOp<RoPEF32Exec> {
public:
    RoPEF32Exec(Backend* bn, mnnb200_exec* h) : ClonedFromOp(bn), mH(h) {}
    static Execution* create(B200Backend* bn, const Op* op) {
        auto rp = op->main_as_RoPEParam();
        if (!rp) return nullptr;
        mnnb200_rope_norm qn, kn;
        auto table = [](const LayerNorm* ln, mnnb200_rope_norm* t) -> const mnnb200_rope_norm* {
            if (!ln || !ln->gamma() || ln->gamma()->size() == 0) return nullptr;
            const int size = (int)ln->gamma()->size();
            *t = mnnb200_rope_norm{ln->gamma()->data(), (ln->beta() && (int)ln->beta()->size() == size) ? ln->beta()->data() : nullptr,
                                   size, ln->epsilon(), ln->useRMSNorm() ? 1 : 0};
            return t;
        };
        mnnb200_exec* h = nullptr;
        if (mnnb200_rope_f32_create(bn->handle(), rp->num_head(), rp->kv_num_head(), rp->head_dim(), rp->rope_cut_head_dim(),
                                    table(rp->q_norm(), &qn), table(rp->k_norm(), &kn), &h) != MNNB200_OK)
            return nullptr;
        return new RoPEF32Exec(bn, h);
    }
    // validRopeC4Input (CPURoPE.cpp:71-84), fp32 everywhere, cos / sin linear with a ropeDim row per token
    static bool takes(const Op* op, const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) {
        auto rp = op->main_as_RoPEParam();
        if (!rp || inputs.size() != 4 || outputs.size() != 2) return false;
        const int heads = rp->num_head(), kvh = rp->kv_num_head(), hd = rp->head_dim();
        if (heads <= 0 || kvh <= 0 || hd <= 0) return false;
        for (auto t : inputs) if (!isF32(t) || isInt8(t)) return false;
        for (auto t : outputs) if (!isF32(t) || isInt8(t)) return false;
        auto q = inputs[0], k = inputs[1];
        for (auto t : {q, k})
            if (TensorUtils::getDescribe(t)->dimensionFormat != MNN_DATA_FORMAT_NC4HW4 || t->dimensions() != 4 || t->length(2) != 1 ||
                t->length(3) != 1)
                return false;
        if (q->length(0) != k->length(0) || q->length(1) != heads * hd || k->length(1) != kvh * hd) return false;
        const int cut = rp->rope_cut_head_dim();
        const size_t ropeDim = (size_t)((cut <= 0 || cut > hd ? hd : cut) / 2 * 2);
        for (int i = 2; i < 4; ++i)
            if (TensorUtils::getDescribe(inputs[i])->dimensionFormat == MNN_DATA_FORMAT_NC4HW4 ||
                elemCount(inputs[i]) < (size_t)q->length(0) * ropeDim)
                return false;
        return elemCount(outputs[0]) == elemCount(q) && elemCount(outputs[1]) == elemCount(k);
    }
    ErrorCode onResize(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>&) override {
        return toErr(mnnb200_rope_f32_resize(mH.get(), inputs[0]->length(0), inputs[0]->length(1), inputs[1]->length(1)), "RoPE fp32 resize");
    }
    ErrorCode launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        return toErr(mnnb200_rope_f32_execute(mH.get(), (const float*)dev(inputs[0]), (const float*)dev(inputs[1]),
                                              (const float*)dev(inputs[2]), (const float*)dev(inputs[3]), (float*)dev(outputs[0]),
                                              (float*)dev(outputs[1])), "RoPE fp32");
    }
private:
    ExecHandle mH;
};

// Interp on float tensors (CPUInterp): the op the geometry stage lowers Interp and Resize to, one 4-D input, NCHW-linear (NC4HW4 is
// stored so here), whose widthScale / heightScale / widthOffset / heightOffset already hold the coordinate transform.  They are
// read as CPUInterpCreator reads them, with the resize type; resize types outside 1-4 and TensorflowCropAndResize (the geometry
// leaves its scales unset) are declined, as are int8 tensors.  The planes are batch * channels, the sizes those of onResize.
class InterpF32Exec : public ClonedFromOp<InterpF32Exec> {
public:
    InterpF32Exec(Backend* bn, mnnb200_exec* h) : ClonedFromOp(bn), mH(h) {}
    static Execution* create(B200Backend* bn, const Op* op) {
        auto ip = op->main_as_Interp();
        if (!ip || ip->resizeType() < 1 || ip->resizeType() > 4 || ip->ctm() == CoordinateTransformationMode_TensorflowCropAndResize)
            return nullptr;
        mnnb200_exec* h = nullptr;
        if (mnnb200_interp_f32_create(bn->handle(), ip->resizeType(), ip->widthScale(), ip->heightScale(), ip->widthOffset(),
                                      ip->heightOffset(), &h) != MNNB200_OK)
            return nullptr;
        return new InterpF32Exec(bn, h);
    }
    static bool takes(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) {
        if (inputs.size() != 1 || outputs.size() != 1) return false;
        auto in = inputs[0], out = outputs[0];
        return isF32(in) && isF32(out) && !isInt8(in) && !isInt8(out) && in->dimensions() == 4 && out->dimensions() == 4 &&
               linearFormat(in) == MNN_DATA_FORMAT_NCHW && linearFormat(out) == MNN_DATA_FORMAT_NCHW &&
               in->batch() == out->batch() && in->channel() == out->channel();
    }
    ErrorCode onResize(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        auto in = inputs[0], out = outputs[0];
        const long long planes = (long long)in->batch() * in->channel();
        if (!takes(inputs, outputs) || planes > 0x7fffffffLL) return NOT_SUPPORT;
        return toErr(mnnb200_interp_f32_resize(mH.get(), (int)planes, in->height(), in->width(), out->height(), out->width()),
                     "Interp fp32 resize");
    }
    ErrorCode launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        return toErr(mnnb200_interp_f32_execute(mH.get(), (const float*)dev(inputs[0]), (float*)dev(outputs[0])), "Interp fp32");
    }
private:
    ExecHandle mH;
};

// GridSample on float tensors (CPUGridSample): x [N, C, (D,) H, W] NCHW-linear (NC4HW4 is stored so here), grid [N, (oD,) oH, oW,
// rank - 2] in a linear format (an NC4HW4 grid is declined: the CPU reads the grid linearly), y [N, C, (oD,) oH, oW].  The op's
// mode, paddingMode and alignCorners are read as CPUGridSampleCreator reads them; REFLECTION samples as CLAMP there and here.
// Declined: the backward form (and its third input), other input / output counts, non-fp32 or int8 tensors, ranks other than 4
// and 5, a batch mismatch, a grid whose last dim is not rank - 2, and any index past 31 bits (resize refuses those).
class GridSampleF32Exec : public ClonedFromOp<GridSampleF32Exec> {
public:
    GridSampleF32Exec(Backend* bn, const Op* op, mnnb200_exec* h) : ClonedFromOp(bn), mOp(op), mH(h) {}
    static Execution* create(B200Backend* bn, const Op* op) {
        auto gp = op->main_as_GridSample();
        if (!gp || gp->backward()) return nullptr;
        mnnb200_exec* h = nullptr;
        if (mnnb200_grid_sample_f32_create(bn->handle(), (int)gp->mode(), (int)gp->paddingMode(), gp->alignCorners() ? 1 : 0, &h) !=
            MNNB200_OK)
            return nullptr;
        return new GridSampleF32Exec(bn, op, h);
    }
    static bool takes(const Op* op, const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) {
        auto gp = op->main_as_GridSample();
        if (!gp || gp->backward() || inputs.size() != 2 || outputs.size() != 1) return false;
        auto x = inputs[0], g = inputs[1], y = outputs[0];
        for (auto t : {x, g, y})
            if (!isF32(t) || isInt8(t)) return false;
        const int rank = x->dimensions();
        if ((rank != 4 && rank != 5) || g->dimensions() != rank || y->dimensions() != rank) return false;
        if (linearFormat(x) != MNN_DATA_FORMAT_NCHW || linearFormat(y) != MNN_DATA_FORMAT_NCHW ||
            TensorUtils::getDescribe(g)->dimensionFormat == MNN_DATA_FORMAT_NC4HW4)
            return false;
        if (g->length(0) != x->length(0) || g->length(rank - 1) != rank - 2) return false;
        if (y->length(0) != x->length(0) || y->length(1) != x->length(1)) return false;
        for (int i = 2; i < rank; ++i)
            if (y->length(i) != g->length(i - 1)) return false;
        return true;
    }
    ErrorCode onResize(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        if (!takes(mOp, inputs, outputs)) return NOT_SUPPORT;
        auto x = inputs[0], g = inputs[1];
        const int rank = x->dimensions();
        int ind[3] = {0, 0, 0}, outd[3] = {0, 0, 0};
        for (int i = 2; i < rank; ++i) {
            ind[i - 2] = x->length(i);
            outd[i - 2] = g->length(i - 1);
        }
        return toErr(mnnb200_grid_sample_f32_resize(mH.get(), rank, x->length(0), x->length(1), ind, outd), "GridSample fp32 resize");
    }
    ErrorCode launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        return toErr(mnnb200_grid_sample_f32_execute(mH.get(), (const float*)dev(inputs[0]), (const float*)dev(inputs[1]),
                                                     (float*)dev(outputs[0])),
                     "GridSample fp32");
    }
private:
    const Op* mOp;
    ExecHandle mH;
};

// Gather / GatherV2 / GatherND / GatherElements (the CPU runs them as While loops of GeometryGather.cpp; under Compiler_Geometry
// they reach the backend unlowered) on tensors of 4-byte elements, fp32 or int32, with int32 indices.  Params and output are
// linear in their logical dim order: any format but NC4HW4, which only a 4-D tensor may have (it is stored NCHW-linear here).
// The axis is read as the geometry reads it: Gather from the op's Axis, else its third input, else 0; GatherND's batch dims
// from the op's Axis; GatherElements' axis from its third input, else 0.  A third input must be a constant (read at resize).
class GatherExec : public ClonedFromOp<GatherExec> {
public:
    GatherExec(Backend* bn, const Op* op, mnnb200_exec* h) : ClonedFromOp(bn), mOp(op), mH(h) {}
    static int mode(const Op* op) {
        return op->type() == OpType_GatherND ? 1 : (op->type() == OpType_GatherElements ? 2 : 0);
    }
    static Execution* create(B200Backend* bn, const Op* op) {
        mnnb200_exec* h = nullptr;
        if (mnnb200_gather_create(bn->handle(), mode(op), &h) != MNNB200_OK) return nullptr;
        return new GatherExec(bn, op, h);
    }
    static bool word(const Tensor* t) {
        const auto f = TensorUtils::getDescribe(t)->dimensionFormat;
        return t->getType().bytes() == 4 && !isInt8(t) && (f != MNN_DATA_FORMAT_NC4HW4 || t->dimensions() == 4);
    }
    static bool takes(const Op* op, const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) {
        const size_t most = op->type() == OpType_GatherND ? 2 : 3;
        if (inputs.size() < 2 || inputs.size() > most || outputs.size() != 1) return false;
        auto x = inputs[0], idx = inputs[1], y = outputs[0];
        const bool i32 = idx->getType().code == halide_type_int && idx->getType().bits == 32 && !isInt8(idx);
        bool ok = i32 && word(x) && word(y) && x->getType() == y->getType() && linearFormat(x) == linearFormat(y) &&
                  x->dimensions() >= 1;
        if (inputs.size() == 3) {
            auto ax = inputs[2];
            ok = ok && ax->getType().code == halide_type_int && ax->getType().bits == 32 && elemCount(ax) >= 1 &&
                 (ax->host<int>() != nullptr || TensorUtils::getDescribe(ax)->usage == Tensor::InsideDescribe::CONSTANT);
        }
        return ok;
    }
    ErrorCode onResize(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        auto x = inputs[0], idx = inputs[1];
        const int m = mode(mOp);
        int axis = 0;
        if (m == 1) {
            if (mOp->main_as_Axis()) axis = mOp->main_as_Axis()->axis();
        } else {
            if (inputs.size() == 3) {
                auto ax = inputs[2];
                if (ax->host<int>()) axis = ax->host<int>()[0];
                else if (mnnb200_memcpy_d2h(rt(), &axis, dev(ax), sizeof(int)) != MNNB200_OK || mnnb200_runtime_sync(rt()) != MNNB200_OK)
                    return toErr(MNNB200_CUDA_ERROR, "Gather axis read");
            }
            if (m == 0 && mOp->main_type() == OpParameter_Axis && mOp->main_as_Axis()) axis = mOp->main_as_Axis()->axis();
        }
        std::vector<int> pd(x->dimensions()), id(std::max(idx->dimensions(), 1));
        for (int i = 0; i < x->dimensions(); ++i) pd[i] = x->length(i);
        if (m == 0) id = {(int)elemCount(idx)};   // Gather reads the indices flat; a scalar index is one
        else for (int i = 0; i < idx->dimensions(); ++i) id[i] = idx->length(i);
        if (m != 0 && idx->dimensions() == 0) id[0] = 1;
        return toErr(mnnb200_gather_resize(mH.get(), pd.data(), (int)pd.size(), id.data(), (int)id.size(), axis), "gather resize");
    }
    ErrorCode launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        return toErr(mnnb200_gather_execute(mH.get(), dev(inputs[0]), (const int*)dev(inputs[1]), dev(outputs[0])), "gather");
    }
private:
    const Op* mOp;
    ExecHandle mH;
};

// ScatterNd(indices, updates, shape[, data]) / ScatterElements(data, indices, updates[, axis]) (GeometryScatter.cpp registers
// their lowering for Compiler_Loop only, so under Compiler_Geometry they reach the backend unlowered) on tensors of 4-byte
// elements, fp32, or int32 without a reduction, with int32 indices; data, updates and output linear in their logical dim order
// as GatherExec's.  The reduction is read as the geometry reads it: the op's BinaryOp opType (ScatterNd: none without one);
// ADD, SUB and MUL are taken, other codes declined.  The ScatterElements axis is a constant fourth input (read at resize), else
// 0.  A 3-input ScatterNd has no data (the output starts zero-filled), so the handle is made at resize, for the inputs given.
class ScatterExec : public ClonedFromOp<ScatterExec> {
public:
    ScatterExec(Backend* bn, const Op* op) : ClonedFromOp(bn), mOp(op) {}
    static Execution* create(B200Backend* bn, const Op* op) { return new ScatterExec(bn, op); }
    static bool elements(const Op* op) { return op->type() == OpType_ScatterElements; }
    static int reduction(const Op* op) { return op->main_as_BinaryOp() ? (int)op->main_as_BinaryOp()->opType() : -1; }
    static Tensor* data(const Op* op, const std::vector<Tensor*>& inputs) {
        return elements(op) ? inputs[0] : (inputs.size() == 4 ? inputs[3] : nullptr);
    }
    static bool takes(const Op* op, const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) {
        if (inputs.size() < 3 || inputs.size() > 4 || outputs.size() != 1) return false;
        if (elements(op) && !op->main_as_BinaryOp()) return false;
        const int red = reduction(op);
        auto idx = inputs[elements(op) ? 1 : 0], upd = inputs[elements(op) ? 2 : 1], y = outputs[0], x = data(op, inputs);
        const bool i32 = idx->getType().code == halide_type_int && idx->getType().bits == 32 && !isInt8(idx);
        bool ok = red <= 2 && i32 && GatherExec::word(upd) && GatherExec::word(y) && upd->getType() == y->getType() &&
                  linearFormat(upd) == linearFormat(y) && y->dimensions() >= 1 && idx->dimensions() >= 1;
        if (red >= 0) ok = ok && y->getType().code == halide_type_float;
        if (x) ok = ok && GatherExec::word(x) && x->getType() == y->getType() && linearFormat(x) == linearFormat(y) &&
                    elemCount(x) == elemCount(y);
        if (elements(op) && inputs.size() == 4) {
            auto ax = inputs[3];
            ok = ok && ax->getType().code == halide_type_int && ax->getType().bits == 32 && elemCount(ax) >= 1 &&
                 (ax->host<int>() != nullptr || TensorUtils::getDescribe(ax)->usage == Tensor::InsideDescribe::CONSTANT);
        }
        return ok;
    }
    ErrorCode onResize(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        if (!takes(mOp, inputs, outputs)) return NOT_SUPPORT;
        const bool withData = data(mOp, inputs) != nullptr;
        if (!mH || withData != mWithData) {
            mnnb200_exec* h = nullptr;
            const mnnb200_status st = mnnb200_scatter_create(rt(), elements(mOp) ? 1 : 0, reduction(mOp), withData ? 1 : 0, &h);
            if (st != MNNB200_OK) return toErr(st, "scatter create");
            mH.reset(h);
            mWithData = withData;
        }
        int axis = 0;
        if (elements(mOp) && inputs.size() == 4) {
            auto ax = inputs[3];
            if (ax->host<int>()) axis = ax->host<int>()[0];
            else if (mnnb200_memcpy_d2h(rt(), &axis, dev(ax), sizeof(int)) != MNNB200_OK || mnnb200_runtime_sync(rt()) != MNNB200_OK)
                return toErr(MNNB200_CUDA_ERROR, "ScatterElements axis read");
        }
        auto dims = [](const Tensor* t) {
            std::vector<int> d(t->dimensions());
            for (int i = 0; i < t->dimensions(); ++i) d[i] = t->length(i);
            return d;
        };
        auto idx = inputs[elements(mOp) ? 1 : 0], upd = inputs[elements(mOp) ? 2 : 1], y = outputs[0];
        const std::vector<int> od = dims(y), id = dims(idx), ud = dims(upd);
        return toErr(mnnb200_scatter_resize(mH.get(), od.data(), (int)od.size(), id.data(), (int)id.size(), ud.data(), (int)ud.size(),
                                            axis, y->getType().code == halide_type_int ? 1 : 0),
                     "scatter resize");
    }
    ErrorCode launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        auto x = data(mOp, inputs);
        auto idx = inputs[elements(mOp) ? 1 : 0], upd = inputs[elements(mOp) ? 2 : 1];
        return toErr(mnnb200_scatter_execute(mH.get(), x ? dev(x) : nullptr, (const int*)dev(idx), dev(upd), dev(outputs[0])), "scatter");
    }
private:
    const Op* mOp;
    ExecHandle mH;
    bool mWithData = false;
};

// ONNX LSTM / RNN (OpType_LSTM / OpType_RNN with X, W, R, B[, h0[, c0]]; GeometryLSTM.cpp registers their lowering for
// Compiler_Loop only, so under Compiler_Geometry they reach the backend unlowered) on fp32 tensors in a linear layout: X [T, B, I],
// W [D, G*H, I], R [D, G*H, H], B of D*G*H elements, h0 / c0 [D, B, H], outputs Y [T, D, B, H], Y_h (and for LSTM Y_c)
// [D, B, H], with H = the op's outputCount and G = 4 (LSTM) or 1 (RNN).  Declined: the Caffe single-input LSTM (one input, one
// output), an RNN with a cell input, int8 / fp16 / NC4HW4 tensors and inconsistent shapes.
class RnnExec : public ClonedFromOp<RnnExec> {
public:
    RnnExec(Backend* bn, const Op* op, mnnb200_exec* h) : ClonedFromOp(bn), mOp(op), mH(h) {}
    static Execution* create(B200Backend* bn, const Op* op) {
        mnnb200_exec* h = nullptr;
        if (mnnb200_rnn_create(bn->handle(), op->type() == OpType_RNN ? 1 : 0, &h) != MNNB200_OK) return nullptr;
        return new RnnExec(bn, op, h);
    }
    static bool f32Linear(const Tensor* t) {
        return isF32(t) && !isInt8(t) && TensorUtils::getDescribe(t)->dimensionFormat != MNN_DATA_FORMAT_NC4HW4;
    }
    static bool shaped(const Tensor* t, std::initializer_list<int> d) {
        if (t->dimensions() != (int)d.size()) return false;
        int i = 0;
        for (int v : d) if (t->length(i++) != v) return false;
        return true;
    }
    static bool takes(const Op* op, const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) {
        const bool lstm = op->type() == OpType_LSTM;
        if (!op->main_as_LSTM() || inputs.size() < 4 || inputs.size() > (lstm ? 6u : 5u) || outputs.size() != (lstm ? 3u : 2u))
            return false;
        for (auto t : inputs) if (!f32Linear(t)) return false;
        for (auto t : outputs) if (!f32Linear(t)) return false;
        auto x = inputs[0], w = inputs[1], r = inputs[2];
        if (x->dimensions() != 3 || w->dimensions() != 3) return false;
        const int T = x->length(0), B = x->length(1), I = x->length(2), D = w->length(0), H = op->main_as_LSTM()->outputCount();
        const int G = lstm ? 4 : 1;
        if (T < 1 || B < 1 || I < 1 || H < 1 || (D != 1 && D != 2)) return false;
        bool ok = shaped(w, {D, G * H, I}) && shaped(r, {D, G * H, H}) && elemCount(inputs[3]) == (size_t)D * G * H &&
                  shaped(outputs[0], {T, D, B, H});
        for (size_t k = 4; k < inputs.size(); ++k) ok = ok && shaped(inputs[k], {D, B, H});
        for (size_t k = 1; k < outputs.size(); ++k) ok = ok && shaped(outputs[k], {D, B, H});
        return ok;
    }
    ErrorCode onResize(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        if (!takes(mOp, inputs, outputs)) return NOT_SUPPORT;
        auto x = inputs[0];
        return toErr(mnnb200_rnn_resize(mH.get(), x->length(0), x->length(1), x->length(2), mOp->main_as_LSTM()->outputCount(),
                                        inputs[1]->length(0), inputs.size() >= 5 ? 1 : 0, inputs.size() >= 6 ? 1 : 0),
                     "rnn resize");
    }
    ErrorCode launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        auto f = [](const Tensor* t) { return (float*)dev(t); };
        return toErr(mnnb200_rnn_execute(mH.get(), f(inputs[0]), f(inputs[1]), f(inputs[2]), f(inputs[3]),
                                         inputs.size() >= 5 ? f(inputs[4]) : nullptr, inputs.size() >= 6 ? f(inputs[5]) : nullptr,
                                         f(outputs[0]), f(outputs[1]), outputs.size() >= 3 ? f(outputs[2]) : nullptr),
                     "rnn");
    }
private:
    const Op* mOp;
    ExecHandle mH;
};

// Cast between int32 and fp32 (CPUCast's CastDataType): an attention mask's int32 -> fp32, or fp32 -> int32 (truncation)
class CastExec : public B200Exec {
public:
    CastExec(Backend* bn, bool toFloat) : B200Exec(bn), mToFloat(toFloat) {}
    static int direction(const Op* op, const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) {
        auto cp = op->main_as_CastParam();
        if (!cp || inputs.size() != 1 || outputs.size() != 1 || isInt8(inputs[0]) || isInt8(outputs[0]) ||
            elemCount(inputs[0]) != elemCount(outputs[0]) || !sameLinear(inputs[0], outputs[0]))
            return -1;
        const auto it = inputs[0]->getType(), ot = outputs[0]->getType();
        const bool iI32 = it.code == halide_type_int && it.bits == 32, iF32 = it.code == halide_type_float && it.bits == 32;
        const bool oI32 = ot.code == halide_type_int && ot.bits == 32, oF32 = ot.code == halide_type_float && ot.bits == 32;
        const auto dst = cp->dstT();
        if (dst == DataType_DT_FLOAT && iI32 && oF32) return 1;
        if ((dst == DataType_DT_INT32 || dst == DataType_DT_INT64) && iF32 && oI32) return 0;
        return -1;
    }
    ErrorCode launch(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) override {
        const long long n = (long long)elemCount(inputs[0]);
        if (mToFloat) return toErr(mnnb200_cast_i32_f32(rt(), (const int*)dev(inputs[0]), (float*)dev(outputs[0]), n), "Cast i32 -> f32");
        return toErr(mnnb200_cast_f32_i32(rt(), (const float*)dev(inputs[0]), (int*)dev(outputs[0]), n), "Cast f32 -> i32");
    }
private:
    bool mToFloat;
};

Execution* B200Backend::onCreate(const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs, const MNN::Op* op) {
    Execution* e = nullptr;
    const bool quantOut = !outputs.empty() && TensorUtils::getDescribe(outputs[0])->quantAttr.get() != nullptr &&
                          TensorUtils::getDescribe(outputs[0])->applyQuant;
    switch (op->type()) {
        case OpType_Convolution:
        case OpType_ConvInt8:
            if (quantOut || op->type() == OpType_ConvInt8) {
                e = ConvInt8Exec::create(this, op);
            } else if (mMemoryLow && inputs.size() == 1 && op->main_as_Convolution2D() && op->main_as_Convolution2D()->quanParameter() &&
                       inputs[0]->getType().code == halide_type_float && linearFormat(inputs[0]) == MNN_DATA_FORMAT_NCHW) {
                e = LinearW8Exec::create(this, op);   // weight-quantised conv on float tensors: W8A8 only under Memory_Low, like the CPU
            }
            // float conv; under Memory_Low the CPU runs an IDST-weight conv as W8A8 dynamic quantisation
            // (ConvolutionFloatFactory.cpp:140-149), which only LinearW8Exec reproduces: such a conv is not taken in fp32
            else if (!quantOut && op->type() == OpType_Convolution && inputs.size() == 1 && isF32Nchw(inputs[0]) &&
                     !(mMemoryLow && op->main_as_Convolution2D() && op->main_as_Convolution2D()->quanParameter()))
                e = ConvF32Exec::create(this, op, inputs[0]->channel());
            break;
        case OpType_MatMul:
            if (!quantOut && inputs.size() >= 2 && op->main_as_MatMul() && inputs[0]->getType().code == halide_type_float &&
                inputs[0]->getType().bytes() == 4 && linearFormat(inputs[0]) == MNN_DATA_FORMAT_NCHW)
                e = new MatMulExec(this, op->main_as_MatMul()->transposeA(), op->main_as_MatMul()->transposeB());
            break;
        case OpType_BatchMatMul:
            if (!quantOut && inputs.size() == 2 && op->main_as_BatchMatMulParam() && isF32(inputs[0]) && isF32(inputs[1]) &&
                linearFormat(inputs[0]) == MNN_DATA_FORMAT_NCHW)
                e = new MatMulExec(this, op->main_as_BatchMatMulParam()->adjX(), op->main_as_BatchMatMulParam()->adjY());
            break;
        case OpType_Gather:
        case OpType_GatherV2:
        case OpType_GatherND:
        case OpType_GatherElements:
            if (!quantOut && GatherExec::takes(op, inputs, outputs)) e = GatherExec::create(this, op);
            break;
        case OpType_ScatterNd:
        case OpType_ScatterElements:
            if (!quantOut && ScatterExec::takes(op, inputs, outputs)) e = ScatterExec::create(this, op);
            break;
        case OpType_LSTM:
        case OpType_RNN:
            if (!quantOut && RnnExec::takes(op, inputs, outputs)) e = RnnExec::create(this, op);
            break;
        case OpType_Cast: {
            const int dir = quantOut ? -1 : CastExec::direction(op, inputs, outputs);
            if (dir >= 0) e = new CastExec(this, dir == 1);
            break;
        }
        case OpType_ConvolutionDepthwise:
        case OpType_DepthwiseConvInt8:
            if (quantOut || op->type() == OpType_DepthwiseConvInt8) e = ConvInt8Exec::create(this, op);
            else if (inputs.size() == 1 && isF32Nchw(inputs[0])) e = ConvF32Exec::create(this, op, inputs[0]->channel());
            break;
        case OpType_Deconvolution:
        case OpType_DeconvolutionDepthwise:
            if (!quantOut && DeconvF32Exec::takes(op, inputs)) e = DeconvF32Exec::create(this, op, inputs[0]->channel());
            break;
        case OpType_FloatToInt8:   // the cast kernels read/write NCHW-linear fp32 (NHWC-format tensors of <= 2 dims are the same bytes)
            // only the pipeline-inserted casts (quant info on the tensor, Pipeline.cpp:361-395); an op that carries its own
            // QuantizedFloatParam.tensorScale is left to the backup backend
            if (inputs.size() == 1 && op->main_type() == OpParameter_NONE && TensorUtils::getDescribe(outputs[0])->quantAttr.get() != nullptr &&
                (linearFormat(inputs[0]) == MNN_DATA_FORMAT_NCHW || inputs[0]->dimensions() <= 2))
                e = new FloatToInt8Exec(this);
            break;
        case OpType_Int8ToFloat:
            if (inputs.size() == 1 && op->main_type() == OpParameter_NONE && TensorUtils::getDescribe(inputs[0])->quantAttr.get() != nullptr &&
                (linearFormat(outputs[0]) == MNN_DATA_FORMAT_NCHW || outputs[0]->dimensions() <= 2))
                e = new Int8ToFloatExec(this);
            break;
        case OpType_BinaryOp:
            if (quantOut && inputs.size() == 2 && op->main_as_BinaryOp() && op->main_as_BinaryOp()->opType() == BinaryOpOperation_ADD &&
                op->main_as_BinaryOp()->activationType() == 0 && elemCount(inputs[0]) == elemCount(inputs[1]) && isInt8(inputs[0]) && isInt8(inputs[1]))
                e = new BinaryAddInt8Exec(this);
            else if (!quantOut && op->main_as_BinaryOp() && BinaryF32Exec::supports(op->main_as_BinaryOp()->opType()) &&
                     (op->main_as_BinaryOp()->activationType() == 0 || op->main_as_BinaryOp()->activationType() == 1) &&
                     BinaryF32Exec::takes(inputs, outputs))
                e = new BinaryF32Exec(this, op->main_as_BinaryOp()->opType(), op->main_as_BinaryOp()->activationType());
            break;
        case OpType_Eltwise: {
            // no coeff: the CPU takes only the {1, 0} copy form of one and fails the rest (CPUEltwise.cpp:35-45)
            auto el = op->main_as_Eltwise();
            bool ok = !quantOut && el && !(el->coeff() && el->coeff()->size() > 0) && EltwiseF32Exec::binaryOp(el->type()) >= 0 &&
                      inputs.size() >= 2 && outputs.size() == 1 && isF32(outputs[0]);
            for (auto t : inputs) ok = ok && isF32(t) && elemCount(t) == elemCount(outputs[0]) && sameLinear(t, outputs[0]);
            if (ok) e = new EltwiseF32Exec(this, EltwiseF32Exec::binaryOp(el->type()));
            break;
        }
        case OpType_UnaryOp:
            if (!quantOut && op->main_as_UnaryOp() && UnaryF32Exec::supports(op->main_as_UnaryOp()->opType()) && inputs.size() == 1 &&
                outputs.size() == 1 && isF32(inputs[0]) && isF32(outputs[0]) && elemCount(inputs[0]) == elemCount(outputs[0]) &&
                sameLinear(inputs[0], outputs[0]))
                e = new UnaryF32Exec(this, op->main_as_UnaryOp()->opType());
            break;
        case OpType_ArgMax:
        case OpType_ArgMin: {
            // the CPU's NC4HW4 input branch is the legacy Caffe form (top-k, float indices): declined, as is any top-k > 1 or
            // value output
            auto am = op->main_as_ArgMax();
            if (!quantOut && am && am->topK() == 1 && am->outMaxVal() == 0 && inputs.size() == 1 && outputs.size() == 1 &&
                isF32(inputs[0]) && outputs[0]->getType().code == halide_type_int && outputs[0]->getType().bytes() == 4 &&
                TensorUtils::getDescribe(inputs[0])->dimensionFormat != MNN_DATA_FORMAT_NC4HW4) {
                int axis = am->axis();
                if (axis < 0) axis += inputs[0]->dimensions();
                if (axis >= 0 && axis < inputs[0]->dimensions()) e = new ArgMaxExec(this, axis, op->type() == OpType_ArgMin);
            }
            break;
        }
        case OpType_Pooling:
            if (!quantOut && op->main_as_Pool() && outputs.size() == 1 && inputs[0]->getType().code == halide_type_float &&
                linearFormat(inputs[0]) == MNN_DATA_FORMAT_NCHW && inputs[0]->dimensions() == 4)
                e = new PoolF32Exec(this, op->main_as_Pool());
            else if (quantOut && op->main_as_Pool() && outputs.size() == 1 && isInt8(inputs[0]) && inputs[0]->dimensions() == 4 &&
                     !(op->main_as_Pool()->pads() && op->main_as_Pool()->pads()->size() > 0))
                e = new PoolInt8Exec(this, op->main_as_Pool());   // equal quant attrs (onSetQuantInfo): the CPU backend's int8 pooling
            break;
        case OpType_Scale:
            if (quantOut && inputs.size() == 1 && isInt8(inputs[0])) e = ScaleInt8Exec::create(this, op);
            else if (!quantOut && inputs.size() == 1 && isF32Nchw(inputs[0]) && op->main_as_Scale() && op->main_as_Scale()->scaleData() &&
                     (int)op->main_as_Scale()->scaleData()->size() == inputs[0]->channel())
                e = ScaleF32Exec::create(this, op);
            break;
        case OpType_ReLU:
            if (!quantOut && inputs.size() == 1 && inputs[0]->getType().code == halide_type_float && inputs[0]->getType().bytes() == 4)
                e = new ReluF32Exec(this, op->main_as_Relu() ? op->main_as_Relu()->slope() : 0.f);
            break;
        case OpType_Reduction: {
            auto rp = op->main_as_ReductionParam();
            int rop = -1;
            if (rp) {
                switch (rp->operation()) {
                    case ReductionType_SUM: rop = 0; break;
                    case ReductionType_MEAN: rop = 1; break;
                    case ReductionType_MAXIMUM: rop = 2; break;
                    case ReductionType_MINIMUM: rop = 3; break;
                    case ReductionType_PROD: rop = 4; break;
                    default: break;
                }
            }
            int axis = rp && rp->dim() && rp->dim()->size() == 1 ? rp->dim()->data()[0] : -1000;
            if (axis < 0 && inputs.size() >= 1) axis += inputs[0]->dimensions();
            if (!quantOut && rop >= 0 && inputs.size() == 1 && axis >= 0 && axis < inputs[0]->dimensions() &&
                inputs[0]->getType().code == halide_type_float && inputs[0]->getType().bytes() == 4 &&
                linearFormat(inputs[0]) == linearFormat(outputs[0]))
                e = new ReduceF32Exec(this, rop, axis);
            break;
        }
        case OpType_Softmax: {
            int axis = op->main_as_Axis() ? op->main_as_Axis()->axis() : 1;
            if (axis < 0) axis += inputs[0]->dimensions();
            bool inner1 = true;
            for (int i = axis + 1; i < inputs[0]->dimensions(); ++i) inner1 = inner1 && inputs[0]->length(i) == 1;
            if (quantOut && isInt8(inputs[0]) && axis == 1 && inner1) e = new SoftmaxInt8Exec(this);
            else if (!quantOut && axis >= 0 && axis < inputs[0]->dimensions() && inputs[0]->getType().code == halide_type_float &&
                     inputs[0]->getType().bytes() == 4 && (linearFormat(inputs[0]) == MNN_DATA_FORMAT_NCHW || inputs[0]->dimensions() <= 2))
                e = new SoftmaxF32Exec(this, axis);   // <= 2 dims: NHWC-format tensors (TF models' logits) are the same bytes
            break;
        }
        case OpType_Raster: {
            bool ok = !outputs.empty() && outputs[0]->getType().bytes() == 4 && !quantOut;
            for (auto t : inputs) ok = ok && t->getType().bytes() == 4 && !isInt8(t);
            if (ok) e = new RasterExec(this);
            break;
        }
        case OpType_LayerNorm:
            if (!quantOut && LayerNormF32Exec::takes(op, inputs, outputs)) e = LayerNormF32Exec::create(this, op);
            break;
        case OpType_RoPE:
            if (!quantOut && RoPEF32Exec::takes(op, inputs, outputs)) e = RoPEF32Exec::create(this, op);
            break;
        case OpType_Interp:
            if (!quantOut && InterpF32Exec::takes(inputs, outputs)) e = InterpF32Exec::create(this, op);
            break;
        case OpType_GridSample:
            if (!quantOut && GridSampleF32Exec::takes(op, inputs, outputs)) e = GridSampleF32Exec::create(this, op);
            break;
        default:
            break;
    }
    if (e) {
        ++g_created;
    } else {
        ++g_declined;
        MNN_PRINT("mnn_b200 plugin: no execution for %s (%s), quantOut=%d\n", EnumNameOpType(op->type()),
                  op->name() ? op->name()->c_str() : "", (int)quantOut);
    }
    return e;
}

// ------------------------------------------------------------------------------------------------ Runtime + creator
class B200Runtime : public Runtime {
public:
    explicit B200Runtime(mnnb200_runtime* h) : mH(h) {}
    ~B200Runtime() override { mnnb200_runtime_destroy(mH); }
    Backend* onCreate(const BackendConfig* config = nullptr, Backend* = nullptr) const override {
        const bool low = config ? config->memory == BackendConfig::Memory_Low : mMemoryLow;
        return new B200Backend(this, mH, low);
    }
    // device time between the last forward's onExecuteBegin and onExecuteEnd (CUDA events on the runtime's stream)
    float onGetLastGpuTimeMs() const override { return mnnb200_runtime_last_gpu_ms(mH); }
    void setDefaultMemoryLow(bool v) { mMemoryLow = v; }
    void onGabageCollect(int) override {}
    CompilerType onGetCompilerType() const override { return Compiler_Geometry; }
    float onGetMemoryInMB() override { return 0.f; }
private:
    mnnb200_runtime* mH;
    bool mMemoryLow = false;
};
const Runtime* B200Backend::getRuntime() { return mRuntime; }

class B200RuntimeCreator : public RuntimeCreator {
public:
    Runtime* onCreate(const Backend::Info& info) const override {
        int device = 0;
        if (info.user && info.user->sharedContext) device = ((MNNDeviceContext*)info.user->sharedContext)->deviceId;
        mnnb200_runtime* h = nullptr;
        if (mnnb200_runtime_create(device, nullptr, &h) != MNNB200_OK) {   // no sm_90 device: unavailable, never a CPU path
            MNN_ERROR("mnn_b200: %s\n", mnnb200_last_error());
            return nullptr;
        }
        auto rt = new B200Runtime(h);
        rt->setDefaultMemoryLow(info.user && info.user->memory == BackendConfig::Memory_Low);
        return rt;
    }
    // Which ops run in int8 here (RuntimeCreator::onSetQuantInfo, Backend.hpp:433-441; model: CPUBackend.cpp:898-980).
    bool onSetQuantInfo(const Op* op, const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) const override {
        if (op == nullptr) return true;   // capability probe (Pipeline.cpp:249)
        bool res = support(op, inputs, outputs);
        for (auto t : outputs) TensorUtils::getDescribe(t)->applyQuant = res;
        return res;
    }
private:
    static bool support(const Op* op, const std::vector<Tensor*>& inputs, const std::vector<Tensor*>& outputs) {
        for (auto t : inputs) {
            auto des = TensorUtils::getDescribe(t);
            if (des->quantAttr == nullptr || des->quantAttr->type != DataType_DT_INT8) return false;
        }
        switch (op->type()) {
            case OpType_Convolution:
            case OpType_ConvolutionDepthwise:
                return inputs.size() == 1 && !(op->main_as_Convolution2D() && op->main_as_Convolution2D()->weight() != nullptr);
            case OpType_ConvInt8:
            case OpType_DepthwiseConvInt8:
                return true;
            case OpType_Softmax:
                return true;
            case OpType_BinaryOp:
                return op->main_as_BinaryOp() && op->main_as_BinaryOp()->opType() == BinaryOpOperation_ADD;
            case OpType_Scale:      // CPUBackend.cpp:957-958
                return inputs.size() == 1 && op->main_as_Scale() != nullptr;
            case OpType_Pooling: {  // CPUBackend.cpp:926-936: int8 only between tensors with the same scale and zero point
                auto qi = TensorUtils::getDescribe(inputs[0])->quantAttr.get();
                auto qo = outputs.empty() ? nullptr : TensorUtils::getDescribe(outputs[0])->quantAttr.get();
                if (!qi || !qo || qi->scale != qo->scale || qi->zero != qo->zero) return false;
                auto pl = op->main_as_Pool();
                return pl && (pl->type() == PoolType_MAXPOOL || pl->type() == PoolType_AVEPOOL) && !(pl->pads() && pl->pads()->size() > 0) &&
                       inputs[0]->dimensions() == 4;
            }
            default:
                return false;   // Raster / ReLU stay float between casts here: with equal attrs dequantise -> copy/relu -> requantise
                                // reproduces the int8 result exactly, with different attrs the CPU does the same
        }
    }
};

struct Registrar {
    Registrar() {
        static std::once_flag once;
        std::call_once(once, [] { MNNInsertExtraRuntimeCreator(MNN_FORWARD_CUDA, new B200RuntimeCreator, false); });
    }
} g_registrar;

}  // namespace
}  // namespace MNN

extern "C" __attribute__((visibility("default"))) void mnnb200_plugin_stats(int* created, int* declined) {
    if (created) *created = MNN::g_created;
    if (declined) *declined = MNN::g_declined;
}
