// rnn.cu -- the recurrence of fp32 LSTM and RNN (OpType_LSTM / OpType_RNN of ONNX models) for libmnn_b200_rnn.so: one launch
// runs all T steps of both directions.
//
// The reference lowers the op in GeometryLSTM.cpp (_ComputeLSTMOnnx) into a projection Gate = X W^T + B over all T * B rows and
// a sequential loop that, per step, computes HR = h_prev R^T, z = Gate_t + HR and
//   LSTM (gate rows i, o, f, c): i = sigmoid(z_i), g = tanh(z_c), f = sigmoid(z_f), o = sigmoid(z_o),
//                                c = i * g + f * c_prev (two products, one sum), h = tanh(c) * o;
//   RNN: h = tanh(z).
// Without h0 the first step has no HR term; without c0 no f * c term.  Direction 1 reads X reversed in time and writes Y at
// T - 1 - s.  The projection is the split-TF32 MatMul of libmnn_b200.so (rnn_capi.cu); this file is the loop.
//
// rnn_recur_f32_kernel<CELL, RESIDENT, KS>: one thread-block cluster per (direction, batch group) walks the T steps.  Each CTA
// of the cluster owns a slice of hidden units and all gate rows of R for them, so its cell state stays in its shared memory for
// the whole sequence.  Every CTA holds the group's whole h_prev, double-buffered: a step computes the slice's gates from the
// local copy, then stores the slice's new h into the other buffer of every CTA of the cluster (distributed shared memory,
// mapa + st.shared::cluster), arrives on each CTA's mbarrier of that buffer and waits on its own, then writes the slice to Y.
// The mbarrier rather than barrier.cluster: its wait is bounded and traps, so a lost arrive fails the launch instead of hanging
// the device.  A one-CTA cluster stores locally and passes __syncthreads.  RESIDENT: the CTA's R rows are loaded into shared
// memory once per launch; otherwise they are read from global memory (L2) every step.  Batch groups and directions are
// independent clusters: no grid-wide barrier, no cooperative launch.
//
// Every gate's dot product h_prev . R_row is 8 partial sums over k mod 8, each in increasing k with fp32 FMA, combined as
// ((s0 + s1) + (s2 + s3)) + ((s4 + s5) + (s6 + s7)) (gate_dots): the result does not depend on how many threads (KS) share
// one dot product, on the cluster, the batch group or T.  The cell update is __fmul_rn / __fadd_rn in the reference's order,
// and sigmoid / tanh are UnaryOp's (activations.cuh).
#include <algorithm>

#include "activations.cuh"
#include "common.cuh"
#include "hopper_common.cuh"
#include "host_util.h"
#include "rnn_ops.h"

namespace mnnb200 {
namespace {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void st_cluster(uint32_t addr, float v) {
    asm volatile("st.shared::cluster.f32 [%0], %1;\n" ::"r"(addr), "f"(v) : "memory");
}
// mbarrier wait with cluster-scope acquire (the stores it orders come from other CTAs), bounded as hop::mbar_wait is
__device__ __forceinline__ uint32_t mbar_try_wait_cluster(uint32_t bar, uint32_t parity, uint32_t hint_ns) {
    uint32_t done;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2, %3;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(done)
        : "r"(bar), "r"(parity), "r"(hint_ns)
        : "memory");
    return done;
}
__device__ __forceinline__ void mbar_wait_cluster(uint32_t bar, uint32_t parity) {
    if (mbar_try_wait_cluster(bar, parity, 0u)) return;
    long long t0 = 0;
    while (!mbar_try_wait_cluster(bar, parity, 100000u)) {
        const long long now = clock64();
        if (t0 == 0) t0 = now;
        else if (now - t0 > 8000000000ll) __trap();
    }
}

// z[q] = sum_k rrow[q * pitch + k] * hv[k] over k < n for the NG gate rows, by KS consecutive lanes (s = this lane's index
// among them): lane s keeps the partial sums of k = a mod 8 for a = s, s + KS, ..., the lanes combine bits 0 .. log2(KS) of a
// by shuffles and then each lane the remaining bits in registers, lowest bit first.  Every lane of the KS returns the sums.
// All 32 lanes of the warp call it (live or not) for the shuffles.
template <int NG, int KS>
__device__ __forceinline__ void gate_dots(float (&z)[NG], const float* __restrict__ rrow, size_t pitch,
                                          const float* __restrict__ hv, int n, int s, bool live) {
    constexpr int M = kRnnPartials / KS;
    float a[NG][M];
#pragma unroll
    for (int q = 0; q < NG; ++q)
#pragma unroll
        for (int m = 0; m < M; ++m) a[q][m] = 0.f;
    if (live) {
        for (int k0 = 0; k0 < n; k0 += kRnnPartials) {
#pragma unroll
            for (int m = 0; m < M; ++m) {
                const int k = k0 + s + KS * m;
                if (k < n) {
                    const float hk = hv[k];
#pragma unroll
                    for (int q = 0; q < NG; ++q) a[q][m] = __fmaf_rn(rrow[q * pitch + k], hk, a[q][m]);
                }
            }
        }
    }
#pragma unroll
    for (int q = 0; q < NG; ++q) {
#pragma unroll
        for (int lvl = 1; lvl < KS; lvl <<= 1)
#pragma unroll
            for (int m = 0; m < M; ++m) a[q][m] = __fadd_rn(a[q][m], __shfl_xor_sync(0xffffffffu, a[q][m], lvl));
#pragma unroll
        for (int st = 1; st < M; st <<= 1)
#pragma unroll
            for (int m = 0; m < M; m += 2 * st) a[q][m] = __fadd_rn(a[q][m], a[q][m + st]);
        z[q] = a[q][0];
    }
}

template <int CELL, bool RESIDENT, int KS>
__global__ void __launch_bounds__(kRnnThreads, 1) rnn_recur_f32_kernel(const RnnParams p) {
    constexpr int NG = CELL == 0 ? 4 : 1;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw);          // [2]: the h buffers' "all slices stored" barriers
    float* hbuf = reinterpret_cast<float*>(smem_raw + 16);           // [2][rows][H]
    float* cst = hbuf + 2 * p.rows * p.h;                            // [rows][hs]
    float* rs = cst + p.rows * p.hs;                                  // [NG][hs][rstride] (RESIDENT)
    const int H = p.h, cs = p.cs, rank = cs > 1 ? (int)hop::cluster_rank() : 0;
    const int dir = blockIdx.z, b0 = blockIdx.y * p.rows, nb = min(p.rows, p.b - b0);
    const int j0 = rank * p.hs, nj = max(0, min(p.hs, H - j0));
    const int tid = threadIdx.x, nt = blockDim.x;
    const size_t gpitch = (size_t)p.d * NG * H;

    for (int i = tid; i < nb * H; i += nt) hbuf[i] = p.h0 ? p.h0[((size_t)dir * p.b + b0) * H + i] : 0.f;
    for (int i = tid; i < nb * nj; i += nt) {
        const int b = i / nj, jj = i % nj;
        cst[b * p.hs + jj] = p.c0 ? p.c0[((size_t)dir * p.b + b0 + b) * H + j0 + jj] : 0.f;
    }
    if (RESIDENT) {
        for (int i = tid; i < NG * nj * H; i += nt) {
            const int row = i / H, k = i % H, q = row / nj, jj = row % nj;
            rs[(q * p.hs + jj) * p.rstride + k] = p.r[((size_t)dir * NG * H + q * H + j0 + jj) * H + k];
        }
    }
    if (cs > 1) {
        if (tid == 0) {
            hop::mbar_init(smem_u32(&bars[0]), cs);
            hop::mbar_init(smem_u32(&bars[1]), cs);
            asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
        }
        hop::cluster_sync_all();   // every CTA's barriers are initialised before anyone arrives on them
    } else {
        __syncthreads();
    }

    const int items = nb * nj, groups = nt / KS, s = tid % KS;
    for (int step = 0; step < p.t; ++step) {
        const int cur = step & 1, nxt = cur ^ 1;
        const int pos = dir ? p.t - 1 - step : step;
        const bool hr = step > 0 || p.h0 != nullptr, fc = step > 0 || p.c0 != nullptr;
        const float* hc = hbuf + cur * p.rows * H;
        for (int base = 0; base < items; base += groups) {
            const int item = base + tid / KS;
            const bool live = item < items;
            const int b = live ? item / nj : 0, jj = live ? item % nj : 0;
            float gv[NG];
            if (live && s == 0) {
                const float* gr = p.g + ((size_t)pos * p.b + b0 + b) * gpitch + (size_t)dir * NG * H + j0 + jj;
#pragma unroll
                for (int q = 0; q < NG; ++q) gv[q] = gr[(size_t)q * H];
            }
            float z[NG];
            if (RESIDENT)
                gate_dots<NG, KS>(z, rs + jj * p.rstride, (size_t)p.hs * p.rstride, hc + b * H, H, s, live && hr);
            else
                gate_dots<NG, KS>(z, p.r + ((size_t)dir * NG * H + j0 + jj) * H, (size_t)H * H, hc + b * H, H, s, live && hr);
            if (live && s == 0) {
#pragma unroll
                for (int q = 0; q < NG; ++q) z[q] = hr ? __fadd_rn(gv[q], z[q]) : gv[q];
                float hv;
                if (CELL == 0) {
                    const float ig = sigmoid_f32(z[0]), og = sigmoid_f32(z[1]), fg = sigmoid_f32(z[2]), gg = tanh_f32(z[3]);
                    float c = __fmul_rn(ig, gg);
                    if (fc) c = __fadd_rn(c, __fmul_rn(fg, cst[b * p.hs + jj]));
                    cst[b * p.hs + jj] = c;
                    hv = __fmul_rn(tanh_f32(c), og);
                } else {
                    hv = tanh_f32(z[0]);
                }
                float* dst = hbuf + nxt * p.rows * H + b * H + j0 + jj;
                if (cs == 1) {
                    *dst = hv;
                } else {
                    const uint32_t a = smem_u32(dst);
                    for (int r = 0; r < cs; ++r) st_cluster(hop::mapa(a, (uint32_t)r), hv);
                }
            }
        }
        if (cs == 1) {
            __syncthreads();
        } else {
            asm volatile("fence.acq_rel.cluster;\n" ::: "memory");
            __syncthreads();
            const uint32_t bar = smem_u32(&bars[nxt]);
            if (tid == 0)
                for (int r = 0; r < cs; ++r) hop::mbar_arrive_cluster(hop::mapa(bar, (uint32_t)r));
            mbar_wait_cluster(bar, (uint32_t)((step >> 1) & 1));   // step s uses buffer nxt for the (s / 2 + 1)-th time
        }
        const float* hn = hbuf + nxt * p.rows * H;
        for (int i = tid; i < nb * nj; i += nt) {
            const int b = i / nj, jj = i % nj;
            p.y[(((size_t)pos * p.d + dir) * p.b + b0 + b) * H + j0 + jj] = hn[b * H + j0 + jj];
        }
    }
    // no peer touches this CTA's shared memory after the last wait: every store into it precedes an arrive it waited for
    const float* hl = hbuf + (p.t & 1) * p.rows * H;
    for (int i = tid; i < nb * nj; i += nt) {
        const int b = i / nj, jj = i % nj;
        const size_t o = ((size_t)dir * p.b + b0 + b) * H + j0 + jj;
        if (p.yh) p.yh[o] = hl[b * H + j0 + jj];
        if (CELL == 0 && p.yc) p.yc[o] = cst[b * p.hs + jj];
    }
}

// An RNN whose items fit 8 threads each (at most 32 per CTA) has a slice of at most 32 rows of R, which always fits in shared
// memory: that kernel streams nothing, so <1, false, 8> is not built (rnn_choose_plan never picks it).
template <int CELL, bool RESIDENT>
const void* kernel_ks(int ks) {
    switch (ks) {
        case 1: return (const void*)rnn_recur_f32_kernel<CELL, RESIDENT, 1>;
        case 2: return (const void*)rnn_recur_f32_kernel<CELL, RESIDENT, 2>;
        case 4: return (const void*)rnn_recur_f32_kernel<CELL, RESIDENT, 4>;
        default:
            if constexpr (CELL == 1 && !RESIDENT) return nullptr;
            else return (const void*)rnn_recur_f32_kernel<CELL, RESIDENT, 8>;
    }
}
const void* kernel_of(int cell, const RnnPlan& pl) {
    if (cell == 0) return pl.resident ? kernel_ks<0, true>(pl.ks) : kernel_ks<0, false>(pl.ks);
    return pl.resident ? kernel_ks<1, true>(pl.ks) : kernel_ks<1, false>(pl.ks);
}

cudaLaunchConfig_t config_of(const RnnPlan& pl, int d, cudaStream_t s, cudaLaunchAttribute* attr) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(pl.cs, pl.groups, d);
    cfg.blockDim = dim3(pl.threads);
    cfg.dynamicSmemBytes = pl.smem;
    cfg.stream = s;
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = pl.cs;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cfg;
}

int ks_of(int items) {
    int ks = kRnnPartials;
    while (ks > 1 && items * ks > kRnnThreads) ks >>= 1;
    return ks;
}

// the plan's CTA geometry and shared memory for cluster size cs
RnnPlan shape(int cell, int h, int rows, int groups, int cs, bool resident) {
    RnnPlan pl;
    pl.cs = cs;
    pl.groups = groups;
    pl.rows = rows;
    pl.hs = (h + cs - 1) / cs;
    const int items = rows * pl.hs;
    pl.ks = ks_of(items);
    pl.threads = std::min(kRnnThreads, (items * pl.ks + 31) / 32 * 32);
    pl.resident = resident ? 1 : 0;
    const int ng = cell == 0 ? 4 : 1;
    const long long rstride = h + (((pl.ks - h) % 32) + 32) % 32;   // rows of the resident slice pitch KS banks apart
    long long bytes = 16 + 4LL * (2LL * rows * h + (long long)rows * pl.hs);
    if (resident) bytes += 4LL * ng * pl.hs * rstride;
    pl.smem = bytes > 0x7fffffffLL ? 0x7fffffff : (int)bytes;
    pl.rstride = (int)rstride;
    return pl;
}

}  // namespace

bool rnn_choose_plan(int cell, int b, int h, int d, int sms, int smem_cap, RnnFits fits, void* ctx, RnnPlan* out) {
    const int max_rows = std::max(1, std::min(kRnnMaxRows, 24576 / h));
    const int groups = (b + max_rows - 1) / max_rows, rows = (b + groups - 1) / groups;
    int top = 1;                                        // the largest power-of-two cluster with a unit per CTA
    while (top * 2 <= std::min(h, kRnnMaxCluster)) top *= 2;
    int cs = 1;                                         // enough CTAs that each has at most 32 items
    while (cs < top && (long long)rows * ((h + cs - 1) / cs) > 32) cs *= 2;
    while (cs > 1 && (long long)cs * groups * d > sms) cs /= 2;   // one CTA per SM where the card has them
    for (;;) {
        RnnPlan pl = shape(cell, h, rows, groups, cs, false);
        for (int c = cs; c <= top; c *= 2) {            // R resident at the smallest cluster, from cs up, whose slice fits
            const RnnPlan r = shape(cell, h, rows, groups, c, true);
            if (r.smem <= smem_cap) {
                pl = r;
                break;
            }
        }
        if (pl.smem <= smem_cap && (!fits || fits(cell, pl, ctx))) {
            *out = pl;
            return true;
        }
        if (cs == 1) return false;
        cs /= 2;
        top = cs;
    }
}

cudaError_t rnn_max_active_clusters(int cell, const RnnPlan& pl, int smem_cap, int* clusters) {
    const void* k = kernel_of(cell, pl);
    if (!k) return cudaErrorInvalidValue;
    cudaError_t e = ensure_max_dynamic_smem(k, smem_cap);
    if (e != cudaSuccess) return e;
    if ((e = cudaFuncSetAttribute(k, cudaFuncAttributeNonPortableClusterSizeAllowed, 1)) != cudaSuccess) return e;
    cudaLaunchAttribute attr[1];
    RnnPlan one = pl;   // what fits depends on one cluster, not on the grid (whose y may pass 65535 here: resize refuses that)
    one.groups = 1;
    const cudaLaunchConfig_t cfg = config_of(one, 1, nullptr, attr);
    return cudaOccupancyMaxActiveClusters(clusters, k, &cfg);
}

cudaError_t launch_rnn_recur(int cell, const RnnParams& p, const RnnPlan& pl, cudaStream_t s) {
    cudaLaunchAttribute attr[1];
    cudaLaunchConfig_t cfg = config_of(pl, p.d, s, attr);
    void* args[] = {const_cast<RnnParams*>(&p)};
    ++g_launch_count;
    return cudaLaunchKernelExC(&cfg, kernel_of(cell, pl), args);
}

}  // namespace mnnb200
