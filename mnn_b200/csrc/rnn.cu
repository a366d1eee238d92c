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
// and sigmoid / tanh are UnaryOp's (activations.cuh).  gate_dots, the cluster store and wait and the plan search are shared
// with gru.cu (recur_common.cuh).
#include "activations.cuh"
#include "common.cuh"
#include "recur_common.cuh"

namespace mnnb200 {
namespace {

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

}  // namespace

bool rnn_choose_plan(int cell, int b, int h, int d, int sms, int smem_cap, RnnFits fits, void* ctx, RnnPlan* out) {
    const RecurSmem m{cell == 0 ? 4 : 1, 2, 0};
    return recur_choose_plan(m, b, h, d, sms, smem_cap, [&](const RnnPlan& pl) { return !fits || fits(cell, pl, ctx); }, out);
}

cudaError_t rnn_max_active_clusters(int cell, const RnnPlan& pl, int smem_cap, int* clusters) {
    return recur_max_active_clusters(kernel_of(cell, pl), pl, smem_cap, clusters);
}

cudaError_t launch_rnn_recur(int cell, const RnnParams& p, const RnnPlan& pl, cudaStream_t s) {
    cudaLaunchAttribute attr[1];
    cudaLaunchConfig_t cfg = recur_config(pl, p.d, s, attr);
    void* args[] = {const_cast<RnnParams*>(&p)};
    ++g_launch_count;
    return cudaLaunchKernelExC(&cfg, kernel_of(cell, pl), args);
}

}  // namespace mnnb200
