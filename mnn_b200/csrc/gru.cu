// gru.cu -- the fp32 GRU (OpType_RNNSequenceGRU) for libmnn_b200_gru.so: a weight repack, and the recurrence of all T steps
// and both directions in one launch.  The projection between them is the split-TF32 MatMul of libmnn_b200.so (gru_capi.cu).
//
// The reference (CPURNNSequenceGRU.cpp) runs per step and batch row, rounding every line in fp32:
//   g = [x_t, h] Wg + bg;  g = g + rb[0:2H];  z = sigmoid(g[0:H]);  r = sigmoid(g[H:2H])
//   linear_before_reset 0: n_pre = [x_t, r * h] Wc + (rb[2H:3H] + bc)
//   linear_before_reset 1: n_pre = ((r * (h Wc[I:] + rb[2H:3H])) + x_t Wc[0:I]) + bc
//   n = tanh(n_pre);  h' = ((h - n) * z) + n
// Here the x parts of all T steps are one MatMul, P = X Wx + (bg | 0) (P_zr carries bg, P_n no bias), and each step adds the
// h parts: g = (P_zr + h . R_zr) + rb_zr, and n_pre = ((P_n + rh . R_n) + (rb_h + bc)) or ((r * (h . R_n + rb_h)) + P_n) + bc.
// Without h0 the first step has no h term (the reference multiplies by zeros).  Direction 1 reads X from t = T - 1 down and
// writes Y at T - 1 - s; Y_h is each direction's last h (Y[T - 1][0] and Y[0][1]).
//
// gru_recur_f32_kernel<LBR, RESIDENT, KS> is rnn_recur_f32_kernel's structure (rnn.cu): one cluster per (direction, batch
// group), each CTA owning a slice of hidden units and their three gate rows of R (z, r, n), h_prev double-buffered in every
// CTA and exchanged through distributed shared memory and the bounded mbarrier wait each step (recur_common.cuh).
//   LBR = 1: one exchange per step; the three dot products h . R_q run together.
//   LBR = 0: the candidate's product reads r * h_prev of every unit, so a step has two exchanges.  Phase A computes z and r of
//   the slice, keeps z, and stores r * h_prev of the slice into every CTA's rh buffer, then arrives on every CTA's rh barrier
//   and waits on its own.  Phase B computes rh . R_n and h', and exchanges h' as LBR = 1 does.
//   rh is single-buffered, and so is its barrier (one phase per step).  A peer stores into this CTA's rh (and arrives on its
//   rh barrier) for step s + 1 only after its h wait of step s, which needs this CTA's h arrive of step s, which follows this
//   CTA's last read of rh in step s (the fence and __syncthreads before the arrive).  And every CTA issues its rh arrives of
//   step s before its h arrive of step s, so when any arrive of step s + 1 reaches a barrier, all cs arrives of step s have
//   reached it: phase s is complete and the parity wait on it cannot be overtaken.
// Every dot product is gate_dots' fixed order (8 partial sums over k mod 8, combined pairwise): the outputs do not depend on
// KS, the cluster, the batch group or T.  The cell update is __fmul_rn / __fadd_rn / __fsub_rn in the reference's order, and
// sigmoid / tanh are UnaryOp's (activations.cuh).
#include "activations.cuh"
#include "common.cuh"
#include "gru_ops.h"
#include "recur_common.cuh"

namespace mnnb200 {
namespace {

constexpr int kTile = 32;

// p.in[k] by selects: a dynamic index into the parameter block would copy it to the stack
__device__ __forceinline__ const float* param_in(const GruRepackParams& p, int k) {
    const float* r = p.in[0];
#pragma unroll
    for (int i = 1; i < 2 * kGruParamsPerDir; ++i) r = i == k ? p.in[i] : r;
    return r;
}

// Wg / Wc of direction z / 3 (gate z % 3: z, r from Wg's columns q H .., n from Wc) as a [I + H][H] source, tiled 32 x 32:
// rows k < I go to wx unchanged, rows k >= I transposed to r.  Block (0, 0) of each (direction, gate) also writes its biases.
__global__ void __launch_bounds__(kTile * 8) gru_repack_f32_kernel(const GruRepackParams p) {
    __shared__ float tile[kTile][kTile + 1];
    const int I = p.i, H = p.h, dz = blockIdx.z / 3, q = blockIdx.z % 3;
    const float* src = q < 2 ? param_in(p, kGruParamsPerDir * dz) + q * H : param_in(p, kGruParamsPerDir * dz + 2);
    const size_t pitch = q < 2 ? 2 * (size_t)H : (size_t)H;
    const size_t wxpitch = (size_t)p.d * 3 * H;
    const int j0 = blockIdx.x * kTile, tx = threadIdx.x % kTile, ty = threadIdx.x / kTile;
    const int ktiles = (I + H + kTile - 1) / kTile;
    for (int kt = blockIdx.y; kt < ktiles; kt += gridDim.y) {
        const int k0 = kt * kTile;
        __syncthreads();
        for (int yy = ty; yy < kTile; yy += 8) {
            const int k = k0 + yy, j = j0 + tx;
            if (k < I + H && j < H) {
                const float v = src[k * pitch + j];
                tile[yy][tx] = v;
                if (k < I) p.wx[k * wxpitch + (size_t)(dz * 3 + q) * H + j] = v;
            }
        }
        __syncthreads();
        for (int yy = ty; yy < kTile; yy += 8) {
            const int j = j0 + yy, k = k0 + tx;
            if (j < H && k >= I && k < I + H) p.r[((size_t)(dz * 3 + q) * H + j) * H + (k - I)] = tile[tx][yy];
        }
    }
    if (blockIdx.x == 0 && blockIdx.y == 0) {
        const float* bg = param_in(p, kGruParamsPerDir * dz + 1);
        const float* bc = param_in(p, kGruParamsPerDir * dz + 3);
        const float* rb = param_in(p, kGruParamsPerDir * dz + 4);
        for (int j = threadIdx.x; j < H; j += blockDim.x) {
            p.bx[(size_t)(dz * 3 + q) * H + j] = q < 2 ? bg[q * H + j] : 0.f;
            p.kb[(size_t)dz * 4 * H + q * H + j] = rb[q * H + j];
            if (q == 2) p.kb[(size_t)dz * 4 * H + 3 * H + j] = bc[j];
        }
    }
}

template <bool LBR, bool RESIDENT, int KS>
__global__ void __launch_bounds__(kRnnThreads, 1) gru_recur_f32_kernel(const GruParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw);          // [2]: the h buffers' barriers; [2] (LBR = 0): rh's
    const int H = p.h, cs = p.cs, rank = cs > 1 ? (int)hop::cluster_rank() : 0;
    float* hbuf = reinterpret_cast<float*>(smem_raw + (LBR ? 16 : 32));   // [2][rows][H]
    float* zst = hbuf + 2 * p.rows * H;                                    // [rows][hs]: z between the phases (LBR = 0)
    float* rh = zst + p.rows * p.hs;                                       // [rows][H]: r * h_prev (LBR = 0)
    float* rs = rh + (LBR ? 0 : p.rows * H);                               // [3][hs][rstride] (RESIDENT)
    const int dir = blockIdx.z, b0 = blockIdx.y * p.rows, nb = min(p.rows, p.b - b0);
    const int j0 = rank * p.hs, nj = max(0, min(p.hs, H - j0));
    const int tid = threadIdx.x, nt = blockDim.x;
    const size_t gpitch = (size_t)p.d * 3 * H;
    const float* kb = p.kb + (size_t)dir * 4 * H + j0;

    for (int i = tid; i < nb * H; i += nt) hbuf[i] = p.h0 ? p.h0[((size_t)dir * p.b + b0) * H + i] : 0.f;
    if (RESIDENT) {
        for (int i = tid; i < 3 * nj * H; i += nt) {
            const int row = i / H, k = i % H, q = row / nj, jj = row % nj;
            rs[(q * p.hs + jj) * p.rstride + k] = p.r[((size_t)dir * 3 * H + q * H + j0 + jj) * H + k];
        }
    }
    if (cs > 1) {
        if (tid == 0) {
            for (int i = 0; i < (LBR ? 2 : 3); ++i) hop::mbar_init(smem_u32(&bars[i]), cs);
            asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
        }
        hop::cluster_sync_all();   // every CTA's barriers are initialised before anyone arrives on them
    } else {
        __syncthreads();
    }
    // gate q's rows of R for unit jj (pitch between gates)
    const float* rbase = RESIDENT ? rs : p.r + (size_t)dir * 3 * H * H + (size_t)j0 * H;
    const int rrow = RESIDENT ? p.rstride : H;
    const size_t rpitch = RESIDENT ? (size_t)p.hs * p.rstride : (size_t)H * H;

    // every CTA's copy of dst (rank r's shared memory) gets v; a one-CTA cluster stores locally
    auto store_all = [&](float* dst, float v) {
        if (cs == 1) {
            *dst = v;
        } else {
            const uint32_t a = smem_u32(dst);
            for (int r = 0; r < cs; ++r) st_cluster(hop::mapa(a, (uint32_t)r), v);
        }
    };
    // every CTA's stores precede every CTA's arrive on barrier `bar`; then this CTA waits for the phase of `parity`
    auto exchange = [&](uint64_t* bar, uint32_t parity) {
        if (cs == 1) {
            __syncthreads();
        } else {
            asm volatile("fence.acq_rel.cluster;\n" ::: "memory");
            __syncthreads();
            const uint32_t a = smem_u32(bar);
            if (tid == 0)
                for (int r = 0; r < cs; ++r) hop::mbar_arrive_cluster(hop::mapa(a, (uint32_t)r));
            mbar_wait_cluster(a, parity);
        }
    };

    const int items = nb * nj, groups = nt / KS, s = tid % KS;
    for (int step = 0; step < p.t; ++step) {
        const int cur = step & 1, nxt = cur ^ 1;
        const int pos = dir ? p.t - 1 - step : step;
        const bool hr = step > 0 || p.h0 != nullptr;
        const float* hc = hbuf + cur * p.rows * H;
        if (LBR) {
            for (int base = 0; base < items; base += groups) {
                const int item = base + tid / KS;
                const bool live = item < items;
                const int b = live ? item / nj : 0, jj = live ? item % nj : 0;
                float d3[3];
                gate_dots<3, KS>(d3, rbase + jj * rrow, rpitch, hc + b * H, H, s, live && hr);
                if (live && s == 0) {
                    const float* gr = p.g + ((size_t)pos * p.b + b0 + b) * gpitch + (size_t)dir * 3 * H + j0 + jj;
                    const float gz = hr ? __fadd_rn(gr[0], d3[0]) : gr[0], gg = hr ? __fadd_rn(gr[H], d3[1]) : gr[H];
                    const float z = sigmoid_f32(__fadd_rn(gz, kb[jj])), r = sigmoid_f32(__fadd_rn(gg, kb[H + jj]));
                    const float hn = hr ? __fadd_rn(d3[2], kb[2 * H + jj]) : kb[2 * H + jj];
                    const float n = tanh_f32(__fadd_rn(__fadd_rn(__fmul_rn(r, hn), gr[2 * H]), kb[3 * H + jj]));
                    const float hp = hc[b * H + j0 + jj];
                    store_all(hbuf + nxt * p.rows * H + b * H + j0 + jj, __fadd_rn(__fmul_rn(__fsub_rn(hp, n), z), n));
                }
            }
        } else {
            for (int base = 0; base < items; base += groups) {   // phase A: z, r and r * h_prev of the slice
                const int item = base + tid / KS;
                const bool live = item < items;
                const int b = live ? item / nj : 0, jj = live ? item % nj : 0;
                float d2[2];
                gate_dots<2, KS>(d2, rbase + jj * rrow, rpitch, hc + b * H, H, s, live && hr);
                if (live && s == 0) {
                    const float* gr = p.g + ((size_t)pos * p.b + b0 + b) * gpitch + (size_t)dir * 3 * H + j0 + jj;
                    const float gz = hr ? __fadd_rn(gr[0], d2[0]) : gr[0], gg = hr ? __fadd_rn(gr[H], d2[1]) : gr[H];
                    zst[b * p.hs + jj] = sigmoid_f32(__fadd_rn(gz, kb[jj]));
                    const float r = sigmoid_f32(__fadd_rn(gg, kb[H + jj]));
                    store_all(rh + b * H + j0 + jj, __fmul_rn(r, hc[b * H + j0 + jj]));
                }
            }
            exchange(&bars[2], (uint32_t)(step & 1));
            for (int base = 0; base < items; base += groups) {   // phase B: the candidate over every unit's r * h_prev, h'
                const int item = base + tid / KS;
                const bool live = item < items;
                const int b = live ? item / nj : 0, jj = live ? item % nj : 0;
                float d1[1];
                gate_dots<1, KS>(d1, rbase + 2 * rpitch + jj * rrow, 0, rh + b * H, H, s, live && hr);
                if (live && s == 0) {
                    const float gn = p.g[((size_t)pos * p.b + b0 + b) * gpitch + (size_t)dir * 3 * H + 2 * H + j0 + jj];
                    const float pre = hr ? __fadd_rn(gn, d1[0]) : gn;
                    const float n = tanh_f32(__fadd_rn(pre, __fadd_rn(kb[2 * H + jj], kb[3 * H + jj])));
                    const float hp = hc[b * H + j0 + jj], z = zst[b * p.hs + jj];
                    store_all(hbuf + nxt * p.rows * H + b * H + j0 + jj, __fadd_rn(__fmul_rn(__fsub_rn(hp, n), z), n));
                }
            }
        }
        exchange(&bars[nxt], (uint32_t)((step >> 1) & 1));   // step s uses buffer nxt for the (s / 2 + 1)-th time
        if (p.y) {
            const float* hn = hbuf + nxt * p.rows * H;
            for (int i = tid; i < nb * nj; i += nt) {
                const int b = i / nj, jj = i % nj;
                p.y[(((size_t)pos * p.d + dir) * p.b + b0 + b) * H + j0 + jj] = hn[b * H + j0 + jj];
            }
        }
    }
    // no peer touches this CTA's shared memory after the last wait: every store into it precedes an arrive it waited for
    if (p.yh) {
        const float* hl = hbuf + (p.t & 1) * p.rows * H;
        for (int i = tid; i < nb * nj; i += nt) {
            const int b = i / nj, jj = i % nj;
            p.yh[((size_t)dir * p.b + b0 + b) * H + j0 + jj] = hl[b * H + j0 + jj];
        }
    }
}

// Items that fit 8 threads each (at most 32 per CTA) come from a cluster whose slice of R fits in shared memory at some cluster
// size up to 16, or from H past ~550 with at least 35 units per CTA: the streamed kernel never runs 8 threads per dot product,
// so <LBR, false, 8> is not built (gru_choose_plan never picks it).
template <bool LBR, bool RESIDENT>
const void* kernel_ks(int ks) {
    switch (ks) {
        case 1: return (const void*)gru_recur_f32_kernel<LBR, RESIDENT, 1>;
        case 2: return (const void*)gru_recur_f32_kernel<LBR, RESIDENT, 2>;
        case 4: return (const void*)gru_recur_f32_kernel<LBR, RESIDENT, 4>;
        default:
            if constexpr (!RESIDENT) return nullptr;
            else return (const void*)gru_recur_f32_kernel<LBR, RESIDENT, 8>;
    }
}
const void* kernel_of(int lbr, const RnnPlan& pl) {
    if (lbr) return pl.resident ? kernel_ks<true, true>(pl.ks) : kernel_ks<true, false>(pl.ks);
    return pl.resident ? kernel_ks<false, true>(pl.ks) : kernel_ks<false, false>(pl.ks);
}

// LBR = 0 keeps a third mbarrier (rh's) and r * h_prev of the group's rows
RecurSmem smem_of(int lbr, int h) { return RecurSmem{3, lbr ? 2 : 3, lbr ? 0 : h}; }

}  // namespace

bool gru_choose_plan(int lbr, int b, int h, int d, int sms, int smem_cap, GruFits fits, void* ctx, RnnPlan* out) {
    return recur_choose_plan(smem_of(lbr, h), b, h, d, sms, smem_cap,
                             [&](const RnnPlan& pl) { return !fits || fits(lbr, pl, ctx); }, out);
}

cudaError_t gru_max_active_clusters(int lbr, const RnnPlan& pl, int smem_cap, int* clusters) {
    return recur_max_active_clusters(kernel_of(lbr, pl), pl, smem_cap, clusters);
}

cudaError_t launch_gru_repack(const GruRepackParams& p, cudaStream_t s) {
    const int ktiles = (p.i + p.h + kTile - 1) / kTile;
    ++g_launch_count;
    gru_repack_f32_kernel<<<dim3((p.h + kTile - 1) / kTile, std::min(ktiles, 65535), 3 * p.d), kTile * 8, 0, s>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_gru_recur(int lbr, const GruParams& p, const RnnPlan& pl, cudaStream_t s) {
    cudaLaunchAttribute attr[1];
    cudaLaunchConfig_t cfg = recur_config(pl, p.d, s, attr);
    void* args[] = {const_cast<GruParams*>(&p)};
    ++g_launch_count;
    return cudaLaunchKernelExC(&cfg, kernel_of(lbr, pl), args);
}

}  // namespace mnnb200
