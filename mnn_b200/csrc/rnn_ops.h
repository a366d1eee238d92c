// rnn_ops.h -- the launch plan and host-callable launcher of libmnn_b200_rnn.so's recurrence kernel (rnn.cu), enqueue-only on
// the given stream.
#pragma once
#include <cuda_runtime.h>

namespace mnnb200 {

constexpr int kRnnThreads = 256;      // most threads of one CTA
constexpr int kRnnMaxCluster = 16;    // non-portable cluster size
constexpr int kRnnMaxHidden = 4096;   // H past this is refused (the double-buffered h of one batch row must fit)
constexpr int kRnnMaxRows = 8;        // most batch rows of one group
constexpr int kRnnPartials = 8;       // every gate's dot product is 8 partial sums over k mod 8 (rnn.cu, gate_dots)

// One cluster per (direction, batch group).  The cluster's `cs` CTAs each own `hs` consecutive hidden units (the last CTA may
// own fewer, or none) and all gate rows of R for them; each (batch row, unit) pair of a CTA is one item, worked by `ks`
// consecutive threads.
struct RnnPlan {
    int cs = 0, groups = 0, rows = 0, hs = 0, ks = 0, threads = 0, resident = 0, smem = 0, rstride = 0;
};

struct RnnParams {
    const float* g;    // [T * B][D * G * H] = X W^T + bias (G = 4 gates for LSTM, 1 for RNN), rows in X's time order
    const float* r;    // [D][G * H][H]
    const float* h0;   // [D][B][H] or null (zeros, and no h_prev R^T term at the first step)
    const float* c0;   // [D][B][H] or null (zeros, and no f * c term at the first step)
    float* y;          // [T][D][B][H]
    float* yh;         // [D][B][H] or null
    float* yc;         // [D][B][H] or null (LSTM)
    int t, b, h, d;
    int cs, rows, hs, rstride;   // rstride: the row pitch of the resident R slice in floats
};

// The plan for (cell: 0 LSTM / 1 RNN, B, H, D) on a device of `sms` SMs with at most `smem_cap` bytes of dynamic shared
// memory per CTA.  Depends on nothing else, T in particular.  `fits(plan)` says whether a cluster of the plan can be resident
// on the device (cudaOccupancyMaxActiveClusters): a plan that cannot halves its cluster.  False when nothing fits.
typedef bool (*RnnFits)(int cell, const RnnPlan& plan, void* ctx);
bool rnn_choose_plan(int cell, int b, int h, int d, int sms, int smem_cap, RnnFits fits, void* ctx, RnnPlan* out);

// cudaOccupancyMaxActiveClusters of the plan's kernel and launch; sets the kernel's attributes (dynamic shared memory up to
// smem_cap, non-portable cluster sizes) that the launch needs, so it precedes the plan's first launch
cudaError_t rnn_max_active_clusters(int cell, const RnnPlan& plan, int smem_cap, int* clusters);

// the recurrence of all T steps, both directions: one launch
cudaError_t launch_rnn_recur(int cell, const RnnParams& p, const RnnPlan& plan, cudaStream_t s);

}  // namespace mnnb200
