// gru_ops.h -- the launch plan and host-callable launchers of libmnn_b200_gru.so's kernels (gru.cu), enqueue-only on the given
// stream.  The plan is the recurrences' (rnn_ops.h RnnPlan, recur_common.cuh).
#pragma once
#include <cuda_runtime.h>

#include "rnn_ops.h"

namespace mnnb200 {

// the op's weights of one direction, in its input order: Wg [I + H][2H], bg [2H], Wc [I + H][H], bc [H], rb [3H]
constexpr int kGruParamsPerDir = 5;

struct GruRepackParams {
    const float* in[2 * kGruParamsPerDir];   // direction d's five tensors at 5 d .. 5 d + 4
    float* wx;                               // [I][D * 3H]: the x parts of Wg (z, r) and Wc (n), per direction
    float* r;                                // [D][3H][H]: the h parts, transposed, rows z, r, n
    float* bx;                               // [D * 3H]: bg on the z / r columns, 0 on the n columns
    float* kb;                               // [D][4H]: rb (Rb_z, Rb_r, Rb_h), then bc
    int i, h, d;
};

struct GruParams {
    const float* g;    // [T * B][D * 3H] = X Wx + bx, rows in X's time order
    const float* r;    // [D][3H][H]
    const float* kb;   // [D][4H]
    const float* h0;   // [D][B][H] or null (zeros, and no h_prev term at the first step)
    float* y;          // [T][D][B][H] or null
    float* yh;         // [D][B][H] or null
    int t, b, h, d;
    int cs, rows, hs, rstride;
};

// The plan for (linear_before_reset, B, H, D) on a device of `sms` SMs with at most `smem_cap` bytes of dynamic shared memory
// per CTA; depends on nothing else, T in particular.  `fits(lbr, plan, ctx)`: whether a cluster of the plan can be resident.
typedef bool (*GruFits)(int lbr, const RnnPlan& plan, void* ctx);
bool gru_choose_plan(int lbr, int b, int h, int d, int sms, int smem_cap, GruFits fits, void* ctx, RnnPlan* out);

// cudaOccupancyMaxActiveClusters of the plan's kernel and launch (and the kernel attributes that launch needs)
cudaError_t gru_max_active_clusters(int lbr, const RnnPlan& plan, int smem_cap, int* clusters);

// the weight repack of every execute: one launch
cudaError_t launch_gru_repack(const GruRepackParams& p, cudaStream_t s);
// the recurrence of all T steps, both directions: one launch
cudaError_t launch_gru_recur(int lbr, const GruParams& p, const RnnPlan& plan, cudaStream_t s);

}  // namespace mnnb200
