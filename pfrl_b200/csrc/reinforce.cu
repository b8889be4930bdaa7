// reinforce.cu -- REINFORCE's loss gradient over every recorded step of an update, in one launch.
//
// Replaces (reference):
//   pfrl/agents/reinforce.py:176-195  accumulate_grad: -R * log_prob - beta * entropy per step,
//                                     torch.stack(losses).sum() / batchsize, and the backward of
//                                     that through one batch-1 graph per step
// The rows are the steps of all episodes of the update, concatenated (or packed); R is each
// step's return, computed on the host by the reference's own expression.  The kernel writes
// d loss / d(distribution parameters) for all rows; the agent applies them with one backward.
//
// The backward of the reference's loss hands log pi(a) and H of one row the fp32 gradients
//   c_lp = fl32(fl32(1 / batchsize) * fl32(-R)),   c_H = -fl32(fl32(1 / batchsize) * fl32(beta))
// (DivBackward, then MulBackward with the Python / numpy scalar rounded to fp32, then the
// subtraction's sign), and these are formed here in fp32 the same way.  Below them, the
// row's d log pi(a) and dH (pg_common.cuh, shared with a3c.cu) are fp64, stored in fp32.
//
// One warp per row, lanes striding the K categories or A action dimensions, rows striding the
// grid: any N, K and A.  No shared memory, no scratch, no atomics: the output is deterministic.
#include <stdint.h>

#include "b2rl_internal.cuh"
#include "pg_common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

struct ReinforceArgs {
    int64_t N;
    int D;                      // K (categorical) or A (Gaussian)
    const float *z;             // [N, K], or null for a Gaussian
    const float *loc, *scale;   // [N, A]; scale null = 1
    const int64_t *act;         // [N] (categorical)
    const float *act_val;       // [N, A] (Gaussian)
    const float *R;             // [N]
    float inv_bs;               // fl32(1 / batchsize)
    float beta;                 // fl32(beta)
    float *g_z, *g_loc, *g_scale;  // g_scale null = not wanted
    float *row_loss, *row_ent;  // [N] each, optional
};

__device__ void categorical_row(const ReinforceArgs &a, int64_t i, int lane, double c_lp,
                                double c_h)
{
    const RowTerms t = categorical_row_grad(a, i, lane, c_lp, c_h);
    if (lane == 0) {
        if (a.row_loss) a.row_loss[i] = (float)((-(double)a.R[i] * t.lp - (double)a.beta * t.h) * (double)a.inv_bs);
        if (a.row_ent) a.row_ent[i] = (float)t.h;
    }
}

__device__ void gaussian_row(const ReinforceArgs &a, int64_t i, int lane, double c_lp,
                             double c_h)
{
    const bool want = a.row_loss || a.row_ent;
    const RowTerms t = gaussian_row_grad(a, i, lane, c_lp, c_h, want);
    if (want && lane == 0) {
        if (a.row_loss) a.row_loss[i] = (float)((-(double)a.R[i] * t.lp - (double)a.beta * t.h) * (double)a.inv_bs);
        if (a.row_ent) a.row_ent[i] = (float)t.h;
    }
}

__global__ void __launch_bounds__(kThreads) k_reinforce_loss(ReinforceArgs a)
{
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * kWarps;
    for (int64_t i = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5); i < a.N; i += warps) {
        // the reference's backward, in fp32: (1 / bs) * (-R) and -((1 / bs) * beta)
        const double c_lp = (double)__fmul_rn(a.inv_bs, -a.R[i]);
        const double c_h = -(double)__fmul_rn(a.inv_bs, a.beta);
        if (a.z) categorical_row(a, i, lane, c_lp, c_h);
        else gaussian_row(a, i, lane, c_lp, c_h);
    }
}

} // namespace

extern "C" int b2rl_reinforce_loss(int64_t N, int32_t D, const float *z, const float *loc,
                                   const float *scale, const int64_t *actions,
                                   const float *action_values, const float *returns,
                                   int32_t batchsize, double beta, float *g_z, float *g_loc,
                                   float *g_scale, float *row_loss, float *row_entropy,
                                   void *stream)
{
    B2RL_REQUIRE(returns, B2RL_ERR_INVALID, "reinforce_loss: null returns");
    B2RL_REQUIRE(z ? (actions && g_z && !loc) : (loc && action_values && g_loc),
                 B2RL_ERR_INVALID,
                 "reinforce_loss: give z, actions and g_z (Categorical) or loc, action_values "
                 "and g_loc (Gaussian)");
    B2RL_REQUIRE(N > 0 && D > 0 && batchsize > 0, B2RL_ERR_RANGE,
                 "reinforce_loss: N %lld, D %d, batchsize %d", (long long)N, D, batchsize);
    ReinforceArgs a{N, D, z, loc, scale, actions, action_values, returns,
                    1.0f / (float)batchsize, (float)beta, g_z, g_loc, g_scale,
                    row_loss, row_entropy};
    const int64_t want = (N + kWarps - 1) / kWarps;
    const int blocks = (int)(want < 132 * 16 ? want : 132 * 16);
    k_reinforce_loss<<<blocks, kThreads, 0, (cudaStream_t)stream>>>(a);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}
