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
// subtraction's sign), and these are formed here in fp32 the same way.  Below them:
//   Categorical, z = Categorical._param (normalised logits), p = softmax(z):
//     d log pi(a) / dz = e_a (log_prob is a gather of z)
//     H = -sum_j c_j p_j with c_j = max(z_j, finfo(fp32).min) (torch's clamp), so
//     dH / dz_j = -p_j (m_j + c_j + H), m_j = [z_j >= finfo.min] (the clamp passes the gradient)
//   Independent(Normal(loc, scale), 1), d = a - loc:
//     d log pi / d loc = d / scale^2,  d log pi / d scale = d^2 / scale^3 - 1 / scale
//     dH / d scale = 1 / scale,        dH / d loc = 0
// Everything past the two coefficients is fp64, stored in fp32.
//
// One warp per row, lanes striding the K categories or A action dimensions, rows striding the
// grid: any N, K and A.  No shared memory, no scratch, no atomics: the output is deterministic.
#include <float.h>
#include <math.h>
#include <stdint.h>

#include "b2rl_internal.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr double kHalfLog2Pi = 0.91893853320467274178; // log(sqrt(2 pi))

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

__device__ __forceinline__ double warp_sum(double v)
{
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ double warp_max(double v)
{
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

__device__ void categorical_row(const ReinforceArgs &a, int64_t i, int lane, double c_lp,
                                double c_h)
{
    const int K = a.D;
    const size_t row = (size_t)i * K;
    const float *z = a.z + row;
    // softmax statistics of the row: lse of z (0 up to rounding, z being normalised)
    double m = -INFINITY;
    for (int k = lane; k < K; k += 32) m = fmax(m, (double)z[k]);
    m = warp_max(m);
    double s = 0.0;
    for (int k = lane; k < K; k += 32) s += exp((double)z[k] - m);
    const double lse = m + log(warp_sum(s));
    // H = -sum p_j clamp(z_j)
    double h = 0.0;
    for (int k = lane; k < K; k += 32) {
        const double p = exp((double)z[k] - lse);
        h -= p * fmax((double)z[k], (double)-FLT_MAX);
    }
    h = warp_sum(h);
    const int64_t act = a.act[i];
    const bool valid = act >= 0 && act < K;
    for (int k = lane; k < K; k += 32) {
        const double zk = (double)z[k], p = exp(zk - lse);
        const double dh = -p * ((zk >= (double)-FLT_MAX ? 1.0 : 0.0) + fmax(zk, (double)-FLT_MAX) + h);
        double g = c_h * dh;
        if (k == act) g += c_lp;
        a.g_z[row + k] = valid ? (float)g : NAN;
    }
    if (lane == 0) {
        const double lp = valid ? (double)z[act] : NAN;
        if (a.row_loss) a.row_loss[i] = (float)((-(double)a.R[i] * lp - (double)a.beta * h) * (double)a.inv_bs);
        if (a.row_ent) a.row_ent[i] = (float)h;
    }
}

__device__ void gaussian_row(const ReinforceArgs &a, int64_t i, int lane, double c_lp,
                             double c_h)
{
    const int A = a.D;
    const size_t row = (size_t)i * A;
    double lp = 0.0, h = 0.0;
    for (int k = lane; k < A; k += 32) {
        const double s = a.scale ? (double)a.scale[row + k] : 1.0;
        const double d = (double)a.act_val[row + k] - (double)a.loc[row + k];
        const double inv_s = 1.0 / s, ls = log(s);
        a.g_loc[row + k] = (float)(c_lp * d * inv_s * inv_s);
        if (a.g_scale)
            a.g_scale[row + k] = (float)(c_lp * (d * d * inv_s * inv_s * inv_s - inv_s) + c_h * inv_s);
        lp += -(d * d) * 0.5 * inv_s * inv_s - ls - kHalfLog2Pi;
        h += 0.5 + kHalfLog2Pi + ls;
    }
    if (a.row_loss || a.row_ent) {
        lp = warp_sum(lp);
        h = warp_sum(h);
        if (lane == 0) {
            if (a.row_loss) a.row_loss[i] = (float)((-(double)a.R[i] * lp - (double)a.beta * h) * (double)a.inv_bs);
            if (a.row_ent) a.row_ent[i] = (float)h;
        }
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
