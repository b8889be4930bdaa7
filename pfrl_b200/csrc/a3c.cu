// a3c.cu -- A3C's loss gradient over the N recorded steps of one segment, in one launch.
//
// Replaces (reference):
//   pfrl/agents/a3c.py:177-204  the returns scan, the advantage, pi_loss = sum(-adv log pi(a)
//                               - beta H), v_loss = mse_loss(v, R, sum) / 2, both scaled by
//                               their factors, and the backward of their sum
// The kernel writes d loss / d(distribution parameters) and d loss / d v for every row; the
// agent applies them with one backward.
//
// Returns: the reference scans in Python floats, R = V(s_T) (0 for a terminal segment), then
// R = R * gamma + r_j from the last step back, and rounds each R to fp32 in torch.as_tensor.
// Each warp redoes that scan serially in fp64 with __dmul_rn / __dadd_rn (no FMA contraction)
// from the last step down to its own row, so every row's R is bit for bit the reference's
// whichever warp computes it; a parallel scan would round differently.  N is t_max or less
// for the agent, so the redone work is a few steps.
//
// The backward of the reference's loss hands log pi(a), H and v of row i the fp32 gradients
//   c_lp = fl32(pf * -adv),   c_H = -fl32(pf * fl32(beta)),
//   g_v  = fl32(fl32(2 * fl32(v - R)) * fl32(vf / 2)),
// with adv = fl32(R - v) (detached), pf = fl32(pi_factor) and vf = fl32(v_factor): the
// factor's MulBackward, the sum's expansion, the product and the subtraction for pi_loss;
// the factor, DivBackward and MseLossBackward (2 * (input - target) * grad) for v_loss.
// They are formed here in fp32 the same way.  Below c_lp and c_H, the row's d log pi(a) and
// dH (pg_common.cuh, shared with reinforce.cu) are fp64, stored in fp32.
//
// One warp per row, lanes striding the K categories or A action dimensions, rows striding the
// grid: any N, K and A.  No shared memory, no scratch, no atomics: the output is deterministic.
//
// ptxas -v, sm_90a: k_a3c_loss<true> (Categorical) 64 registers, k_a3c_loss<false> (Gaussian)
// 40 registers; no stack frame, no spills.
#include <stdint.h>

#include "b2rl_internal.cuh"
#include "pg_common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

struct A3CArgs {
    int64_t N;
    int D;                      // K (categorical) or A (Gaussian)
    const float *z;             // [N, K], or null for a Gaussian
    const float *loc, *scale;   // [N, A]; scale null = 1
    const int64_t *act;         // [N] (categorical)
    const float *act_val;       // [N, A] (Gaussian)
    const float *v;             // [N]
    const double *rewards;      // [N]
    const float *bootstrap;     // [1], null = terminal (R = 0)
    double gamma;
    float beta, pf, vf;         // fl32(beta), fl32(pi_factor), fl32(v_factor)
    float *g_z, *g_loc, *g_scale;  // g_scale null = not wanted
    float *g_v;                 // [N]
    float *returns;             // [N], optional
    float *row_pi, *row_v;      // [N] each, optional: each row's pi_loss and v_loss term
};

template <bool kCategorical>
__global__ void __launch_bounds__(kThreads) k_a3c_loss(A3CArgs a)
{
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * kWarps;
    const int64_t first = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (first >= a.N) return;
    // this warp's rows from the last one down, so that the scan carries over between them
    int64_t i = first + (a.N - 1 - first) / warps * warps;
    double R = a.bootstrap ? (double)*a.bootstrap : 0.0;
    int64_t j = a.N;  // rewards [j, N) are in R
    for (; i >= 0; i -= warps) {
        for (; j > i; --j) R = __dadd_rn(__dmul_rn(R, a.gamma), a.rewards[j - 1]);
        const float R32 = __double2float_rn(R);
        const float v = a.v[i];
        const float adv = __fsub_rn(R32, v);
        const double c_lp = (double)__fmul_rn(a.pf, -adv);
        const double c_h = -(double)__fmul_rn(a.pf, a.beta);
        const bool want = a.row_pi != nullptr;
        const RowTerms t = kCategorical ? categorical_row_grad(a, i, lane, c_lp, c_h)
                                        : gaussian_row_grad(a, i, lane, c_lp, c_h, want);
        if (lane == 0) {
            const float d = __fsub_rn(v, R32);
            a.g_v[i] = __fmul_rn(__fmul_rn(2.0f, d), __fdiv_rn(a.vf, 2.0f));
            if (a.returns) a.returns[i] = R32;
            if (want) {
                a.row_pi[i] = (float)((-(double)adv * t.lp - (double)a.beta * t.h) * (double)a.pf);
                a.row_v[i] = (float)((double)d * (double)d * 0.5 * (double)a.vf);
            }
        }
    }
}

} // namespace

extern "C" int b2rl_a3c_loss(int64_t N, int32_t D, const float *z, const float *loc,
                             const float *scale, const int64_t *actions,
                             const float *action_values, const float *v,
                             const double *rewards, const float *bootstrap, double gamma,
                             double beta, double pi_factor, double v_factor, float *g_z,
                             float *g_loc, float *g_scale, float *g_v, float *returns,
                             float *row_pi_loss, float *row_v_loss, void *stream)
{
    B2RL_REQUIRE(v && rewards && g_v, B2RL_ERR_INVALID, "a3c_loss: null v, rewards or g_v");
    B2RL_REQUIRE(z ? (actions && g_z && !loc) : (loc && action_values && g_loc),
                 B2RL_ERR_INVALID,
                 "a3c_loss: give z, actions and g_z (Categorical) or loc, action_values "
                 "and g_loc (Gaussian)");
    B2RL_REQUIRE(!row_pi_loss == !row_v_loss, B2RL_ERR_INVALID,
                 "a3c_loss: give both row_pi_loss and row_v_loss, or neither");
    B2RL_REQUIRE(N > 0 && D > 0, B2RL_ERR_RANGE, "a3c_loss: N %lld, D %d", (long long)N, D);
    A3CArgs a{N, D, z, loc, scale, actions, action_values, v, rewards, bootstrap, gamma,
              (float)beta, (float)pi_factor, (float)v_factor, g_z, g_loc, g_scale, g_v,
              returns, row_pi_loss, row_v_loss};
    const int64_t want = (N + kWarps - 1) / kWarps;
    const int blocks = (int)(want < 132 * 16 ? want : 132 * 16);
    if (z) k_a3c_loss<true><<<blocks, kThreads, 0, (cudaStream_t)stream>>>(a);
    else k_a3c_loss<false><<<blocks, kThreads, 0, (cudaStream_t)stream>>>(a);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}
