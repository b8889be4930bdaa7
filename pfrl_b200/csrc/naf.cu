// naf.cu -- normalized advantage functions (NAF, arXiv:1603.00748) for the DQN family.
//
// Replaces (reference):
//   pfrl/q_functions/state_q_functions.py:194-219  FCQuadraticStateQFunction.forward after the
//     linear layers: torch.exp of the diagonal, lower_triangular_matrix (zeros + two index_puts
//     with host index arrays), and the bmm L L^T (or mat_diag**2 when n = 1)
//   pfrl/action_value.py QuadraticActionValue  max / evaluate_actions / compute_advantage in the
//     _compute_y_and_t of pfrl/agents/dqn.py, double_dqn.py, al.py, pal.py, double_pal.py and
//     dpp.py (DPPGreedy), with the value loss of dqn.py:44-104
//
// Head.  L[i][i] = exp(diag_pre[i]), L[i][k] = non_diag[i (i - 1) / 2 + k] for k < i (the order
// of np.tril_indices(n, -1)), 0 above the diagonal; mat = L L^T.  One thread per entry of the
// lower triangle of one sample, summing k = 0 .. i in order, and writing mat[i][j] and mat[j][i].
// The terms with min(i, j) < k <= i are a zero times L[i][k]; they are kept so that an infinite
// diagonal gives NaN where the reference's bmm puts it (0 * inf).  The backward is
// grad_L = G L + G^T L on the lower triangle (G not assumed symmetric), then the exp's
// gradient on the diagonal.
//
// Loss.  Q(u) = v - 1/2 (u - mu)^T P (u - mu), max = v without bounds, else Q(clamp(mu)) (the
// reference's greedy action, even when mu lies outside the box).  One warp per sample, lanes
// over the columns of P.  y = Q(s, a) of the online net, t by mode (include/b2rl.h); then the
// same y / t / |y - t| / loss outputs and gradient as b2rl_td_loss_fwd / _bwd.  The quadratic
// forms are summed in a different order than torch's bmm (DESIGN section 7a).
#include <math.h>
#include <stdint.h>

#include "b2rl_internal.cuh"
#include "td_common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

// L[i][k] of one sample
__device__ __forceinline__ float tril_at(const float *diag_pre, const float *non_diag, int i,
                                         int k)
{
    if (k == i) return expf(diag_pre[i]);
    if (k < i) return non_diag[i * (i - 1) / 2 + k];
    return 0.f;
}

// p-th entry (row-major) of the lower triangle, diagonal included: row i >= column j
__device__ __forceinline__ void tri_decode(int64_t p, int *i, int *j)
{
    int r = (int)((sqrt(8.0 * (double)p + 1.0) - 1.0) * 0.5);
    while ((int64_t)r * (r + 1) / 2 > p) --r;
    while ((int64_t)(r + 1) * (r + 2) / 2 <= p) ++r;
    *i = r;
    *j = (int)(p - (int64_t)r * (r + 1) / 2);
}

__global__ void __launch_bounds__(kThreads) k_naf_head_fwd(const float *diag_pre,
                                                           const float *non_diag, int B, int n,
                                                           float *mat)
{
    const int64_t tri = (int64_t)n * (n + 1) / 2, m = (int64_t)n * (n - 1) / 2;
    const int64_t total = (int64_t)B * tri;
    for (int64_t x = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; x < total;
         x += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = x / tri;
        int i, j;
        tri_decode(x - b * tri, &i, &j);
        const float *dp = diag_pre + b * n, *nd = non_diag + b * m;
        float s = 0.f;
        for (int k = 0; k <= i; ++k)
            s = fmaf(tril_at(dp, nd, i, k), tril_at(dp, nd, j, k), s);
        float *out = mat + b * n * n;
        out[(int64_t)i * n + j] = s;
        out[(int64_t)j * n + i] = s;
    }
}

// grad_L[i][k] = sum_j G[i][j] L[j][k] + sum_j G[j][i] L[j][k] for k <= i (L[j][k] = 0 for j < k)
__global__ void __launch_bounds__(kThreads) k_naf_head_bwd(const float *diag_pre,
                                                           const float *non_diag,
                                                           const float *grad_mat, int B, int n,
                                                           float *grad_diag_pre,
                                                           float *grad_non_diag)
{
    const int64_t tri = (int64_t)n * (n + 1) / 2, m = (int64_t)n * (n - 1) / 2;
    const int64_t total = (int64_t)B * tri;
    for (int64_t x = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; x < total;
         x += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = x / tri;
        int i, k;
        tri_decode(x - b * tri, &i, &k);
        const float *dp = diag_pre + b * n, *nd = non_diag + b * m;
        const float *G = grad_mat + b * n * n;
        float gl = 0.f, gtl = 0.f;
        for (int j = k; j < n; ++j) {
            const float l = tril_at(dp, nd, j, k);
            gl = fmaf(G[(int64_t)i * n + j], l, gl);
            gtl = fmaf(G[(int64_t)j * n + i], l, gtl);
        }
        const float g = __fadd_rn(gl, gtl);
        if (k == i)
            grad_diag_pre[b * n + i] = __fmul_rn(g, expf(dp[i])); // exp's backward: g * result
        else
            grad_non_diag[b * m + i * (i - 1) / 2 + k] = g;
    }
}

// torch.max / torch.min of two values: NaN if either is NaN
__device__ __forceinline__ float nan_max(float a, float b)
{
    return isnan(a) ? a : (isnan(b) ? b : fmaxf(a, b));
}
__device__ __forceinline__ float nan_min(float a, float b)
{
    return isnan(a) ? a : (isnan(b) ? b : fminf(a, b));
}

// d_i = x_i - m_i with x = src clamped to [lo, hi] where the bound is given
// (QuadraticActionValue.greedy_actions: max with the lower bound first, then min with the upper)
__device__ __forceinline__ float diff_at(const float *src, const float *m, const float *lo,
                                         const float *hi, int i)
{
    float x = src[i];
    if (lo) x = nan_max(lo[i], x);
    if (hi) x = nan_min(hi[i], x);
    return __fsub_rn(x, m[i]);
}

// -1/2 d^T P d + v on every lane (evaluate_actions: (d^T P) d, times -0.5, plus v)
__device__ __forceinline__ float warp_q(const float *P, const float *src, const float *m,
                                        const float *lo, const float *hi, float v, int n,
                                        int lane)
{
    float s = 0.f;
    for (int j = lane; j < n; j += 32) {
        float r = 0.f;
        for (int i = 0; i < n; ++i) r = fmaf(diff_at(src, m, lo, hi, i), P[(int64_t)i * n + j], r);
        s = fmaf(r, diff_at(src, m, lo, hi, j), s);
    }
    s = warp_sum(s);
    return __fadd_rn(__fmul_rn(-0.5f, s), v);
}

struct NafTdArgs {
    const float *mu, *mat, *v;       // online net at s: [B, n], [B, n, n], [B]
    const float *action;             // [B, n]
    const float *tmu, *tmat, *tv;    // target net at s, or null (DQN, DOUBLE_DQN)
    const float *tnmu, *tnmat, *tnv; // target net at s'
    const float *nmu;                // online net's mu at s' (DOUBLE_DQN, DOUBLE_PAL), or null
    const float *lo, *hi;            // [n] target net's bounds, each may be null
    const float *nlo, *nhi;          // [n] online net's bounds (its greedy action at s')
    const float *reward, *discount, *terminal, *weights;
    float alpha;
    int mode, B, n, clip_delta, mean;
    float *y_out, *t_out, *delta_out, *term, *loss_out;
    unsigned ticket;
};

// QuadraticActionValue.max of sample i: v, or Q at the clamped mu when a bound is given
__device__ __forceinline__ float warp_max(const float *mu, const float *P, float v,
                                          const float *lo, const float *hi, int n, int lane)
{
    if (!lo && !hi) return v;
    return warp_q(P, mu, mu, lo, hi, v, n, lane);
}

__global__ void __launch_bounds__(kThreads) k_naf_td_fwd(NafTdArgs a)
{
    __shared__ float sh[32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int i = blockIdx.x * kWarps + warp;
    if (i < a.B) {
        const int n = a.n;
        const int64_t vo = (int64_t)i * n, mo = vo * n;
        const float *act = a.action + vo;
        const float y = warp_q(a.mat + mo, act, a.mu + vo, nullptr, nullptr, a.v[i], n, lane);
        const float *tnmu = a.tnmu + vo, *tnmat = a.tnmat + mo;
        const float tnv = a.tnv[i];
        float next_v;
        if (a.mode == B2RL_NAF_DOUBLE_DQN || a.mode == B2RL_ADV_DOUBLE_PAL)
            next_v = warp_q(tnmat, a.nmu + vo, tnmu, a.nlo, a.nhi, tnv, n, lane);
        else
            next_v = warp_max(tnmu, tnmat, tnv, a.lo, a.hi, n, lane);
        const float tb = bellman_target(a.reward[i], a.discount[i], a.terminal[i], next_v);
        float t = tb;
        if (a.mode != B2RL_NAF_DQN && a.mode != B2RL_NAF_DOUBLE_DQN) {
            const float *tmu = a.tmu + vo, *tmat = a.tmat + mo;
            const float tv = a.tv[i];
            const float tq_a = warp_q(tmat, act, tmu, nullptr, nullptr, tv, n, lane);
            const float tq_max = warp_max(tmu, tmat, tv, a.lo, a.hi, n, lane);
            if (a.mode == B2RL_ADV_DPP_GREEDY) { // Q'(s, a) + T(max'(s')) - max'(s), dpp.py
                t = __fsub_rn(__fadd_rn(tq_a, tb), tq_max);
            } else {
                float adv = __fsub_rn(tq_a, tq_max); // target_qout.compute_advantage, al.py
                if (a.mode != B2RL_ADV_AL) {         // torch.max(cur, next), pal.py
                    const float tnq_a = warp_q(tnmat, act, tnmu, nullptr, nullptr, tnv, n, lane);
                    const float adv_next =
                        __fsub_rn(tnq_a, warp_max(tnmu, tnmat, tnv, a.lo, a.hi, n, lane));
                    adv = (isnan(adv) || adv > adv_next) ? adv : adv_next;
                }
                t = __fadd_rn(tb, __fmul_rn(a.alpha, adv));
            }
        }
        if (lane == 0)
            td_outputs(y, t, i, a.clip_delta, a.weights, a.y_out, a.t_out, a.delta_out, a.term);
    }
    finish_sum(a.term, a.B, a.mean ? (float)a.B : 1.0f, a.loss_out, sh, a.ticket);
}

struct NafTdBwdArgs {
    const float *mu, *mat, *action, *y, *t, *weights, *grad_loss;
    int B, n, clip_delta, mean;
    float *grad_mu, *grad_mat, *grad_v;
};

// y = v + (-0.5 * s), s = r d, r = d^T P, d = a - mu; with gs = -0.5 g (g = d loss / d y):
//   grad_v = g, grad_P[i][j] = d_i (gs d_j), grad_mu_i = -(sum_j P[i][j] (gs d_j) + gs r_i)
__global__ void __launch_bounds__(kThreads) k_naf_td_bwd(NafTdBwdArgs a)
{
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.x * kWarps + warp;
    if (b >= a.B) return;
    const int n = a.n;
    const int64_t vo = (int64_t)b * n, mo = vo * n;
    const float *mu = a.mu + vo, *act = a.action + vo, *P = a.mat + mo;
    const float g = td_grad(a.y, a.t, a.weights, a.grad_loss, b, a.B, a.clip_delta, a.mean);
    const float gs = __fmul_rn(-0.5f, g);
    if (lane == 0) a.grad_v[b] = g;
    for (int i = lane; i < n; i += 32) {
        float pgd = 0.f, r = 0.f;
        for (int j = 0; j < n; ++j) {
            const float dj = __fsub_rn(act[j], mu[j]);
            pgd = fmaf(P[(int64_t)i * n + j], __fmul_rn(gs, dj), pgd);
            r = fmaf(dj, P[(int64_t)j * n + i], r);
        }
        a.grad_mu[vo + i] = -__fadd_rn(pgd, __fmul_rn(gs, r));
    }
    for (int i = 0; i < n; ++i) {
        const float di = __fsub_rn(act[i], mu[i]);
        for (int j = lane; j < n; j += 32)
            a.grad_mat[mo + (int64_t)i * n + j] = __fmul_rn(di, __fmul_rn(gs, __fsub_rn(act[j], mu[j])));
    }
}

int grid_for(int64_t threads)
{
    const int64_t blocks = (threads + kThreads - 1) / kThreads;
    return (int)(blocks < 65535 * 16 ? blocks : 65535 * 16);
}

} // namespace

extern "C" int b2rl_naf_head_fwd(const float *diag_pre, const float *non_diag, int32_t B,
                                 int32_t n, float *mat, void *stream)
{
    B2RL_REQUIRE(diag_pre && mat && (n == 1 || non_diag), B2RL_ERR_INVALID,
                 "naf_head_fwd: null argument");
    B2RL_REQUIRE(B > 0 && n > 0, B2RL_ERR_RANGE, "naf_head_fwd: need B > 0 and n > 0");
    k_naf_head_fwd<<<grid_for((int64_t)B * n * (n + 1) / 2), kThreads, 0,
                     (cudaStream_t)stream>>>(diag_pre, non_diag, B, n, mat);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}

extern "C" int b2rl_naf_head_bwd(const float *diag_pre, const float *non_diag,
                                 const float *grad_mat, int32_t B, int32_t n,
                                 float *grad_diag_pre, float *grad_non_diag, void *stream)
{
    B2RL_REQUIRE(diag_pre && grad_mat && grad_diag_pre && (n == 1 || (non_diag && grad_non_diag)),
                 B2RL_ERR_INVALID, "naf_head_bwd: null argument");
    B2RL_REQUIRE(B > 0 && n > 0, B2RL_ERR_RANGE, "naf_head_bwd: need B > 0 and n > 0");
    k_naf_head_bwd<<<grid_for((int64_t)B * n * (n + 1) / 2), kThreads, 0,
                     (cudaStream_t)stream>>>(diag_pre, non_diag, grad_mat, B, n, grad_diag_pre,
                                             grad_non_diag);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}

extern "C" int b2rl_naf_td_loss_fwd(
    int mode, const float *mu, const float *mat, const float *v, const float *action,
    const float *tmu, const float *tmat, const float *tv, const float *tnmu, const float *tnmat,
    const float *tnv, const float *nmu, const float *lo, const float *hi, const float *nlo,
    const float *nhi, const float *reward, const float *discount, const float *terminal,
    const float *weights, int32_t B, int32_t n, double alpha, int clip_delta, int mean,
    float *y_out, float *t_out, float *delta_out, float *scratch, float *loss_out, void *stream)
{
    B2RL_REQUIRE(mode == B2RL_ADV_AL || mode == B2RL_ADV_PAL || mode == B2RL_ADV_DOUBLE_PAL ||
                     mode == B2RL_ADV_DPP_GREEDY || mode == B2RL_NAF_DQN ||
                     mode == B2RL_NAF_DOUBLE_DQN,
                 B2RL_ERR_INVALID, "naf_td_loss_fwd: unknown mode %d", mode);
    B2RL_REQUIRE(mu && mat && v && action && tnmu && tnmat && tnv && reward && discount &&
                     terminal && y_out && t_out && delta_out && scratch && loss_out,
                 B2RL_ERR_INVALID, "naf_td_loss_fwd: null argument");
    const bool needs_t = mode != B2RL_NAF_DQN && mode != B2RL_NAF_DOUBLE_DQN;
    B2RL_REQUIRE(!needs_t || (tmu && tmat && tv), B2RL_ERR_INVALID,
                 "naf_td_loss_fwd: mode %d needs the target net at s", mode);
    B2RL_REQUIRE((mode != B2RL_NAF_DOUBLE_DQN && mode != B2RL_ADV_DOUBLE_PAL) || nmu,
                 B2RL_ERR_INVALID, "naf_td_loss_fwd: mode %d needs the online net's mu at s'",
                 mode);
    B2RL_REQUIRE(B > 0 && n > 0, B2RL_ERR_RANGE, "naf_td_loss_fwd: need B > 0 and n > 0");
    NafTdArgs a{mu, mat, v, action, tmu, tmat, tv, tnmu, tnmat, tnv, nmu, lo, hi, nlo, nhi,
                reward, discount, terminal, weights};
    a.alpha = (float)alpha;
    a.mode = mode;
    a.B = B;
    a.n = n;
    a.clip_delta = clip_delta;
    a.mean = mean;
    a.y_out = y_out;
    a.t_out = t_out;
    a.delta_out = delta_out;
    a.term = scratch;
    a.loss_out = loss_out;
    a.ticket = b2rl_next_ticket();
    k_naf_td_fwd<<<(B + kWarps - 1) / kWarps, kThreads, 0, (cudaStream_t)stream>>>(a);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}

extern "C" int b2rl_naf_td_loss_bwd(const float *mu, const float *mat, const float *action,
                                    const float *y, const float *t, const float *weights,
                                    const float *grad_loss, int32_t B, int32_t n, int clip_delta,
                                    int mean, float *grad_mu, float *grad_mat, float *grad_v,
                                    void *stream)
{
    B2RL_REQUIRE(mu && mat && action && y && t && grad_loss && grad_mu && grad_mat && grad_v,
                 B2RL_ERR_INVALID, "naf_td_loss_bwd: null argument");
    B2RL_REQUIRE(B > 0 && n > 0, B2RL_ERR_RANGE, "naf_td_loss_bwd: need B > 0 and n > 0");
    NafTdBwdArgs a{mu, mat, action, y, t, weights, grad_loss, B, n, clip_delta, mean,
                   grad_mu, grad_mat, grad_v};
    k_naf_td_bwd<<<(B + kWarps - 1) / kWarps, kThreads, 0, (cudaStream_t)stream>>>(a);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}
