// losses.cu -- fused TD-error / loss kernels of the DQN family.
//
// Replaces chains of small ATen launches + host round trips in the reference:
//   pfrl/agents/dqn.py:44-104,388-470          Huber / MSE value loss, |y-t|
//   pfrl/agents/al.py, pal.py, double_pal.py,  advantage-learning and DPP targets
//     dpp.py (_compute_y_and_t)                (row max / argmax / softmax / logsumexp)
//   pfrl/agents/categorical_dqn.py:7-57        _apply_categorical_projection
//   pfrl/agents/categorical_dqn.py:60-97,178-204  cross entropy, per-sample
//                                              priority error, weighted sum
//   pfrl/agents/iqn.py:176-208                 quantile Huber loss
//
// All arithmetic is fp32 in the reference's operation order (no FMA
// contraction where the reference rounds between ops), so losses agree to
// ~1e-7 relative; the batch reductions are deterministic (fixed-order tree in
// the last CTA to finish).
#include <math.h>

#include "b2rl_internal.cuh"
#include "td_common.cuh"

namespace {

// ---------------------------------------------------------------------------
// C51: one warp per sample.
// ---------------------------------------------------------------------------
constexpr int C51_MAX_ATOMS = 256;
constexpr int C51_WARPS = 8;

struct C51Args {
    const float *y;       // [B, n] predicted probabilities of the taken action
    const float *next_p;  // [B, n] target-net probabilities of the greedy next action
    const float *reward, *discount, *terminal; // [B]
    const float *weights; // [B] or null
    const float *z;       // [n] atom values
    int B, n, mean;
    float *t_out;     // [B, n] projected target (saved for backward)
    float *delta_out; // [B] per-sample loss = priority error
    float *term;      // [B] scratch: w_i * delta_i
    float *loss_out;  // [1]
    unsigned ticket;  // completion counter of this launch
};

__global__ void __launch_bounds__(C51_WARPS * 32) k_c51_fwd(C51Args a)
{
    __shared__ float zt[C51_WARPS][C51_MAX_ATOMS];
    __shared__ float sh[32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int i = blockIdx.x * C51_WARPS + warp;
    const int n = a.n;
    if (i < a.B) {
        float *row = zt[warp];
        for (int j = lane; j < n; j += 32) row[j] = 0.f;
        __syncwarp();
        const float v_min = a.z[0], v_max = a.z[n - 1];
        const float delta_z = __fsub_rn(a.z[1], a.z[0]);
        const float r = a.reward[i];
        // (1 - terminal) * discount, then * z, then + r: categorical_dqn.py:147-152
        const float scale = __fmul_rn(__fsub_rn(1.0f, a.terminal[i]), a.discount[i]);
        for (int j = lane; j < n; j += 32) {
            float tz = __fadd_rn(r, __fmul_rn(scale, a.z[j]));
            tz = fminf(fmaxf(tz, v_min), v_max);
            float bj = __fdiv_rn(__fsub_rn(tz, v_min), delta_z);
            bj = fminf(fmaxf(bj, 0.f), (float)(n - 1));
            const float lo = floorf(bj), up = ceilf(bj);
            const float frac = __fsub_rn(bj, lo);
            const float p = a.next_p[(size_t)i * n + j];
            atomicAdd(&row[(int)lo], __fmul_rn(p, __fsub_rn(1.0f, frac)));
            atomicAdd(&row[(int)up], __fmul_rn(p, frac));
        }
        __syncwarp();
        float acc = 0.f;
        for (int j = lane; j < n; j += 32) {
            const float t = row[j];
            a.t_out[(size_t)i * n + j] = t;
            const float yc = fminf(fmaxf(a.y[(size_t)i * n + j], 1e-10f), 1.0f);
            acc += __fmul_rn(-t, logf(yc)); // -t * log(clamp(y, 1e-10, 1)), :183
        }
        acc = warp_sum(acc);
        if (lane == 0) {
            a.delta_out[i] = acc;
            a.term[i] = a.weights ? __fmul_rn(acc, a.weights[i]) : acc;
        }
    }
    finish_sum(a.term, a.B, a.mean ? (float)a.B : 1.0f, a.loss_out, sh, a.ticket);
}

struct C51BwdArgs {
    const float *y, *t, *weights, *grad_loss;
    int B, n, mean;
    float *grad_y;
};

__global__ void k_c51_bwd(C51BwdArgs a)
{
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= a.B * a.n) return;
    const int i = idx / a.n;
    float g = a.grad_loss[0];
    if (a.mean) g = g / (float)a.B;
    if (a.weights) g *= a.weights[i];
    const float y = a.y[idx];
    // d/dy [-t log(clamp(y))] = -t / y inside the clamp range, 0 outside
    a.grad_y[idx] = (y >= 1e-10f && y <= 1.0f) ? g * (-a.t[idx] / y) : 0.f;
}

// ---------------------------------------------------------------------------
// Scalar TD loss (DQN / DoubleDQN): y = Q(s)[a], t = r + disc (1-term) next_q
// ---------------------------------------------------------------------------
struct TdArgs {
    const float *q;        // [B, nA]
    const long long *action; // [B]
    const float *next_q;   // [B] max / double-Q value of the next state
    const float *reward, *discount, *terminal, *weights;
    int B, nA, clip_delta, mean;
    float *y_out, *t_out, *delta_out, *term, *loss_out;
    unsigned ticket;
};

__global__ void __launch_bounds__(256) k_td_fwd(TdArgs a)
{
    __shared__ float sh[32];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < a.B) {
        const float y = a.q[(size_t)i * a.nA + a.action[i]];
        const float t = bellman_target(a.reward[i], a.discount[i], a.terminal[i], a.next_q[i]);
        td_outputs(y, t, i, a.clip_delta, a.weights, a.y_out, a.t_out, a.delta_out, a.term);
    }
    finish_sum(a.term, a.B, a.mean ? (float)a.B : 1.0f, a.loss_out, sh, a.ticket);
}

// ---------------------------------------------------------------------------
// Advantage-learning and DPP targets (AL, PAL, DoublePAL, DPP, DPPL, DPPGreedy):
// y = Q(s)[a] as for DQN, t from row reductions over the target net's action
// values at s and s'.  One warp per sample, lanes strided over the actions.
// ---------------------------------------------------------------------------
constexpr int ADV_WARPS = 8;

struct AdvTdArgs {
    const float *q;          // [B, nA] online net at s
    const long long *action; // [B]
    const float *tq, *tnq;   // [B, nA] target net at s and s'
    const float *nq;         // [B, nA] online net at s' (DOUBLE_PAL) or null
    const float *reward, *discount, *terminal, *weights;
    float alpha;             // fp32(alpha), as torch rounds a Python float factor
    float eta, inv_eta;      // fp32(eta) and fp32(1 / fp32(eta)): torch's x / eta on CUDA
    int mode, B, nA, clip_delta, mean;
    float *y_out, *t_out, *delta_out, *term, *loss_out;
    unsigned ticket;
};

// v at j beats the best so far (bv at bj): torch's max / argmax order, NaN
// greatest, the first index among equals.
__device__ __forceinline__ bool beats(float v, int j, float bv, int bj)
{
    if (isnan(v)) return !isnan(bv) || j < bj;
    if (isnan(bv)) return false;
    return v > bv || (v == bv && j < bj);
}

// max over row[0..n) and its first index, on every lane of the warp (n >= 1)
__device__ __forceinline__ float warp_row_max(const float *row, int n, int lane, int *idx)
{
    float bv = 0.f;
    int bj = -1; // this lane has seen no element yet
    for (int j = lane; j < n; j += 32) {
        const float v = row[j];
        if (bj < 0 || beats(v, j, bv, bj)) bv = v, bj = j;
    }
    for (int o = 16; o > 0; o >>= 1) {
        const float v = __shfl_xor_sync(0xffffffffu, bv, o);
        const int j = __shfl_xor_sync(0xffffffffu, bj, o);
        if (j >= 0 && (bj < 0 || beats(v, j, bv, bj))) bv = v, bj = j;
    }
    *idx = bj;
    return bv;
}

// DPP's L operators over one row of action values x with maximum xmax, on every lane.
// Softmax and logsumexp take z = fp32(eta) * x first, as `eta * q_values` does, and
// subtract max z before exp (torch's softmax and logsumexp do the same).
__device__ __forceinline__ float warp_l_operator(int mode, const float *row, int n, int lane,
                                                 float xmax, float eta, float inv_eta)
{
    if (mode == B2RL_ADV_DPP_GREEDY) return xmax;
    // eta > 0, so max z = fp32(eta * max x)
    float zmax = __fmul_rn(eta, xmax);
    if (mode == B2RL_ADV_DPPL && isinf(zmax)) zmax = 0.f; // logsumexp's masked_fill
    float s = 0.f, sx = 0.f;
    for (int j = lane; j < n; j += 32) {
        const float x = row[j];
        const float e = expf(__fsub_rn(__fmul_rn(eta, x), zmax));
        s = __fadd_rn(s, e);
        sx = __fadd_rn(sx, __fmul_rn(e, x));
    }
    s = warp_sum(s);
    if (mode == B2RL_ADV_DPPL) // logsumexp(eta * x) / eta, dpp.py:105
        return __fmul_rn(__fadd_rn(logf(s), zmax), inv_eta);
    // sum(softmax(eta * x) * x), action_value.py:78-79: normalise once after the sum
    sx = warp_sum(sx);
    return __fdiv_rn(sx, s);
}

__global__ void __launch_bounds__(ADV_WARPS * 32) k_adv_td_fwd(AdvTdArgs a)
{
    __shared__ float sh[32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int i = blockIdx.x * ADV_WARPS + warp;
    if (i < a.B) {
        const int n = a.nA;
        const size_t off = (size_t)i * n;
        const int act = (int)a.action[i];
        const float *tq = a.tq + off, *tnq = a.tnq + off;
        int jmax;
        const float tq_max = warp_row_max(tq, n, lane, &jmax);
        const float tnq_max = warp_row_max(tnq, n, lane, &jmax);
        const float tq_a = tq[act], tnq_a = tnq[act];
        const float r = a.reward[i], disc = a.discount[i], term = a.terminal[i];
        float t;
        if (a.mode == B2RL_ADV_AL || a.mode == B2RL_ADV_PAL || a.mode == B2RL_ADV_DOUBLE_PAL) {
            float next_v = tnq_max;
            if (a.mode == B2RL_ADV_DOUBLE_PAL) { // Q'(s', argmax_a Q(s', a)), double_pal.py:48-51
                int jg;
                warp_row_max(a.nq + off, n, lane, &jg);
                next_v = tnq[jg];
            }
            const float tb = bellman_target(r, disc, term, next_v);
            float adv = __fsub_rn(tq_a, tq_max); // target_qout.compute_advantage, al.py:69
            if (a.mode != B2RL_ADV_AL) {         // torch.max(cur, next), pal.py:73-77
                const float adv_next = __fsub_rn(tnq_a, tnq_max);
                adv = (isnan(adv) || adv > adv_next) ? adv : adv_next;
            }
            t = __fadd_rn(tb, __fmul_rn(a.alpha, adv));
        } else { // Q'(s,a) + (r + disc (1 - term) L Q'(s')) - L Q'(s), dpp.py:34-76
            const float l_next = warp_l_operator(a.mode, tnq, n, lane, tnq_max, a.eta, a.inv_eta);
            const float l_cur = warp_l_operator(a.mode, tq, n, lane, tq_max, a.eta, a.inv_eta);
            t = __fsub_rn(__fadd_rn(tq_a, bellman_target(r, disc, term, l_next)), l_cur);
        }
        if (lane == 0)
            td_outputs(a.q[off + act], t, i, a.clip_delta, a.weights, a.y_out, a.t_out,
                       a.delta_out, a.term);
    }
    finish_sum(a.term, a.B, a.mean ? (float)a.B : 1.0f, a.loss_out, sh, a.ticket);
}

struct TdBwdArgs {
    const float *y, *t, *weights, *grad_loss;
    const long long *action;
    int B, nA, clip_delta, mean;
    float *grad_q; // [B, nA]
};

__global__ void k_td_bwd(TdBwdArgs a)
{
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= a.B * a.nA) return;
    const int i = idx / a.nA, j = idx - i * a.nA;
    float gq = 0.f;
    if (j == (int)a.action[i])
        gq = td_grad(a.y, a.t, a.weights, a.grad_loss, i, a.B, a.clip_delta, a.mean);
    a.grad_q[idx] = gq;
}

// ---------------------------------------------------------------------------
// Quantile Huber loss (IQN): y [B, N], t [B, N'], taus [B, N]
// ---------------------------------------------------------------------------
struct QhArgs {
    const float *y, *t, *taus, *weights;
    int B, N, Np, mean;
    float *delta_out, *term, *loss_out;
    unsigned ticket;
};

// one CTA per sample, N x N' pairs strided over the threads
__global__ void __launch_bounds__(256) k_qh_fwd(QhArgs a)
{
    __shared__ float sh[32];
    __shared__ float s_tot;
    const int i = blockIdx.x;
    float acc = 0.f;
    const int pairs = a.N * a.Np;
    for (int p = threadIdx.x; p < pairs; p += blockDim.x) {
        const int n = p / a.Np, m = p - n * a.Np;
        const float y = a.y[(size_t)i * a.N + n];
        const float t = a.t[(size_t)i * a.Np + m];
        const float tau = a.taus[(size_t)i * a.N + n];
        const float d = __fsub_rn(t, y);
        const float ad = fabsf(d);
        // smooth_l1 (beta = 1): iqn.py:198-203
        const float hub = ad < 1.0f ? __fmul_rn(__fmul_rn(0.5f, d), d) : __fsub_rn(ad, 0.5f);
        const float I = d < 0.f ? 1.0f : 0.0f; // bellman error < 0
        acc += __fmul_rn(fabsf(__fsub_rn(tau, I)), hub);
    }
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x < 32) {
        float s = threadIdx.x < (blockDim.x >> 5) ? sh[threadIdx.x] : 0.f;
        s = warp_sum(s);
        if (threadIdx.x == 0) s_tot = s;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        // loss per sample: mean over N' then sum over N (iqn.py:210-250)
        const float li = s_tot / (float)a.Np;
        a.delta_out[i] = s_tot / (float)(a.N * a.Np); // eltwise_loss.mean((1, 2)), iqn.py:388
        a.term[i] = a.weights ? __fmul_rn(li, a.weights[i]) : li;
    }
    finish_sum(a.term, a.B, a.mean ? (float)a.B : 1.0f, a.loss_out, sh, a.ticket);
}

struct QhBwdArgs {
    const float *y, *t, *taus, *weights, *grad_loss;
    int B, N, Np, mean;
    float *grad_y; // [B, N]
};

__global__ void k_qh_bwd(QhBwdArgs a)
{
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= a.B * a.N) return;
    const int i = idx / a.N;
    float g = a.grad_loss[0] / (float)a.Np;
    if (a.mean) g = g / (float)a.B;
    if (a.weights) g *= a.weights[i];
    const float y = a.y[idx], tau = a.taus[idx];
    float acc = 0.f;
    for (int m = 0; m < a.Np; m++) {
        const float d = a.t[(size_t)i * a.Np + m] - y;
        const float I = d < 0.f ? 1.0f : 0.0f;
        // d hub / dy = -clamp(d, -1, 1)
        acc += fabsf(tau - I) * -fminf(fmaxf(d, -1.0f), 1.0f);
    }
    a.grad_y[idx] = g * acc;
}

} // namespace

extern "C" int b2rl_c51_loss_fwd(const float *y, const float *next_p, const float *reward,
                                 const float *discount, const float *terminal,
                                 const float *weights, const float *z, int32_t B, int32_t n_atoms,
                                 int mean, float *t_out, float *delta_out, float *scratch,
                                 float *loss_out, void *stream)
{
    B2RL_REQUIRE(y && next_p && reward && discount && terminal && z && t_out && delta_out &&
                     scratch && loss_out, B2RL_ERR_INVALID, "c51_loss_fwd: null argument");
    B2RL_REQUIRE(B > 0 && n_atoms >= 2 && n_atoms <= C51_MAX_ATOMS, B2RL_ERR_RANGE,
                 "c51_loss_fwd: need B > 0 and 2 <= n_atoms <= %d", C51_MAX_ATOMS);
    C51Args a{y, next_p, reward, discount, terminal, weights, z, B, n_atoms, mean,
              t_out, delta_out, scratch, loss_out};
    a.ticket = b2rl_next_ticket();
    k_c51_fwd<<<(B + C51_WARPS - 1) / C51_WARPS, C51_WARPS * 32, 0, (cudaStream_t)stream>>>(a);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}

extern "C" int b2rl_c51_loss_bwd(const float *y, const float *t, const float *weights,
                                 const float *grad_loss, int32_t B, int32_t n_atoms, int mean,
                                 float *grad_y, void *stream)
{
    B2RL_REQUIRE(y && t && grad_loss && grad_y, B2RL_ERR_INVALID, "c51_loss_bwd: null argument");
    C51BwdArgs a{y, t, weights, grad_loss, B, n_atoms, mean, grad_y};
    const int total = B * n_atoms;
    k_c51_bwd<<<(total + 255) / 256, 256, 0, (cudaStream_t)stream>>>(a);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}

extern "C" int b2rl_td_loss_fwd(const float *q, const int64_t *action, const float *next_q,
                                const float *reward, const float *discount,
                                const float *terminal, const float *weights, int32_t B,
                                int32_t n_actions, int clip_delta, int mean, float *y_out,
                                float *t_out, float *delta_out, float *scratch, float *loss_out,
                                void *stream)
{
    B2RL_REQUIRE(q && action && next_q && reward && discount && terminal && y_out && t_out &&
                     delta_out && scratch && loss_out, B2RL_ERR_INVALID,
                 "td_loss_fwd: null argument");
    B2RL_REQUIRE(B > 0 && n_actions > 0, B2RL_ERR_RANGE, "td_loss_fwd: empty batch");
    TdArgs a{q, (const long long *)action, next_q, reward, discount, terminal, weights, B,
             n_actions, clip_delta, mean, y_out, t_out, delta_out, scratch, loss_out};
    a.ticket = b2rl_next_ticket();
    k_td_fwd<<<(B + 255) / 256, 256, 0, (cudaStream_t)stream>>>(a);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}

extern "C" int b2rl_adv_td_loss_fwd(int mode, const float *q, const int64_t *action,
                                    const float *tq, const float *tnq, const float *nq,
                                    const float *reward, const float *discount,
                                    const float *terminal, const float *weights, int32_t B,
                                    int32_t n_actions, double alpha, double eta, int clip_delta,
                                    int mean, float *y_out, float *t_out, float *delta_out,
                                    float *scratch, float *loss_out, void *stream)
{
    B2RL_REQUIRE(q && action && tq && tnq && reward && discount && terminal && y_out && t_out &&
                     delta_out && scratch && loss_out, B2RL_ERR_INVALID,
                 "adv_td_loss_fwd: null argument");
    B2RL_REQUIRE(mode >= B2RL_ADV_AL && mode <= B2RL_ADV_DPP_GREEDY, B2RL_ERR_INVALID,
                 "adv_td_loss_fwd: unknown mode %d", mode);
    B2RL_REQUIRE(mode != B2RL_ADV_DOUBLE_PAL || nq, B2RL_ERR_INVALID,
                 "adv_td_loss_fwd: DOUBLE_PAL needs the online net's next-state values");
    B2RL_REQUIRE(B > 0 && n_actions > 0, B2RL_ERR_RANGE, "adv_td_loss_fwd: empty batch");
    const bool softmax_mode = mode == B2RL_ADV_DPP || mode == B2RL_ADV_DPPL;
    B2RL_REQUIRE(!softmax_mode || (float)eta > 0.f, B2RL_ERR_RANGE,
                 "adv_td_loss_fwd: need eta > 0, got %g", eta);
    AdvTdArgs a{q, (const long long *)action, tq, tnq, nq, reward, discount, terminal, weights};
    a.alpha = (float)alpha;
    a.eta = (float)eta;
    a.inv_eta = softmax_mode ? 1.0f / a.eta : 0.f;
    a.mode = mode;
    a.B = B;
    a.nA = n_actions;
    a.clip_delta = clip_delta;
    a.mean = mean;
    a.y_out = y_out;
    a.t_out = t_out;
    a.delta_out = delta_out;
    a.term = scratch;
    a.loss_out = loss_out;
    a.ticket = b2rl_next_ticket();
    k_adv_td_fwd<<<(B + ADV_WARPS - 1) / ADV_WARPS, ADV_WARPS * 32, 0, (cudaStream_t)stream>>>(a);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}

extern "C" int b2rl_td_loss_bwd(const float *y, const float *t, const float *weights,
                                const int64_t *action, const float *grad_loss, int32_t B,
                                int32_t n_actions, int clip_delta, int mean, float *grad_q,
                                void *stream)
{
    B2RL_REQUIRE(y && t && action && grad_loss && grad_q, B2RL_ERR_INVALID,
                 "td_loss_bwd: null argument");
    TdBwdArgs a{y, t, weights, grad_loss, (const long long *)action, B, n_actions, clip_delta,
                mean, grad_q};
    const int total = B * n_actions;
    k_td_bwd<<<(total + 255) / 256, 256, 0, (cudaStream_t)stream>>>(a);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}

extern "C" int b2rl_quantile_huber_fwd(const float *y, const float *t, const float *taus,
                                       const float *weights, int32_t B, int32_t N, int32_t Np,
                                       int mean, float *delta_out, float *scratch,
                                       float *loss_out, void *stream)
{
    B2RL_REQUIRE(y && t && taus && delta_out && scratch && loss_out, B2RL_ERR_INVALID,
                 "quantile_huber_fwd: null argument");
    B2RL_REQUIRE(B > 0 && N > 0 && Np > 0, B2RL_ERR_RANGE, "quantile_huber_fwd: empty");
    QhArgs a{y, t, taus, weights, B, N, Np, mean, delta_out, scratch, loss_out};
    a.ticket = b2rl_next_ticket();
    k_qh_fwd<<<B, 256, 0, (cudaStream_t)stream>>>(a);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}

extern "C" int b2rl_quantile_huber_bwd(const float *y, const float *t, const float *taus,
                                       const float *weights, const float *grad_loss, int32_t B,
                                       int32_t N, int32_t Np, int mean, float *grad_y,
                                       void *stream)
{
    B2RL_REQUIRE(y && t && taus && grad_loss && grad_y, B2RL_ERR_INVALID,
                 "quantile_huber_bwd: null argument");
    QhBwdArgs a{y, t, taus, weights, grad_loss, B, N, Np, mean, grad_y};
    const int total = B * N;
    k_qh_bwd<<<(total + 255) / 256, 256, 0, (cudaStream_t)stream>>>(a);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}
