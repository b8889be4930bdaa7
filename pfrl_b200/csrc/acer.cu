// acer.cu -- ACER's discrete-action loss gradient for one sequence, in one launch.
//
// Replaces (reference):
//   pfrl/agents/acer.py:16-115   compute_importance, compute_full_importance and the policy
//                                gradient with truncated importance weights and the full
//                                bias correction
//   pfrl/agents/acer.py:207-248  compute_loss_with_kl_constraint: two torch.autograd.grad
//                                calls per step and the efficient-TRPO projection
//   pfrl/agents/acer.py:423-552  compute_one_step_pi_loss / compute_loss: the Retrace and
//                                Q_opc scan, the entropy bonus, the Q loss, the scaling
// The reference runs these per step on a batch of one and reads about five device scalars
// back to Python per step.  This kernel writes d total / d z and d total / d q for all T
// steps; the agent applies them with one backward, with no host synchronisation.
//
// z is the policy's Categorical._param: torch normalises the logits it is given, so z holds
// log-probabilities, and every gradient below is taken with respect to z as the
// reference's autograd.grad takes it (log_prob(a) is a gather of z, so d/dz of it is e_a).
// With p = softmax(z), lp = log p, v = sum p q, Q = q[a], per step t (reversed):
//   rho = exp(lp[a] - lmu[a])  (1 on the online update, where mu is NULL)
//   Q_ret = r + gamma Q_ret,  Q_opc = r + gamma Q_opc,  A = (Q_opc or Q_ret) - v
//   g = -rho A e_a                                         (truncation None, or on-policy)
//   g = -min(c, rho) A e_a - cw * (q - v),  cw_j = relu(1 - c exp(lmu_j - lp_j)) p_j
//   trust region: k_j = avg_j where neither avg_j nor p_j is 0 (the terms torch's
//     Categorical KL(avg || pi) does not mask), else 0;
//     k_factor = max(0, (k.g - delta) / k.k) if k.k > 0 else 0 (NaN gives 0);
//     g -= k_factor k;  average_kl += (1 - decay) (KL_t - average_kl)
//   entropy: g_j += beta p_j (1 + lp_j + H) where p_j != 0 (d(-beta H)/dz_j)
//   g_q[a] = Q - fl32(Q_ret)
//   then Q_ret = min(1, rho) (Q_ret - Q) + v,  Q_opc += v - Q
// and finally g_z = pi_loss_coef g, g_q *= Q_loss_coef, both / T when normalising.
// The scan runs in fp64 like the reference's Python floats; everything else accumulates in
// fp64 and is stored in fp32.
//
// One CTA of 512 threads: the rows' softmax statistics, rho, v, KL and entropy one warp per
// row; the scan on one thread (it is serial in t); the gradients one warp per row again.
// Per-row values pass between the phases through an fp64 scratch of kScratch doubles per row.
#include <math.h>
#include <stdint.h>

#include "b2rl_internal.cuh"

namespace {

constexpr int kThreads = 512;
constexpr int kWarps = kThreads / 32;
// per-row scratch: lse(z), lse(mu), lse(avg), v, Q, rho, KL, H, A, Q_ret
enum { S_LSE, S_LSE_MU, S_LSE_AVG, S_V, S_Q, S_RHO, S_KL, S_H, S_ADV, S_QRET, kScratch };

struct AcerArgs {
    int T, K;
    const float *z, *q, *avg, *mu; // [T, K]; avg / mu may be null
    const int64_t *act;            // [T]
    const double *rew;             // [T]
    const float *boot;             // bootstrap value, null = terminal (R = 0)
    double gamma;
    int truncate;                  // 0: truncation_threshold None
    double c;
    int trust;
    double delta, beta, pi_coef, q_coef;
    int normalize, q_opc;
    double *avg_kl, kl_decay;
    double *s;                     // [T, kScratch]
    float *g_z, *g_q;              // [T, K]
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

// log-sum-exp of one row across the warp; -inf for a row of -inf
__device__ double warp_lse(const float *x, int K, int lane)
{
    double m = -INFINITY;
    for (int k = lane; k < K; k += 32) m = fmax(m, (double)x[k]);
    m = warp_max(m);
    if (m == -INFINITY) return m;
    double s = 0.0;
    for (int k = lane; k < K; k += 32) s += exp((double)x[k] - m);
    return m + log(warp_sum(s));
}

// torch decides p == 0 on the fp32 probabilities (trpo.cu's rule)
__device__ __forceinline__ bool prob_nonzero(double p) { return (float)p != 0.0f; }

// torch.relu: NaN stays NaN (fmax would drop it)
__device__ __forceinline__ double relu_nan(double x) { return x > 0.0 ? x : (x != x ? x : 0.0); }

// Phase 1: per-row statistics
__device__ void row_stats(const AcerArgs &a, int t, int lane)
{
    const size_t row = (size_t)t * a.K;
    const float *z = a.z + row, *q = a.q + row;
    const double lse = warp_lse(z, a.K, lane);
    double v = 0.0, h = 0.0;
    for (int k = lane; k < a.K; k += 32) {
        const double lp = (double)z[k] - lse, p = exp(lp);
        v += p * (double)q[k];
        if (prob_nonzero(p)) h -= p * lp;
    }
    v = warp_sum(v);
    h = warp_sum(h);
    const int64_t act = a.act[t];
    double lse_mu = 0.0, rho = 1.0;
    if (a.mu) {
        lse_mu = warp_lse(a.mu + row, a.K, lane);
        rho = exp(((double)z[act] - lse) - ((double)a.mu[row + act] - lse_mu));
    }
    double lse_avg = 0.0, kl = 0.0;
    if (a.trust) {
        const float *w = a.avg + row;
        lse_avg = warp_lse(w, a.K, lane);
        for (int k = lane; k < a.K; k += 32) {
            const double la = (double)w[k] - lse_avg, pa = exp(la);
            const double lp = (double)z[k] - lse;
            // _kl_categorical_categorical(avg, pi): avg == 0 -> 0, else pi == 0 -> inf
            if (prob_nonzero(pa)) kl += prob_nonzero(exp(lp)) ? pa * (la - lp) : INFINITY;
        }
        kl = warp_sum(kl);
    }
    if (lane == 0) {
        double *s = a.s + (size_t)t * kScratch;
        s[S_LSE] = lse;
        s[S_LSE_MU] = lse_mu;
        s[S_LSE_AVG] = lse_avg;
        s[S_V] = v;
        s[S_Q] = (double)q[act];
        s[S_RHO] = rho;
        s[S_KL] = kl;
        s[S_H] = h;
    }
}

// Phase 2: the Retrace / Q_opc scan, serial in t, fp64 like the reference's Python floats
__device__ void scan(const AcerArgs &a)
{
    double q_ret = a.boot ? (double)*a.boot : 0.0, q_opc = q_ret;
    double avg_kl = a.avg_kl ? *a.avg_kl : 0.0;
    for (int t = a.T - 1; t >= 0; t--) {
        double *s = a.s + (size_t)t * kScratch;
        const double r = a.rew[t], v = s[S_V], Q = s[S_Q];
        q_ret = r + a.gamma * q_ret;
        q_opc = r + a.gamma * q_opc;
        s[S_ADV] = (a.q_opc ? q_opc : q_ret) - v;
        s[S_QRET] = q_ret;
        if (a.trust) avg_kl += (1.0 - a.kl_decay) * (s[S_KL] - avg_kl);
        q_ret = fmin(1.0, s[S_RHO]) * (q_ret - Q) + v;
        q_opc = q_opc - Q + v;
    }
    if (a.trust && a.avg_kl) *a.avg_kl = avg_kl;
}

// Phase 3: the gradients of one row
__device__ void row_grads(const AcerArgs &a, int t, int lane)
{
    const size_t row = (size_t)t * a.K;
    const float *z = a.z + row, *q = a.q + row;
    const double *s = a.s + (size_t)t * kScratch;
    const double lse = s[S_LSE], v = s[S_V], rho = s[S_RHO], adv = s[S_ADV], h = s[S_H];
    const int64_t act = a.act[t];
    const bool corr = a.mu && a.truncate;
    // the policy-gradient term's weight on e_a
    const double w = corr ? fmin(a.c, rho) : rho;
    // g_j of the policy-gradient term (before the projection)
    auto g_of = [&](int k) -> double {
        double g = (k == act) ? -w * adv : 0.0;
        if (corr) {
            const double lp = (double)z[k] - lse;
            const double lmu = (double)a.mu[row + k] - s[S_LSE_MU];
            const double cw = relu_nan(1.0 - a.c * exp(lmu - lp)) * exp(lp);
            g -= cw * ((double)q[k] - v);
        }
        return g;
    };
    auto k_of = [&](int k) -> double {
        const double pa = exp((double)a.avg[row + k] - s[S_LSE_AVG]);
        return prob_nonzero(pa) && prob_nonzero(exp((double)z[k] - lse)) ? pa : 0.0;
    };
    double kf = 0.0;
    if (a.trust) {
        double kg = 0.0, kk = 0.0;
        for (int k = lane; k < a.K; k += 32) {
            const double kv = k_of(k);
            kg += kv * g_of(k);
            kk += kv * kv;
        }
        kg = warp_sum(kg);
        kk = warp_sum(kk);
        if (kk > 0.0) {
            const double f = (kg - a.delta) / kk;
            kf = f > 0.0 ? f : 0.0; // Python's max(0, f): NaN gives 0
        }
    }
    const double scale = a.normalize ? 1.0 / a.T : 1.0;
    const double cz = a.pi_coef * scale, cq = a.q_coef * scale;
    for (int k = lane; k < a.K; k += 32) {
        double g = g_of(k);
        if (kf != 0.0) g -= kf * k_of(k);
        const double lp = (double)z[k] - lse, p = exp(lp);
        if (prob_nonzero(p)) g += a.beta * p * (1.0 + lp + h);
        a.g_z[row + k] = (float)(cz * g);
        // mse_loss(torch.tensor(Q_ret), Q) / 2: the target is rounded to fp32
        a.g_q[row + k] =
            k == act ? (float)(cq * ((double)q[k] - (double)(float)s[S_QRET])) : 0.0f;
    }
}

__global__ void __launch_bounds__(kThreads, 1) k_acer_loss(AcerArgs a)
{
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int t = warp; t < a.T; t += kWarps) row_stats(a, t, lane);
    __syncthreads();
    if (threadIdx.x == 0) scan(a);
    __syncthreads();
    for (int t = warp; t < a.T; t += kWarps) row_grads(a, t, lane);
}

} // namespace

extern "C" int b2rl_acer_loss(int32_t T, int32_t K, const float *z, const float *q,
                              const float *avg_z, const float *mu_z, const int64_t *actions,
                              const double *rewards, const float *bootstrap, double gamma,
                              int32_t truncate, double truncation_threshold,
                              int32_t use_trust_region, double delta, double beta,
                              double pi_loss_coef, double q_loss_coef, int32_t normalize_by_steps,
                              int32_t use_q_opc, double *average_kl, double average_kl_decay,
                              double *scratch, float *g_z, float *g_q, void *stream)
{
    B2RL_REQUIRE(z && q && actions && rewards && scratch && g_z && g_q, B2RL_ERR_INVALID,
                 "acer_loss: null argument");
    B2RL_REQUIRE(!use_trust_region || (avg_z && average_kl), B2RL_ERR_INVALID,
                 "acer_loss: the trust region needs the average model's logits and average_kl");
    B2RL_REQUIRE(T > 0 && K > 0, B2RL_ERR_RANGE, "acer_loss: T %d, K %d", T, K);
    AcerArgs a{T, K, z, q, avg_z, mu_z, actions, rewards, bootstrap, gamma, truncate,
               truncation_threshold, use_trust_region, delta, beta, pi_loss_coef, q_loss_coef,
               normalize_by_steps, use_q_opc, average_kl, average_kl_decay, scratch, g_z, g_q};
    k_acer_loss<<<1, kThreads, 0, (cudaStream_t)stream>>>(a);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}
