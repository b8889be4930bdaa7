// trpo.cu -- TRPO's full-batch policy update as fused kernels.
//
// Replaces (reference):
//   pfrl/agents/trpo.py:415-420  _compute_gain (surrogate gain + entropy bonus)
//   pfrl/agents/trpo.py:557-598  _compute_kl_constrained_step: mean KL(old||new), its
//                                Hessian-vector product by double backward, CG, and the
//                                step scale sqrt(2 max_kl / (d^T I d + 1e-8))
//   pfrl/agents/trpo.py:600-699  _line_search: 2^-i backtracking, the first candidate with
//                                a finite gain and KL, gain improvement >= 0 and
//                                KL <= max_kl wins; otherwise theta_old is restored
//   pfrl/utils/conjugate_gradient.py
//
// Distributions: kind 0 = Independent(Normal(loc, scale), 1) (params loc, scale [N, A]),
// kind 1 = Categorical(logits) (params logits [N, K]; the kernel normalises them again,
// which is what torch's Categorical does to the logits it is given).
//
// The Fisher-vector product is the Gauss-Newton form J^T M J v: M is the Hessian of
// KL(old||new) in the distribution parameters at new == old (diag(1/s^2, 2/s^2) for the
// Gaussian, diag(p) - p p^T for the categorical).  It equals the reference's double-backward
// Hessian of mean KL at theta_old in exact arithmetic (d KL / d params vanishes there).
//
// CG computes A p once per iteration; the reference's conjugate_gradient.py evaluates
// A_product_func(p) twice per iteration (once for alpha, once for the residual), the same
// value both times.  Its dots are fp64 (the reference's are fp32 torch.matmul).  The CG
// kernel is one CTA: each iteration has two dependent reductions over the parameter vector
// (p.Ap, then r.r after the update), and the vector is the policy's parameter count
// (10^3 .. 10^5), which one CTA streams in a few microseconds; a multi-CTA version would
// need a grid-wide barrier between the two.
#include <math.h>
#include <stdint.h>

#include "b2rl_internal.cuh"

namespace {

__device__ unsigned int g_trpo_counter[B2RL_N_TICKETS];

constexpr double kLogSqrt2Pi = 0.91893853320467274178; // log(sqrt(2 pi)) as torch's math.log
constexpr double kHalfLog2PiE = 1.41893853320467274178; // 0.5 + 0.5 log(2 pi)

struct ObjArgs {
    int kind, N, A;            // A = action dims (Gaussian) or categories K
    const float *p0, *p1;      // loc, scale [N, A] or logits [N, K] (p1 unused)
    const float *o0, *o1;      // the old distribution's parameters
    const float *act_f;        // [N, A] actions (Gaussian)
    const int64_t *act_i;      // [N] actions (categorical)
    const float *log_prob_old; // [N]
    const float *adv;          // [N]
    const float *adv_stats;    // [2] mean, std or null
    double entropy_coef;
    float *g0, *g1;            // [N, A] d gain / d params, or null (forward only)
    double *partial;           // [gridDim.x, 3] scratch
    float *out;                // [3] gain, kl, mean entropy
    unsigned ticket;
};

// log-sum-exp of one row; -inf for a row of -inf (torch gives NaN normalised logits there)
__device__ double row_lse(const float *z, int K)
{
    double m = -INFINITY;
    for (int k = 0; k < K; k++) m = fmax(m, (double)z[k]);
    if (m == -INFINITY) return m;
    double s = 0.0;
    for (int k = 0; k < K; k++) s += exp((double)z[k] - m);
    return m + log(s);
}

// Whether a category's probability counts as nonzero.  torch decides p == 0 on the fp32
// probabilities of a float32 Categorical (the KL's inf and 0 terms, the entropy's clamped
// logits), so the test is on the fp32 rounding of p; the value used is still the fp64 one.
// p = e^l rounds to 0 below l = -103.97 (half the smallest subnormal).
__device__ __forceinline__ bool prob_nonzero(double p) { return (float)p != 0.0f; }

__global__ void __launch_bounds__(256) k_trpo_objective(ObjArgs a)
{
    __shared__ double sh[3][8];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    double surr = 0.0, kl = 0.0, ent = 0.0;
    if (i < a.N) {
        float advf = a.adv[i];
        // (adv - mean) / (std + 1e-8) in fp32, as the reference standardises
        if (a.adv_stats) advf = (advf - a.adv_stats[0]) / (a.adv_stats[1] + 1e-8f);
        const double adv = (double)advf;
        const size_t row = (size_t)i * a.A;
        double lp = 0.0;
        if (a.kind == 0) {
            for (int j = 0; j < a.A; j++) {
                const double mu = a.p0[row + j], sd = a.p1[row + j];
                const double d = (double)a.act_f[row + j] - mu;
                lp += -(d * d) / (2.0 * sd * sd) - log(sd) - kLogSqrt2Pi;
                ent += kHalfLog2PiE + log(sd);
                // torch's _kl_normal_normal(p = old, q = new)
                const double so = a.o1[row + j];
                const double vr = (so / sd) * (so / sd);
                const double t1 = ((a.o0[row + j] - mu) / sd) * ((a.o0[row + j] - mu) / sd);
                kl += 0.5 * (vr + t1 - 1.0 - log(vr));
            }
        } else {
            const float *z = a.p0 + row, *zo = a.o0 + row;
            const double lse = row_lse(z, a.A), lse_o = row_lse(zo, a.A);
            const int64_t act = a.act_i[i];
            lp = (double)z[act] - lse;
            for (int k = 0; k < a.A; k++) {
                const double l = (double)z[k] - lse, lo = (double)zo[k] - lse_o;
                const double p = exp(l), po = exp(lo);
                // Categorical.entropy clamps the logits at finfo.min: p = 0 adds nothing
                if (prob_nonzero(p)) ent -= p * l;
                // _kl_categorical_categorical: p_old = 0 -> 0, else q = 0 -> inf
                if (prob_nonzero(po)) kl += prob_nonzero(p) ? po * (lo - l) : INFINITY;
            }
        }
        const double ratio = exp(lp - (double)a.log_prob_old[i]);
        surr = ratio * adv;
        if (a.g0) {
            const double invN = 1.0 / a.N, ra = ratio * adv * invN, c = a.entropy_coef * invN;
            if (a.kind == 0) {
                for (int j = 0; j < a.A; j++) {
                    const double mu = a.p0[row + j], sd = a.p1[row + j];
                    const double d = (double)a.act_f[row + j] - mu, v = sd * sd;
                    a.g0[row + j] = (float)(ra * d / v);
                    a.g1[row + j] = (float)(ra * (d * d / (v * sd) - 1.0 / sd) + c / sd);
                }
            } else {
                const float *z = a.p0 + row;
                const double lse = row_lse(z, a.A);
                const int64_t act = a.act_i[i];
                double h = 0.0;
                for (int k = 0; k < a.A; k++) {
                    const double l = (double)z[k] - lse, p = exp(l);
                    if (prob_nonzero(p)) h -= p * l;
                }
                // d logp(a)/dz_k = [k == a] - p_k;  dH/dz_k = -p_k (log p_k + H)
                for (int k = 0; k < a.A; k++) {
                    const double l = (double)z[k] - lse, p = exp(l);
                    const double dh = prob_nonzero(p) ? -p * (l + h) : 0.0;
                    a.g0[row + k] = (float)(ra * ((k == act ? 1.0 : 0.0) - p) + c * dh);
                }
            }
        }
    }
    for (int o = 16; o > 0; o >>= 1) {
        surr += __shfl_xor_sync(0xffffffffu, surr, o);
        kl += __shfl_xor_sync(0xffffffffu, kl, o);
        ent += __shfl_xor_sync(0xffffffffu, ent, o);
    }
    const int warp = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) {
        sh[0][warp] = surr;
        sh[1][warp] = kl;
        sh[2][warp] = ent;
    }
    __syncthreads();
    __shared__ bool last;
    if (threadIdx.x == 0) {
        double x = 0, y = 0, z = 0;
        for (int w = 0; w < (blockDim.x >> 5); w++) {
            x += sh[0][w];
            y += sh[1][w];
            z += sh[2][w];
        }
        a.partial[blockIdx.x * 3 + 0] = x;
        a.partial[blockIdx.x * 3 + 1] = y;
        a.partial[blockIdx.x * 3 + 2] = z;
        __threadfence();
        const unsigned int prev = atomicInc(&g_trpo_counter[a.ticket], gridDim.x - 1);
        last = (prev == gridDim.x - 1);
    }
    __syncthreads();
    if (last && threadIdx.x == 0) {
        __threadfence();
        double x = 0, y = 0, z = 0;
        for (unsigned b = 0; b < gridDim.x; b++) {
            x += __ldcg(a.partial + b * 3 + 0);
            y += __ldcg(a.partial + b * 3 + 1);
            z += __ldcg(a.partial + b * 3 + 2);
        }
        const double ent_mean = z / a.N;
        a.out[0] = (float)(x / a.N + a.entropy_coef * ent_mean);
        a.out[1] = (float)(y / a.N);
        a.out[2] = (float)ent_mean;
    }
}

// M u / N per row (see the header); u0/u1 are the tangents of the distribution parameters
__global__ void __launch_bounds__(256) k_trpo_fisher(int kind, int N, int A, const float *p0,
                                                     const float *p1, const float *u0,
                                                     const float *u1, float *m0, float *m1)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const size_t row = (size_t)i * A;
    const double invN = 1.0 / N;
    if (kind == 0) {
        for (int j = 0; j < A; j++) {
            const double sd = p1[row + j], w = invN / (sd * sd);
            m0[row + j] = (float)(w * u0[row + j]);
            if (m1) m1[row + j] = (float)(2.0 * w * u1[row + j]);
        }
        return;
    }
    const double lse = row_lse(p0 + row, A);
    double pu = 0.0;
    for (int k = 0; k < A; k++) {
        const double p = exp((double)p0[row + k] - lse);
        if (p > 0.0) pu += p * u0[row + k];
    }
    for (int k = 0; k < A; k++) {
        const double p = exp((double)p0[row + k] - lse);
        m0[row + k] = p > 0.0 ? (float)(invN * p * ((double)u0[row + k] - pu)) : 0.0f;
    }
}

// fixed-order block sum of a double (blockDim.x == 1024)
__device__ double block_sum(double v, double *sh)
{
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int warp = threadIdx.x >> 5;
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sh[warp] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int w = 0; w < (blockDim.x >> 5); w++) s += sh[w];
        sh[32] = s;
    }
    __syncthreads();
    return sh[32];
}

// state[0] = r.r, state[1] = 1 once ||r|| < tol (later iterations leave x alone)
__global__ void __launch_bounds__(1024) k_trpo_cg_init(int64_t n, const float *b, float *x,
                                                       float *r, float *p, double *state)
{
    __shared__ double sh[33];
    double rr = 0.0;
    for (int64_t k = threadIdx.x; k < n; k += blockDim.x) {
        const float v = b[k];
        x[k] = 0.0f;
        r[k] = v;
        p[k] = v;
        rr += (double)v * v;
    }
    rr = block_sum(rr, sh);
    if (threadIdx.x == 0) {
        state[0] = rr;
        state[1] = 0.0;
    }
}

__global__ void __launch_bounds__(1024) k_trpo_cg_iter(int64_t n, const float *Ap, float *x,
                                                       float *r, float *p, double *state,
                                                       double tol)
{
    __shared__ double sh[33];
    if (state[1] != 0.0) return; // converged: the reference returned x here
    double pap = 0.0;
    for (int64_t k = threadIdx.x; k < n; k += blockDim.x) pap += (double)p[k] * Ap[k];
    pap = block_sum(pap, sh);
    const double rr = state[0];
    const float alpha = (float)(rr / pap);
    double rr1 = 0.0;
    for (int64_t k = threadIdx.x; k < n; k += blockDim.x) {
        x[k] = __fadd_rn(x[k], __fmul_rn(p[k], alpha));
        const float rk = __fsub_rn(r[k], __fmul_rn(Ap[k], alpha));
        r[k] = rk;
        rr1 += (double)rk * rk;
    }
    rr1 = block_sum(rr1, sh);
    if (sqrt(rr1) < tol) {
        if (threadIdx.x == 0) state[1] = 1.0;
        return;
    }
    const float beta = (float)(rr1 / rr);
    for (int64_t k = threadIdx.x; k < n; k += blockDim.x)
        p[k] = __fadd_rn(r[k], __fmul_rn(beta, p[k]));
    __syncthreads();
    if (threadIdx.x == 0) state[0] = rr1;
}

// dId = x.(F x + lambda x), rounded to fp32 as float(tensor) reads it; full = scale * x
__global__ void __launch_bounds__(1024) k_trpo_cg_step(int64_t n, const float *x,
                                                       const float *Ax, double max_kl,
                                                       float *full, float *dId_out)
{
    __shared__ double sh[33];
    double d = 0.0;
    for (int64_t k = threadIdx.x; k < n; k += blockDim.x) d += (double)x[k] * Ax[k];
    d = block_sum(d, sh);
    const float dId = (float)d;
    const float scale = (float)sqrt(2.0 * max_kl / ((double)dId + 1e-8));
    for (int64_t k = threadIdx.x; k < n; k += blockDim.x) full[k] = __fmul_rn(scale, x[k]);
    if (threadIdx.x == 0 && dId_out) *dId_out = dId;
}

// cand [n_cand][3] = gain, kl, entropy of theta_old + 2^-i full; gain0 [3] at theta_old.
// record[0] = winner's KL, [1] = its step size (0: none), [2] = 1 if one won.
// theta = theta_old + s * full (fp32 mul then add, as flat_params + step_size * full_step),
// or theta_old itself when nothing won.
__global__ void __launch_bounds__(256) k_trpo_line_search(int n_cand, const float *cand,
                                                          const float *gain0, double max_kl,
                                                          int64_t n, const float *theta_old,
                                                          const float *full, float *theta,
                                                          float *record)
{
    __shared__ int win;
    if (threadIdx.x == 0) {
        win = -1;
        for (int c = 0; c < n_cand && win < 0; c++) {
            const float g = cand[c * 3 + 0], kl = cand[c * 3 + 1];
            const double improve = (double)g - (double)gain0[0];
            if (isfinite(g) && isfinite(kl) && !(improve < 0.0) && !((double)kl > max_kl))
                win = c;
        }
        if (blockIdx.x == 0) {
            record[0] = win >= 0 ? cand[win * 3 + 1] : 0.0f;
            record[1] = win >= 0 ? ldexpf(1.0f, -win) : 0.0f;
            record[2] = win >= 0 ? 1.0f : 0.0f;
        }
    }
    __syncthreads();
    const float s = win >= 0 ? ldexpf(1.0f, -win) : 0.0f;
    for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < n;
         k += (int64_t)gridDim.x * blockDim.x)
        theta[k] = win >= 0 ? __fadd_rn(theta_old[k], __fmul_rn(s, full[k])) : theta_old[k];
}

int grid_for(int64_t n, int threads, int cap)
{
    const int64_t g = (n + threads - 1) / threads;
    return (int)(g < cap ? g : cap);
}

} // namespace

extern "C" int b2rl_trpo_objective(int32_t kind, int32_t N, int32_t A, const float *p0,
                                   const float *p1, const float *old0, const float *old1,
                                   const void *actions, const float *log_prob_old,
                                   const float *adv, const float *adv_stats, double entropy_coef,
                                   float *g0, float *g1, double *scratch, float *out,
                                   void *stream)
{
    B2RL_REQUIRE(kind == 0 || kind == 1, B2RL_ERR_INVALID, "trpo_objective: kind %d", kind);
    B2RL_REQUIRE(p0 && old0 && actions && log_prob_old && adv && scratch && out,
                 B2RL_ERR_INVALID, "trpo_objective: null argument");
    B2RL_REQUIRE(kind == 1 || (p1 && old1), B2RL_ERR_INVALID,
                 "trpo_objective: the Gaussian needs scale and old scale");
    B2RL_REQUIRE(!g0 || kind == 1 || g1, B2RL_ERR_INVALID,
                 "trpo_objective: the Gaussian gradient needs both outputs");
    B2RL_REQUIRE(N > 0 && A > 0, B2RL_ERR_RANGE, "trpo_objective: empty batch");
    ObjArgs a{kind, N, A, p0, p1, old0, old1,
              kind == 0 ? (const float *)actions : nullptr,
              kind == 1 ? (const int64_t *)actions : nullptr,
              log_prob_old, adv, adv_stats, entropy_coef, g0, g1, scratch, out};
    a.ticket = b2rl_next_ticket();
    k_trpo_objective<<<(N + 255) / 256, 256, 0, (cudaStream_t)stream>>>(a);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}

extern "C" int b2rl_trpo_fisher(int32_t kind, int32_t N, int32_t A, const float *p0,
                                const float *p1, const float *u0, const float *u1, float *m0,
                                float *m1, void *stream)
{
    B2RL_REQUIRE(kind == 0 || kind == 1, B2RL_ERR_INVALID, "trpo_fisher: kind %d", kind);
    B2RL_REQUIRE(p0 && u0 && m0 && (kind == 1 || p1), B2RL_ERR_INVALID,
                 "trpo_fisher: null argument");
    B2RL_REQUIRE(!m1 || u1, B2RL_ERR_INVALID, "trpo_fisher: m1 needs u1");
    B2RL_REQUIRE(N > 0 && A > 0, B2RL_ERR_RANGE, "trpo_fisher: empty batch");
    k_trpo_fisher<<<(N + 255) / 256, 256, 0, (cudaStream_t)stream>>>(kind, N, A, p0, p1, u0, u1,
                                                                    m0, m1);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}

extern "C" int b2rl_trpo_cg_init(int64_t n, const float *b, float *x, float *r, float *p,
                                 double *state, void *stream)
{
    B2RL_REQUIRE(b && x && r && p && state, B2RL_ERR_INVALID, "trpo_cg_init: null argument");
    B2RL_REQUIRE(n > 0, B2RL_ERR_RANGE, "trpo_cg_init: empty vector");
    k_trpo_cg_init<<<1, 1024, 0, (cudaStream_t)stream>>>(n, b, x, r, p, state);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}

extern "C" int b2rl_trpo_cg_iter(int64_t n, const float *Ap, float *x, float *r, float *p,
                                 double *state, double tol, void *stream)
{
    B2RL_REQUIRE(Ap && x && r && p && state, B2RL_ERR_INVALID, "trpo_cg_iter: null argument");
    B2RL_REQUIRE(n > 0, B2RL_ERR_RANGE, "trpo_cg_iter: empty vector");
    k_trpo_cg_iter<<<1, 1024, 0, (cudaStream_t)stream>>>(n, Ap, x, r, p, state, tol);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}

extern "C" int b2rl_trpo_cg_step(int64_t n, const float *x, const float *Ax, double max_kl,
                                 float *full_step, float *dId, void *stream)
{
    B2RL_REQUIRE(x && Ax && full_step, B2RL_ERR_INVALID, "trpo_cg_step: null argument");
    B2RL_REQUIRE(n > 0, B2RL_ERR_RANGE, "trpo_cg_step: empty vector");
    k_trpo_cg_step<<<1, 1024, 0, (cudaStream_t)stream>>>(n, x, Ax, max_kl, full_step, dId);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}

extern "C" int b2rl_trpo_line_search(int32_t n_cand, const float *cand, const float *gain0,
                                     double max_kl, int64_t n, const float *theta_old,
                                     const float *full_step, float *theta, float *record,
                                     void *stream)
{
    B2RL_REQUIRE(cand && gain0 && theta_old && full_step && theta && record, B2RL_ERR_INVALID,
                 "trpo_line_search: null argument");
    B2RL_REQUIRE(n_cand > 0 && n_cand <= 64 && n > 0, B2RL_ERR_RANGE,
                 "trpo_line_search: %d candidates over %lld parameters", n_cand, (long long)n);
    k_trpo_line_search<<<grid_for(n, 256, 1024), 256, 0, (cudaStream_t)stream>>>(
        n_cand, cand, gain0, max_kl, n, theta_old, full_step, theta, record);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}
