// sac.cu -- K9: the launch-bound elementwise tail of the SAC / TD3 / DDPG update.
//
// Replaces (reference, one tiny ATen launch per tensor and per operator):
//   pfrl/utils/copy_param.py:9-22              soft_copy_param (Polyak averaging,
//                                              2 launches per state_dict entry)
//   pfrl/agents/soft_actor_critic.py:225-240   entropy-regularised TD target
//                                              (min, mul, sub, flatten, mul, mul, add)
//   pfrl/agents/td3.py:20-24                   target-policy smoothing (randn_like aside:
//                                              mul, clamp, add, clamp)
//   pfrl/agents/td3.py:181-236,                clipped double-Q / 1-step target, both
//   pfrl/agents/ddpg.py:150-173                critics' mse_loss and its backward
// All are rounded exactly like the reference's sequence of separate fp32
// operations (no FMA contraction), so parameters stay bit-identical to an
// eager run.  The losses are the one exception: they are sums, reduced in a
// fixed order of their own (deterministic, not torch's order).
#include "b2rl_internal.cuh"
#include "td_common.cuh"

namespace {

constexpr int POLYAK_MAX = 96;      // tensor pairs per launch (kernel parameter space)
constexpr int POLYAK_CHUNK = 2048;  // elements per CTA

struct PolyakArgs {
    float *dst[POLYAK_MAX];
    const float *src[POLYAK_MAX];
    int first_block[POLYAK_MAX + 1]; // prefix sum of ceil(numel / CHUNK)
    long long numel[POLYAK_MAX];
    int n;
    float keep, tau; // float(1 - tau), float(tau): what mul_(1 - tau) / tau * source use
};

__global__ void __launch_bounds__(256) k_polyak(const __grid_constant__ PolyakArgs a)
{
    // which tensor does this CTA work on? (n <= 96: a short scan of the prefix table)
    int t = 0;
    while (t + 1 < a.n && (int)blockIdx.x >= a.first_block[t + 1]) t++;
    const long long base = (long long)(blockIdx.x - a.first_block[t]) * POLYAK_CHUNK;
    float *d = a.dst[t];
    const float *s = a.src[t];
    const long long n = a.numel[t];
#pragma unroll
    for (int j = 0; j < POLYAK_CHUNK / 256; j++) {
        const long long i = base + j * 256 + threadIdx.x;
        if (i < n) {
            // target.mul_(1 - tau); target.add_(tau * source): three roundings
            d[i] = __fadd_rn(__fmul_rn(d[i], a.keep), __fmul_rn(a.tau, s[i]));
        }
    }
}

__global__ void __launch_bounds__(256) k_sac_target(const float *reward, const float *discount,
                                                    const float *terminal, const float *q1,
                                                    const float *q2, const float *log_prob,
                                                    const float *temperature_dev,
                                                    float temperature, int n, float *out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float alpha = temperature_dev ? *temperature_dev : temperature;
    const float a = q1[i], b = q2[i];
    // torch.min(q1', q2'): NaN if either head is NaN (fminf alone would drop it)
    const float next_q = (isnan(a) || isnan(b)) ? __int_as_float(0x7fffffff) : fminf(a, b);
    const float entropy_term = __fmul_rn(alpha, log_prob[i]);        // temperature * log_prob
    const float soft = __fsub_rn(next_q, entropy_term);              // next_q - entropy_term
    const float w = __fmul_rn(discount[i], __fsub_rn(1.0f, terminal[i])); // discount * (1 - term)
    out[i] = __fadd_rn(reward[i], __fmul_rn(w, soft));               // reward + w * soft
}

// torch.min(a, b) elementwise (at::minimum): the first NaN operand, else fminf
__device__ __forceinline__ float torch_min(float a, float b)
{
    return isnan(a) ? a : (isnan(b) ? b : fminf(a, b));
}

// torch.clamp(v, lo, hi): a NaN passes through
__device__ __forceinline__ float torch_clamp(float v, float lo, float hi)
{
    return isnan(v) ? v : fminf(fmaxf(v, lo), hi);
}

// default_target_policy_smoothing_func: clamp(a + clamp(0.2 * eps, -0.5, 0.5), -1, 1)
__global__ void __launch_bounds__(256) k_td3_smooth(const float *action, const float *noise,
                                                    long long n, float *out)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float eps = torch_clamp(__fmul_rn(0.2f, noise[i]), -0.5f, 0.5f);
    out[i] = torch_clamp(__fadd_rn(action[i], eps), -1.0f, 1.0f);
}

constexpr int CRITIC_THREADS = 256;
constexpr int CRITIC_ROWS = 4 * CRITIC_THREADS; // rows per CTA (B2RL_CRITIC_LOSS_ROWS_PER_CTA)
static_assert(CRITIC_ROWS == B2RL_CRITIC_LOSS_ROWS_PER_CTA, "b2rl.h documents the CTA size");

struct CriticLossArgs {
    const float *reward, *discount, *terminal, *next_q1, *next_q2, *pred_q1, *pred_q2;
    float gamma;    // the discount of every row when discount is NULL (DDPG)
    float norm;     // float(2.0 / n): mse_loss_backward's factor for reduction="mean"
    int n;
    float *target, *grad1, *grad2, *loss1, *loss2;
    float *partial; // [2][gridDim.x] CTA sums when gridDim.x > 1
    unsigned ticket;
};

// Sums v1 / v2 over the CTA in a fixed order; the result is valid in thread 0.
__device__ __forceinline__ void cta_sum2(float &v1, float &v2)
{
    __shared__ float sh[2][CRITIC_THREADS / 32];
    v1 = warp_sum(v1);
    v2 = warp_sum(v2);
    if ((threadIdx.x & 31) == 0) {
        sh[0][threadIdx.x >> 5] = v1;
        sh[1][threadIdx.x >> 5] = v2;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        v1 = sh[0][0];
        v2 = sh[1][0];
        for (int w = 1; w < CRITIC_THREADS / 32; w++) {
            v1 = __fadd_rn(v1, sh[0][w]);
            v2 = __fadd_rn(v2, sh[1][w]);
        }
    }
}

// One launch of the critic update's elementwise tail and loss: the target of td3.py /
// ddpg.py, then, per critic, mse_loss(target, pred) (mean) and its gradient with respect
// to pred, float(2/n) * (pred - target) -- what torch's mse_loss backward forms before it
// multiplies by the upstream gradient.  Each CTA sums its rows' squared errors in a fixed
// order; with more than one CTA, the last to arrive sums the CTA sums in a fixed order.
__global__ void __launch_bounds__(CRITIC_THREADS) k_td3_critic_loss(const CriticLossArgs a)
{
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int k = 0; k < CRITIC_ROWS / CRITIC_THREADS; k++) {
        const int i = blockIdx.x * CRITIC_ROWS + k * CRITIC_THREADS + threadIdx.x;
        if (i >= a.n) break;
        const float next_q = a.next_q2 ? torch_min(a.next_q1[i], a.next_q2[i]) : a.next_q1[i];
        const float y = bellman_target(a.reward[i], a.discount ? a.discount[i] : a.gamma,
                                       a.terminal[i], next_q);
        a.target[i] = y;
        const float d1 = __fsub_rn(a.pred_q1[i], y);
        a.grad1[i] = __fmul_rn(a.norm, d1);
        s1 = __fadd_rn(s1, __fmul_rn(d1, d1));
        if (a.pred_q2) {
            const float d2 = __fsub_rn(a.pred_q2[i], y);
            a.grad2[i] = __fmul_rn(a.norm, d2);
            s2 = __fadd_rn(s2, __fmul_rn(d2, d2));
        }
    }
    cta_sum2(s1, s2);
    const float n = (float)a.n;
    if (gridDim.x == 1) {
        if (threadIdx.x == 0) {
            *a.loss1 = __fdiv_rn(s1, n);
            if (a.pred_q2) *a.loss2 = __fdiv_rn(s2, n);
        }
        return;
    }
    __shared__ bool last;
    if (threadIdx.x == 0) {
        a.partial[blockIdx.x] = s1;
        a.partial[gridDim.x + blockIdx.x] = s2;
        __threadfence();
        last = atomicInc(&g_done_counter[a.ticket], gridDim.x - 1) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    s1 = s2 = 0.f;
    for (int j = threadIdx.x; j < (int)gridDim.x; j += CRITIC_THREADS) {
        s1 = __fadd_rn(s1, __ldcg(a.partial + j));
        s2 = __fadd_rn(s2, __ldcg(a.partial + gridDim.x + j));
    }
    cta_sum2(s1, s2);
    if (threadIdx.x == 0) {
        *a.loss1 = __fdiv_rn(s1, n);
        if (a.pred_q2) *a.loss2 = __fdiv_rn(s2, n);
    }
}

} // namespace

extern "C" int b2rl_polyak(const b2rl_tensor_pair *pairs_host, int32_t n_pairs, double tau,
                           void *stream)
{
    B2RL_REQUIRE(pairs_host || n_pairs == 0, B2RL_ERR_INVALID, "polyak: null pairs");
    B2RL_REQUIRE(n_pairs >= 0, B2RL_ERR_RANGE, "polyak: negative count");
    B2RL_REQUIRE(tau >= 0.0 && tau <= 1.0, B2RL_ERR_RANGE, "polyak: tau must be in [0, 1]");
    // every pair is checked before the first launch, so a refused call changes no target
    for (int i = 0; i < n_pairs; i++) {
        const b2rl_tensor_pair &p = pairs_host[i];
        B2RL_REQUIRE(p.dst && p.src && p.numel >= 0, B2RL_ERR_INVALID, "polyak: bad pair %d", i);
    }
    cudaStream_t s = (cudaStream_t)stream;
    for (int done = 0; done < n_pairs; done += POLYAK_MAX) {
        PolyakArgs a;
        a.n = n_pairs - done < POLYAK_MAX ? n_pairs - done : POLYAK_MAX;
        a.keep = (float)(1.0 - tau);
        a.tau = (float)tau;
        int blocks = 0;
        for (int i = 0; i < a.n; i++) {
            const b2rl_tensor_pair &p = pairs_host[done + i];
            a.dst[i] = (float *)p.dst;
            a.src[i] = (const float *)p.src;
            a.numel[i] = p.numel;
            a.first_block[i] = blocks;
            blocks += (int)((p.numel + POLYAK_CHUNK - 1) / POLYAK_CHUNK);
        }
        a.first_block[a.n] = blocks;
        if (blocks == 0) continue;
        k_polyak<<<blocks, 256, 0, s>>>(a);
        B2RL_CUDA(cudaGetLastError());
    }
    return B2RL_OK;
}

extern "C" int b2rl_sac_target(const float *reward, const float *discount, const float *terminal,
                               const float *q1, const float *q2, const float *log_prob,
                               const float *temperature_dev, float temperature, int32_t n,
                               float *out, void *stream)
{
    B2RL_REQUIRE(reward && discount && terminal && q1 && q2 && log_prob && out, B2RL_ERR_INVALID,
                 "sac_target: null argument");
    B2RL_REQUIRE(n > 0, B2RL_ERR_RANGE, "sac_target: empty batch");
    k_sac_target<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(
        reward, discount, terminal, q1, q2, log_prob, temperature_dev, temperature, n, out);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}

extern "C" int b2rl_td3_smooth(const float *action, const float *noise, int64_t n, float *out,
                               void *stream)
{
    B2RL_REQUIRE(action && noise && out, B2RL_ERR_INVALID, "td3_smooth: null argument");
    B2RL_REQUIRE(n > 0 && (n + 255) / 256 <= INT32_MAX, B2RL_ERR_RANGE,
                 "td3_smooth: need 0 < n < 2^39, got %lld", (long long)n);
    k_td3_smooth<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(action, noise,
                                                                                 n, out);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}

extern "C" int b2rl_td3_critic_loss(const float *reward, const float *discount, float gamma,
                                    const float *terminal, const float *next_q1,
                                    const float *next_q2, const float *pred_q1,
                                    const float *pred_q2, int32_t n, float *target, float *grad1,
                                    float *grad2, float *loss1, float *loss2, float *partial,
                                    void *stream)
{
    B2RL_REQUIRE(reward && terminal && next_q1 && pred_q1 && target && grad1 && loss1,
                 B2RL_ERR_INVALID, "td3_critic_loss: null argument");
    B2RL_REQUIRE(!pred_q2 || (grad2 && loss2), B2RL_ERR_INVALID,
                 "td3_critic_loss: a second critic needs grad2 and loss2");
    B2RL_REQUIRE(n > 0, B2RL_ERR_RANGE, "td3_critic_loss: empty batch");
    const int ctas = (n + CRITIC_ROWS - 1) / CRITIC_ROWS;
    B2RL_REQUIRE(ctas == 1 || partial, B2RL_ERR_INVALID,
                 "td3_critic_loss: n = %d > %d needs the partial-sum workspace", (int)n,
                 CRITIC_ROWS);
    CriticLossArgs a{reward, discount, terminal, next_q1, next_q2, pred_q1, pred_q2};
    a.gamma = gamma;
    a.norm = (float)(2.0 / (double)n);
    a.n = n;
    a.target = target;
    a.grad1 = grad1;
    a.grad2 = grad2;
    a.loss1 = loss1;
    a.loss2 = loss2;
    a.partial = partial;
    a.ticket = b2rl_next_ticket();
    k_td3_critic_loss<<<ctas, CRITIC_THREADS, 0, (cudaStream_t)stream>>>(a);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}
