// sac.cu -- K9: the launch-bound elementwise tail of the SAC / TD3 / DDPG update.
//
// Replaces (reference, one tiny ATen launch per tensor and per operator):
//   pfrl/utils/copy_param.py:9-22              soft_copy_param (Polyak averaging,
//                                              2 launches per state_dict entry)
//   pfrl/agents/soft_actor_critic.py:225-240   entropy-regularised TD target
//                                              (min, mul, sub, flatten, mul, mul, add)
// Both are rounded exactly like the reference's sequence of separate fp32
// operations (no FMA contraction), so parameters stay bit-identical to an
// eager run.
#include "b2rl_internal.cuh"

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
