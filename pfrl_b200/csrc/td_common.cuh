// td_common.cuh -- pieces of the scalar TD losses shared by losses.cu and naf.cu: the
// reference's Bellman target, the per-sample outputs and loss term, its gradient, and the
// deterministic batch reduction.  Each translation unit that includes this file gets its own
// completion counters; a launch uses the one of its own unit.
#pragma once
#include <math.h>

#include "b2rl_internal.cuh"

namespace {

__device__ unsigned int g_done_counter[B2RL_N_TICKETS]; // zero-initialised, self-resetting

__device__ __forceinline__ float warp_sum(float v)
{
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Deterministic final reduction: the last CTA to arrive sums term[i] for
// i < n in a fixed order and writes *out = sum / divisor.
__device__ void finish_sum(const float *term, int n, float divisor, float *out, float *sh,
                           unsigned ticket)
{
    __shared__ bool last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int prev = atomicInc(&g_done_counter[ticket], gridDim.x - 1);
        last = (prev == gridDim.x - 1);
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    float s = 0.f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) s += __ldcg(term + i);
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 32) {
        s = threadIdx.x < (blockDim.x >> 5) ? sh[threadIdx.x] : 0.f;
        s = warp_sum(s);
        if (threadIdx.x == 0) *out = __fdiv_rn(s, divisor);
    }
}

// r + discount * (1 - terminal) * next_v, dqn.py:405
__device__ __forceinline__ float bellman_target(float r, float discount, float terminal,
                                                float next_v)
{
    return __fadd_rn(r, __fmul_rn(__fmul_rn(discount, __fsub_rn(1.0f, terminal)), next_v));
}

// Writes y, t, |y - t| and the (weighted) Huber / 0.5 MSE term of sample i (dqn.py:44-104).
__device__ __forceinline__ void td_outputs(float y, float t, int i, int clip_delta,
                                           const float *weights, float *y_out, float *t_out,
                                           float *delta_out, float *term)
{
    const float d = __fsub_rn(y, t);
    const float ad = fabsf(d);
    float l;
    if (clip_delta)
        l = ad < 1.0f ? __fmul_rn(__fmul_rn(0.5f, d), d) : __fsub_rn(ad, 0.5f);
    else
        l = __fmul_rn(__fmul_rn(d, d), 0.5f);
    y_out[i] = y;
    t_out[i] = t;
    delta_out[i] = ad;
    term[i] = weights ? __fmul_rn(l, weights[i]) : l;
}

// d loss / d y of sample i for the scalar TD loss (Huber'(y - t) with delta = 1, or y - t),
// times the upstream gradient, divided by B for "mean", times the importance weight.
__device__ __forceinline__ float td_grad(const float *y, const float *t, const float *weights,
                                         const float *grad_loss, int i, int B, int clip_delta,
                                         int mean)
{
    float g = grad_loss[0];
    if (mean) g = g / (float)B;
    if (weights) g *= weights[i];
    float d = y[i] - t[i];
    if (clip_delta) d = fminf(fmaxf(d, -1.0f), 1.0f); // Huber'(d), delta = 1
    return g * d;
}

} // namespace
