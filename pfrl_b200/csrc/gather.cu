// gather.cu -- minibatch assembly straight out of the HBM part ring.
//
// Replaces (reference, pure Python + torch collate + H2D copy):
//   pfrl/replay_buffer.py:157-212     batch_experiences
//   pfrl/utils/batch_states.py:18-36  batch_states (phi per observation,
//                                      default_collate, .to(device))
//
// Traffic per sampled experience (Atari, f32 out): up to 2*stack parts read
// (7 056 B each, the shared ones hit L2) and 2*stack*part_bytes*4 B written.
// The kernel is a pure stream: every thread turns one 32-bit word of a part
// (4 pixels) into one 128-bit store, so both the loads (128 B per warp
// instruction) and the stores (512 B per warp instruction) are fully
// coalesced.
#include <math.h>

#include "b2rl_internal.cuh"

struct GatherArgs {
    const uint8_t *parts;
    const int32_t *state_parts, *next_parts;
    const uint8_t *action;
    const double *rewards;
    const uint8_t *len, *terminal;
    const B2rlDevState *st;
    const int32_t *slots;      // slots of the last sample, or null
    const long long *index;    // logical indices, or null
    double gamma_pow[9];       // gamma**i, i <= n_step (<= 8), passed by value
    long long nslots;
    int n, stack, part_bytes, n_step, action_bytes;
    int obs_mode;
    float obs_scale;
    uint8_t *o_state, *o_next, *o_action;
    float *o_reward, *o_terminal, *o_discount;
    double *o_step_rewards;
    uint8_t *o_len;
};

__device__ __forceinline__ long long gather_slot(const GatherArgs &a, int k)
{
    if (a.slots) return a.slots[k];
    return b2rl_logical_slot(a.st, a.nslots, a.index[k]);
}

// Grid: one CTA per (experience, side, part, piece) (GATHER_SPLIT pieces per
// part, b2rl_internal.cuh); the slot / part-index lookups are done once per
// CTA.  The first `tail` CTAs additionally emit the scalars.
__global__ void __launch_bounds__(256) k_gather(GatherArgs a)
{
    const int items = a.n * 2 * a.stack * GATHER_SPLIT;
    const int b = blockIdx.x;
    if (b < items) {
        const int piece = b % GATHER_SPLIT;
        const int item = b / GATHER_SPLIT;
        const int part = item % a.stack;
        const int side = (item / a.stack) & 1;
        const int k = item / (2 * a.stack);
        uint8_t *out = side ? a.o_next : a.o_state;
        if (out) {
            const long long slot = gather_slot(a, k);
            const int32_t ps = (side ? a.next_parts : a.state_parts)[slot * a.stack + part];
            const uint8_t *src = a.parts + (size_t)ps * a.part_bytes;
            b2rl_gather_part_piece(src, out, (size_t)k * a.stack + part, a.part_bytes, piece,
                                   a.obs_mode, a.obs_scale);
        }
    }
    // scalar tail: one thread per experience
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= a.n) return;
    const long long slot = gather_slot(a, k);
    const int len = a.len[slot];
    if (a.o_reward) {
        // sum((gamma**i) * r_i) evaluated like CPython's float sum():
        // Neumaier-compensated accumulation (replay_buffer.py:183-190)
        double s = 0.0, c = 0.0;
        for (int i = 0; i < len; i++) {
            const double x = __dmul_rn(a.gamma_pow[i], a.rewards[slot * a.n_step + i]);
            const double t = __dadd_rn(s, x);
            if (fabs(s) >= fabs(x))
                c = __dadd_rn(c, __dadd_rn(__dsub_rn(s, t), x));
            else
                c = __dadd_rn(c, __dadd_rn(__dsub_rn(x, t), s));
            s = t;
        }
        a.o_reward[k] = (float)__dadd_rn(s, c);
    }
    if (a.o_terminal) a.o_terminal[k] = a.terminal[slot] ? 1.0f : 0.0f;
    if (a.o_discount) a.o_discount[k] = (float)a.gamma_pow[len]; // gamma ** len(elem), :203
    if (a.o_len) a.o_len[k] = (uint8_t)len;
    if (a.o_step_rewards)
        for (int i = 0; i < a.n_step; i++)
            a.o_step_rewards[(size_t)k * a.n_step + i] = i < len ? a.rewards[slot * a.n_step + i] : 0.0;
    if (a.o_action) {
        const uint8_t *src = a.action + slot * a.action_bytes;
        uint8_t *dst = a.o_action + (size_t)k * a.action_bytes;
        for (int i = 0; i < a.action_bytes; i++) dst[i] = src[i];
    }
}

extern "C" int b2rl_replay_gather(b2rl_replay *h, const int64_t *index_dev, int32_t n,
                                  const double *gamma_pow_host, int obs_mode, float obs_scale,
                                  const b2rl_batch_out *out, void *stream)
{
    B2RL_REQUIRE(h && out && gamma_pow_host, B2RL_ERR_INVALID, "null argument");
    B2RL_REQUIRE(n > 0, B2RL_ERR_RANGE, "gather: n must be > 0");
    B2RL_REQUIRE(obs_mode == B2RL_OBS_RAW || obs_mode == B2RL_OBS_U8_TO_F32, B2RL_ERR_INVALID,
                 "unknown obs_mode %d", obs_mode);
    if (!index_dev)
        B2RL_REQUIRE(h->wait_priority && n == h->last_n, B2RL_ERR_PROTOCOL,
                     "gather(index=NULL) needs a pending sample of the same size");
    cudaStream_t s = (cudaStream_t)stream;
    B2RL_CUDA(cudaSetDevice(h->cfg.device));
    const b2rl_replay_config &c = h->cfg;
    GatherArgs a;
    a.parts = h->parts;
    a.state_parts = h->state_parts;
    a.next_parts = h->next_parts;
    a.action = h->action;
    a.rewards = h->rewards;
    a.len = h->len;
    a.terminal = h->terminal;
    a.st = h->st;
    a.slots = index_dev ? nullptr : h->last_slots;
    a.index = (const long long *)index_dev;
    for (int i = 0; i <= c.n_step; i++) a.gamma_pow[i] = gamma_pow_host[i];
    a.nslots = h->nslots;
    a.n = n;
    a.stack = c.stack;
    a.part_bytes = c.part_bytes;
    a.n_step = c.n_step;
    a.action_bytes = c.action_bytes;
    a.obs_mode = obs_mode;
    a.obs_scale = obs_scale;
    a.o_state = (uint8_t *)out->state;
    a.o_next = (uint8_t *)out->next_state;
    a.o_action = (uint8_t *)out->action;
    a.o_reward = out->reward;
    a.o_terminal = out->terminal;
    a.o_discount = out->discount;
    a.o_step_rewards = out->step_rewards;
    a.o_len = out->len;
    const int tail = (n + 255) / 256;
    int grid = n * 2 * c.stack * GATHER_SPLIT;
    if (grid < tail) grid = tail;
    k_gather<<<grid, 256, 0, s>>>(a);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}
