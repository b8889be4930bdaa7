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

GatherArgs b2rl_gather_args(const b2rl_replay *h, int n, const double *gamma_pow_host,
                            int obs_mode, float obs_scale, const b2rl_batch_out *out)
{
    const b2rl_replay_config &c = h->cfg;
    GatherArgs g;
    g.parts = h->parts;
    g.state_parts = h->state_parts;
    g.next_parts = h->next_parts;
    g.action = h->action;
    g.rewards = h->rewards;
    g.len = h->len;
    g.terminal = h->terminal;
    g.slots = h->last_slots;
    for (int i = 0; i <= c.n_step; i++) g.gamma_pow[i] = gamma_pow_host[i];
    g.n = n;
    g.stack = c.stack;
    g.part_bytes = c.part_bytes;
    g.n_step = c.n_step;
    g.action_bytes = c.action_bytes;
    g.obs_mode = obs_mode;
    g.obs_scale = obs_scale;
    g.o_side[0] = (uint8_t *)out->state;
    g.o_side[1] = (uint8_t *)out->next_state;
    g.o_action = (uint8_t *)out->action;
    g.o_reward = out->reward;
    g.o_terminal = out->terminal;
    g.o_discount = out->discount;
    g.o_step_rewards = out->step_rewards;
    g.o_len = out->len;
    return g;
}

// slot of experience k: logical index index[k], or the last sample's k-th draw (index null)
__device__ __forceinline__ long long gather_slot(const GatherArgs &a, const long long *index,
                                                 const B2rlDevState *st, long long nslots, int k)
{
    if (!index) return a.slots[k];
    return b2rl_logical_slot(st, nslots, index[k]);
}

// Grid: one CTA per (experience, side, part, piece) (GATHER_SPLIT pieces per
// part, b2rl_internal.cuh); the slot / part-index lookups are done once per
// CTA.  The first `tail` CTAs additionally emit the scalars.
__global__ void __launch_bounds__(256) k_gather(GatherArgs a, const long long *index,
                                                const B2rlDevState *st, long long nslots)
{
    const int items = a.n * 2 * a.stack * GATHER_SPLIT;
    const int b = blockIdx.x;
    if (b < items) {
        const int piece = b % GATHER_SPLIT;
        const int item = b / GATHER_SPLIT;
        const int part = item % a.stack;
        const int side = (item / a.stack) & 1;
        const int k = item / (2 * a.stack);
        uint8_t *out = a.o_side[side];
        if (out) {
            const long long slot = gather_slot(a, index, st, nslots, k);
            const int32_t ps = (side ? a.next_parts : a.state_parts)[slot * a.stack + part];
            const uint8_t *src = a.parts + (size_t)ps * a.part_bytes;
            b2rl_gather_part_piece(src, out, (size_t)k * a.stack + part, a.part_bytes, piece,
                                   a.obs_mode, a.obs_scale);
        }
    }
    // scalar tail: one thread per experience
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= a.n) return;
    b2rl_gather_scalars(a, k, gather_slot(a, index, st, nslots, k));
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
    const GatherArgs a = b2rl_gather_args(h, n, gamma_pow_host, obs_mode, obs_scale, out);
    const int tail = (n + 255) / 256;
    int grid = n * 2 * h->cfg.stack * GATHER_SPLIT;
    if (grid < tail) grid = tail;
    k_gather<<<grid, 256, 0, s>>>(a, (const long long *)index_dev, h->st, h->nslots);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}
