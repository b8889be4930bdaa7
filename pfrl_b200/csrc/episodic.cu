// episodic.cu -- the minibatch of a recurrent (episodic) update in one launch.
//
// Replaces (reference, pure Python + torch collate + two copies):
//   pfrl/replay_buffer.py:219-287    batch_recurrent_experiences (batch_states per
//                                    episode, Python lists of actions / rewards /
//                                    terminals, concatenate_recurrent_states, H2D)
//   pfrl/utils/recurrent.py:249-277  pack_sequences_recursive (pack_sequence copies
//                                    everything again into time-major order)
//
// The rows are written straight to their packed (time-major) positions: step t of
// sequence b goes to row sum_{t' < t} batch_sizes[t'] + b = sum_b' min(len[b'], t) + b,
// which each CTA computes from the lengths it is launched with.  The observation copy
// is the one of k_gather (b2rl_gather_part_piece), one CTA per (packed row, side, part,
// piece) -- the grid follows sum(len), not B * max(len), so whole long episodes cost no
// idle CTAs; each CTA finds the (step, sequence) of its row by a binary search over the
// row offsets.  The scalars and the first records' recurrent states are written by
// grid-strided threads.
#include "b2rl_internal.cuh"

struct SeqArgs {
    const uint8_t *parts;
    const int32_t *state_parts, *next_parts;
    const uint8_t *action;
    const double *rewards; // n_step = 1: one reward per record
    const uint8_t *terminal;
    const B2rlDevState *st;
    long long nslots;
    int B, Lmax, N, stack, part_bytes, action_bytes, obs_mode;
    float obs_scale;
    int has_states;
    uint8_t *o_state, *o_next, *o_action;
    float *o_reward, *o_terminal;
    b2rl_seq_states rs;
    long long first[B2RL_SEQ_MAX_B];
    int len[B2RL_SEQ_MAX_B];
};

// sum_b min(len[b], t): the packed row of step t of sequence 0.  All lanes read
// the same length at a time (a constant-bank broadcast).
__device__ __forceinline__ int seq_row0_thread(const SeqArgs &a, int t)
{
    int s = 0;
    for (int j = 0; j < a.B; j++) s += min(a.len[j], t);
    return s;
}

// Same sum, computed by the whole 256-thread CTA (t uniform over the CTA).
__device__ __forceinline__ int seq_row0_block(const SeqArgs &a, int t)
{
    __shared__ int part[8];
    int s = 0;
    for (int j = threadIdx.x; j < a.B; j += 256) s += min(a.len[j], t);
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
    __syncthreads();
    s = 0;
#pragma unroll
    for (int w = 0; w < 8; w++) s += part[w];
    __syncthreads(); // part[] is rewritten by the next call
    return s;
}

__global__ void __launch_bounds__(256) k_seq_gather(const __grid_constant__ SeqArgs a)
{
    const long long items = (long long)a.N * 2 * a.stack * GATHER_SPLIT;
    const long long blk = blockIdx.x;
    if (blk < items) {
        const int piece = (int)(blk % GATHER_SPLIT);
        const long long item = blk / GATHER_SPLIT;
        const int part = (int)(item % a.stack);
        const int side = (int)((item / a.stack) & 1);
        const int row = (int)(item / (2 * a.stack));
        uint8_t *out = side ? a.o_next : a.o_state;
        if (out) { // uniform over the CTA
            const int t =
                b2rl_packed_step(row, a.Lmax, [&](int u) { return seq_row0_block(a, u); });
            const int b = row - seq_row0_block(a, t);
            const long long slot = b2rl_logical_slot(a.st, a.nslots, a.first[b] + t);
            const int32_t ps = (side ? a.next_parts : a.state_parts)[slot * a.stack + part];
            b2rl_gather_part_piece(a.parts + (size_t)ps * a.part_bytes, out,
                                   (size_t)row * a.stack + part, a.part_bytes, piece,
                                   a.obs_mode, a.obs_scale);
        }
    }
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long nthreads = (long long)gridDim.x * blockDim.x;
    // scalars: one thread per (sequence, step)
    for (long long k = gid; k < (long long)a.B * a.Lmax; k += nthreads) {
        const int b = (int)(k / a.Lmax), t = (int)(k % a.Lmax);
        if (t < a.len[b]) {
            const long long row = seq_row0_thread(a, t) + b;
            const long long slot = b2rl_logical_slot(a.st, a.nslots, a.first[b] + t);
            if (a.o_reward) a.o_reward[row] = (float)a.rewards[slot];
            if (a.o_terminal) a.o_terminal[row] = a.terminal[slot] ? 1.0f : 0.0f;
            if (a.o_action) {
                const uint8_t *src = a.action + slot * a.action_bytes;
                uint8_t *dst = a.o_action + row * a.action_bytes;
                for (int i = 0; i < a.action_bytes; i++) dst[i] = src[i];
            }
        }
    }
    // recurrent states of each sequence's first record: [side][b][float of the row]
    if (a.has_states) {
        b2rl_seq_states_write(a, gid, nthreads, [&](int b) {
            return (a.st->npop + a.first[b]) % a.rs.ring_rows;
        });
    }
}

extern "C" int b2rl_replay_gather_sequences(b2rl_replay *h, const int64_t *first_host,
                                            const int32_t *len_host, const int64_t *end_host,
                                            int32_t B, int obs_mode, float obs_scale,
                                            const b2rl_seq_out *out,
                                            const b2rl_seq_states *states, void *stream)
{
    B2RL_REQUIRE(h && out && first_host && len_host && end_host, B2RL_ERR_INVALID,
                 "null argument");
    B2RL_REQUIRE(B > 0 && B <= B2RL_SEQ_MAX_B, B2RL_ERR_RANGE,
                 "gather_sequences: B = %d must be in [1, %d]", B, B2RL_SEQ_MAX_B);
    B2RL_REQUIRE(obs_mode == B2RL_OBS_RAW || obs_mode == B2RL_OBS_U8_TO_F32, B2RL_ERR_INVALID,
                 "unknown obs_mode %d", obs_mode);
    const b2rl_replay_config &c = h->cfg;
    B2RL_REQUIRE(c.n_step == 1, B2RL_ERR_INVALID,
                 "gather_sequences needs a store built with n_step = 1 (has %d)", c.n_step);
    const int64_t live = h->napp - h->npop;
    for (int b = 0; b < B; b++) {
        B2RL_REQUIRE(len_host[b] >= 1, B2RL_ERR_RANGE,
                     "gather_sequences: len[%d] = %d must be >= 1", b, len_host[b]);
        B2RL_REQUIRE(b == 0 || len_host[b] <= len_host[b - 1], B2RL_ERR_RANGE,
                     "gather_sequences: lengths must be sorted longest first (len[%d] = %d > "
                     "len[%d] = %d)", b, len_host[b], b - 1, len_host[b - 1]);
        B2RL_REQUIRE(first_host[b] >= 0 && end_host[b] <= live, B2RL_ERR_RANGE,
                     "gather_sequences: sequence %d [%lld, %lld) outside the %lld live records",
                     b, (long long)first_host[b], (long long)end_host[b], (long long)live);
        B2RL_REQUIRE(first_host[b] + len_host[b] <= end_host[b], B2RL_ERR_RANGE,
                     "gather_sequences: sequence %d (first %lld, len %d) runs past the end of "
                     "its episode (%lld)", b, (long long)first_host[b], len_host[b],
                     (long long)end_host[b]);
    }
    if (states) {
        B2RL_REQUIRE(states->ring && states->present && states->ring_rows > 0 &&
                         states->row_floats > 0 && states->n_leaves >= 1 &&
                         states->n_leaves <= B2RL_SEQ_MAX_LEAVES,
                     B2RL_ERR_INVALID, "gather_sequences: invalid recurrent-state ring");
        for (int i = 0; i < states->n_leaves; i++)
            B2RL_REQUIRE(states->offset[i] >= 0 && states->d0[i] >= 1 && states->inner[i] >= 1 &&
                             states->offset[i] + (int64_t)states->d0[i] * states->inner[i] <=
                                 states->row_floats,
                         B2RL_ERR_INVALID, "gather_sequences: leaf %d outside the ring row", i);
    }
    cudaStream_t s = (cudaStream_t)stream;
    B2RL_CUDA(cudaSetDevice(c.device));
    SeqArgs a;
    a.parts = h->parts;
    a.state_parts = h->state_parts;
    a.next_parts = h->next_parts;
    a.action = h->action;
    a.rewards = h->rewards;
    a.terminal = h->terminal;
    a.st = h->st;
    a.nslots = h->nslots;
    a.B = B;
    a.Lmax = len_host[0];
    long long total = 0;
    for (int b = 0; b < B; b++) total += len_host[b];
    B2RL_REQUIRE(total < (1LL << 30), B2RL_ERR_RANGE, "gather_sequences: batch too large");
    a.N = (int)total;
    a.stack = c.stack;
    a.part_bytes = c.part_bytes;
    a.action_bytes = c.action_bytes;
    a.obs_mode = obs_mode;
    a.obs_scale = obs_scale;
    a.o_state = (uint8_t *)out->state;
    a.o_next = (uint8_t *)out->next_state;
    a.o_action = (uint8_t *)out->action;
    a.o_reward = out->reward;
    a.o_terminal = out->terminal;
    a.has_states = states != nullptr;
    if (states) a.rs = *states;
    else memset(&a.rs, 0, sizeof(a.rs));
    for (int b = 0; b < B; b++) {
        a.first[b] = first_host[b];
        a.len[b] = len_host[b];
    }
    long long grid = total * 2 * c.stack * GATHER_SPLIT;
    if (states) {
        // grid-strided: at most 1024 CTAs are spent on the states alone
        long long need = (2LL * B * states->row_floats + 255) / 256;
        if (need > 1024) need = 1024;
        if (grid < need) grid = need;
    }
    B2RL_REQUIRE(grid < (1LL << 31), B2RL_ERR_RANGE, "gather_sequences: batch too large");
    k_seq_gather<<<(unsigned)grid, 256, 0, s>>>(a);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}
