// rollout.cu -- the packed-sequence minibatch of a recurrent PPO update in one launch.
//
// Replaces (reference, pure Python + torch collate + copies):
//   pfrl/agents/ppo.py:56-107   _add_log_prob_and_value_to_episodes_recurrent (batch_states
//                               per episode, concatenate_recurrent_states, pack_sequence)
//   pfrl/agents/ppo.py:534-606  _update_once_recurrent (the same, plus torch.tensor of the
//                               per-transition action, adv, log_prob, v_pred, v_teacher)
//
// The rollout is time-major on the device: flat slot s = t * E + e.  Sequence b is env
// first[b] % E from step first[b] / E on, so its step t is the flat slot first[b] + t * E,
// written to the packed row row_off[t] + b (pack_sequence order).  Every column is copied
// by grid-strided threads in units of 16, 8, 4 or 1 bytes (the widest that divides the
// row and both base addresses); each thread finds the (step, sequence) of its row by a
// binary search over the row offsets, which sit in L1 after the first touch.  One extra
// grid plane writes the flat slot of every row and the first slots' recurrent states
// (b2rl_seq_states_write, shared with k_seq_gather).
#include "b2rl_internal.cuh"

struct RolloutArgs {
    const long long *tab; // device: first[B], len[B], row_off[Lmax + 1]
    long long E;
    int B, Lmax, N, n_cols;
    const uint8_t *src[B2RL_ROLLOUT_MAX_COLS];
    uint8_t *dst[B2RL_ROLLOUT_MAX_COLS];
    long long units[B2RL_ROLLOUT_MAX_COLS]; // copy units per row
    int lw[B2RL_ROLLOUT_MAX_COLS];          // log2 of the unit's bytes: 4, 3, 2 or 0
    long long *index_out;
    int has_states;
    b2rl_seq_states rs;
};

template <class V>
__device__ __forceinline__ void rollout_copy_unit(const uint8_t *src, uint8_t *dst,
                                                  long long s_unit, long long d_unit)
{
    reinterpret_cast<V *>(dst)[d_unit] = __ldg(reinterpret_cast<const V *>(src) + s_unit);
}

__global__ void __launch_bounds__(256) k_rollout_seq_gather(const __grid_constant__ RolloutArgs a)
{
    const long long *first = a.tab;
    const long long *row_off = a.tab + 2 * a.B;
    auto row0 = [&](int t) { return __ldg(row_off + t); };
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long nthreads = (long long)gridDim.x * blockDim.x;
    const int c = blockIdx.y;
    if (c < a.n_cols) {
        const long long units = a.units[c];
        const long long total = units * a.N;
        const int lw = a.lw[c];
        for (long long u = gid; u < total; u += nthreads) {
            const int row = (int)(u / units);
            const long long k = u - (long long)row * units;
            const int t = b2rl_packed_step(row, a.Lmax, row0);
            const int b = row - (int)row0(t);
            const long long slot = __ldg(first + b) + (long long)t * a.E;
            const long long s_unit = slot * units + k;
            if (lw == 4) rollout_copy_unit<uint4>(a.src[c], a.dst[c], s_unit, u);
            else if (lw == 3) rollout_copy_unit<uint2>(a.src[c], a.dst[c], s_unit, u);
            else if (lw == 2) rollout_copy_unit<uint32_t>(a.src[c], a.dst[c], s_unit, u);
            else rollout_copy_unit<uint8_t>(a.src[c], a.dst[c], s_unit, u);
        }
        return;
    }
    if (a.index_out) {
        for (long long row = gid; row < a.N; row += nthreads) {
            const int t = b2rl_packed_step((int)row, a.Lmax, row0);
            const int b = (int)row - (int)row0(t);
            a.index_out[row] = __ldg(first + b) + (long long)t * a.E;
        }
    }
    if (a.has_states)
        b2rl_seq_states_write(a, gid, nthreads, [&](int b) { return __ldg(first + b); });
}

static int rollout_unit_log2(const void *src, const void *dst, int64_t row_bytes)
{
    const uintptr_t bits = (uintptr_t)src | (uintptr_t)dst | (uintptr_t)row_bytes;
    if (bits % 16 == 0) return 4;
    if (bits % 8 == 0) return 3;
    if (bits % 4 == 0) return 2;
    return 0;
}

extern "C" int b2rl_rollout_gather_sequences(const int64_t *table_host, int64_t *table_dev,
                                             int64_t table_dev_capacity, int32_t B, int64_t T,
                                             int64_t E, const b2rl_rollout_col *cols,
                                             int32_t n_cols, int64_t *index_out,
                                             const b2rl_seq_states *states, void *stream)
{
    B2RL_REQUIRE(table_host && table_dev && (cols || n_cols == 0), B2RL_ERR_INVALID,
                 "rollout_gather_sequences: null argument");
    B2RL_REQUIRE(B >= 1 && T >= 1 && E >= 1 && T * E < (1LL << 40), B2RL_ERR_RANGE,
                 "rollout_gather_sequences: B = %d, T = %lld, E = %lld", B, (long long)T,
                 (long long)E);
    B2RL_REQUIRE(n_cols >= 0 && n_cols <= B2RL_ROLLOUT_MAX_COLS, B2RL_ERR_RANGE,
                 "rollout_gather_sequences: %d columns (at most %d)", n_cols,
                 B2RL_ROLLOUT_MAX_COLS);
    const int64_t *first = table_host, *len = table_host + B, *row_off = table_host + 2 * (int64_t)B;
    for (int b = 0; b < B; b++) {
        B2RL_REQUIRE(len[b] >= 1, B2RL_ERR_RANGE,
                     "rollout_gather_sequences: len[%d] = %lld must be >= 1", b, (long long)len[b]);
        B2RL_REQUIRE(b == 0 || len[b] <= len[b - 1], B2RL_ERR_RANGE,
                     "rollout_gather_sequences: lengths must be sorted longest first (len[%d] = "
                     "%lld > len[%d] = %lld)", b, (long long)len[b], b - 1, (long long)len[b - 1]);
        B2RL_REQUIRE(first[b] >= 0 && first[b] / E + len[b] <= T, B2RL_ERR_RANGE,
                     "rollout_gather_sequences: sequence %d (env %lld, step %lld, len %lld) runs "
                     "past the %lld steps of the rollout", b, (long long)(first[b] % E),
                     (long long)(first[b] / E), (long long)len[b], (long long)T);
    }
    const int64_t Lmax = len[0];
    B2RL_REQUIRE(2 * (int64_t)B + Lmax + 1 <= table_dev_capacity, B2RL_ERR_RANGE,
                 "rollout_gather_sequences: the device table holds %lld values, %lld needed",
                 (long long)table_dev_capacity, (long long)(2 * (int64_t)B + Lmax + 1));
    // row_off[t + 1] - row_off[t] = #{b : len[b] > t} = batch_sizes[t]
    B2RL_REQUIRE(row_off[0] == 0, B2RL_ERR_RANGE, "rollout_gather_sequences: row_off[0] != 0");
    for (int64_t t = 0, live = B; t < Lmax; t++) {
        while (live > 0 && len[live - 1] <= t) live--;
        B2RL_REQUIRE(row_off[t + 1] - row_off[t] == live, B2RL_ERR_RANGE,
                     "rollout_gather_sequences: row_off[%lld] is not the row offset of the "
                     "lengths", (long long)(t + 1));
    }
    const int64_t N = row_off[Lmax];
    B2RL_REQUIRE(N < (1LL << 31) - 1, B2RL_ERR_RANGE, "rollout_gather_sequences: batch too large");
    RolloutArgs a;
    memset(&a, 0, sizeof(a));
    a.tab = (const long long *)table_dev;
    a.E = E;
    a.B = B;
    a.Lmax = (int)Lmax;
    a.N = (int)N;
    a.n_cols = n_cols;
    long long max_units = N;
    for (int c = 0; c < n_cols; c++) {
        B2RL_REQUIRE(cols[c].src && cols[c].dst && cols[c].row_bytes >= 1, B2RL_ERR_INVALID,
                     "rollout_gather_sequences: column %d is invalid", c);
        a.src[c] = (const uint8_t *)cols[c].src;
        a.dst[c] = (uint8_t *)cols[c].dst;
        a.lw[c] = rollout_unit_log2(cols[c].src, cols[c].dst, cols[c].row_bytes);
        a.units[c] = cols[c].row_bytes >> a.lw[c];
        B2RL_REQUIRE(a.units[c] * N < (1LL << 50), B2RL_ERR_RANGE,
                     "rollout_gather_sequences: column %d too large", c);
        if (a.units[c] * N > max_units) max_units = a.units[c] * N;
    }
    a.index_out = (long long *)index_out;
    if (states) {
        B2RL_REQUIRE(states->ring && states->present && states->ring_rows >= T * E &&
                         states->row_floats > 0 && states->n_leaves >= 1 &&
                         states->n_leaves <= B2RL_SEQ_MAX_LEAVES,
                     B2RL_ERR_INVALID, "rollout_gather_sequences: invalid recurrent-state ring");
        for (int i = 0; i < states->n_leaves; i++)
            B2RL_REQUIRE(states->offset[i] >= 0 && states->d0[i] >= 1 && states->inner[i] >= 1 &&
                             states->offset[i] + (int64_t)states->d0[i] * states->inner[i] <=
                                 states->row_floats,
                         B2RL_ERR_INVALID, "rollout_gather_sequences: leaf %d outside the ring row",
                         i);
        a.has_states = 1;
        a.rs = *states;
        if (2LL * B * states->row_floats > max_units) max_units = 2LL * B * states->row_floats;
    }
    cudaStream_t s = (cudaStream_t)stream;
    B2RL_CUDA(cudaMemcpyAsync(table_dev, table_host, (2 * (size_t)B + Lmax + 1) * sizeof(int64_t),
                              cudaMemcpyHostToDevice, s));
    // grid-strided: one thread per unit up to 4096 CTAs per plane
    long long gx = (max_units + 255) / 256;
    if (gx > 4096) gx = 4096;
    const unsigned planes = (unsigned)n_cols + ((index_out || states) ? 1u : 0u);
    if (planes == 0) return B2RL_OK;
    k_rollout_seq_gather<<<dim3((unsigned)gx, planes), 256, 0, s>>>(a);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}
