// Internal declarations shared by the translation units of libb2rl.so.
// Not part of the ABI (see include/b2rl.h).
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "b2rl.h"

// ---- error plumbing --------------------------------------------------------
void b2rl_set_error(const char *fmt, ...);

#define B2RL_CUDA(call)                                                        \
    do {                                                                       \
        cudaError_t e__ = (call);                                              \
        if (e__ != cudaSuccess) {                                              \
            b2rl_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call,       \
                           cudaGetErrorString(e__));                           \
            return B2RL_ERR_CUDA;                                              \
        }                                                                      \
    } while (0)

#define B2RL_REQUIRE(cond, status, ...)                                        \
    do {                                                                       \
        if (!(cond)) {                                                         \
            b2rl_set_error(__VA_ARGS__);                                       \
            return (status);                                                   \
        }                                                                      \
    } while (0)

// pass a failing B2RL status of an internal call on to the caller
#define TRY(x)                                                                 \
    do {                                                                       \
        int rc__ = (x);                                                        \
        if (rc__ != B2RL_OK) return rc__;                                      \
    } while (0)

// ---- device-side scalar state ----------------------------------------------
// Lives in HBM so that kernels never need host-supplied counters; the host
// keeps mirrors for the (deterministic) host-driven paths.
struct B2rlDevState {
    long long napp;      // absolute append counter
    long long npop;      // absolute pop counter
    double max_priority; // collections/prioritized.py:32,114
    double last_total;   // sum-tree root read before the last sample's draws
    double last_min;     // min-tree root at the last sample
    int last_n;          // size of the last sample
    int pad;
};

static constexpr int B2RL_U_RING = 8;

// ---- the handle --------------------------------------------------------------
struct b2rl_replay {
    b2rl_replay_config cfg;
    int64_t P;      // pow2 >= capacity
    int64_t nslots; // 2P leaf / record slots, slot = abs_index mod 2P
    int levels;     // log2(nslots): leaves live at heap level `levels`

    // HBM
    uint8_t *parts;        // [part_capacity][part_bytes]
    int32_t *state_parts;  // [nslots][stack]
    int32_t *next_parts;   // [nslots][stack]
    uint8_t *action;       // [nslots][action_bytes]
    double *rewards;       // [nslots][n_step]
    uint8_t *len;          // [nslots]
    uint8_t *terminal;     // [nslots]
    double *sum;           // heap [2*nslots], node 1 = top, leaves at [nslots, 2*nslots)
    double *mn;            // same layout, empty = +inf
    B2rlDevState *st;
    int32_t *last_slots;   // [max_batch] slots drawn by the last sample
    double *last_prio;     // [max_batch] their priorities (as found)
    double *new_prio;      // [max_batch] scratch for update
    int32_t *winner;       // [nslots] scratch for duplicate resolution (-1 idle)
    int64_t device_bytes;

    // host mirrors
    int64_t napp, npop;
    int64_t part_head; // next part sequence number
    bool wait_priority;
    int last_n;

    // ring of pinned slots for host-drawn uniforms (b2rl_upload_u); fused replay step
    // (step.cu): cross-CTA "draws ready" counter, launch sequence number; deferred write-back
    unsigned long long *ready_dev;
    unsigned long long *times_dev; // [8 + 256] %globaltimer stamps of the last fused launch
    int last_step_grid;
    uint64_t step_seq;
    double *u_ring_pin, *u_ring_dev;
    cudaEvent_t u_ev[B2RL_U_RING];
    uint64_t u_head;
    int sm_count;
    bool pending;          // TD errors of the last sample registered, trees not yet updated
    const void *pend_err;
    int pend_is_f64, pend_n;
    double pend_alpha, pend_eps, pend_emin, pend_emax;

    // staging (host pinned + device), guarded by an event
    uint8_t *pin;
    uint8_t *stage;
    size_t stage_bytes;
    cudaEvent_t stage_ev;
    bool stage_busy;
};

static inline int b2rl_ilog2(int64_t x)
{
    int l = 0;
    while ((int64_t(1) << l) < x) l++;
    return l;
}

// Make sure the staging buffers hold `bytes`; waits for the previous user.
int b2rl_stage_acquire(b2rl_replay *h, size_t bytes);
int b2rl_stage_release(b2rl_replay *h, cudaStream_t s);

// "Last CTA finishes the reduction" elections use one of B2RL_N_TICKETS device
// counters per LAUNCH (rotating ticket, self-resetting atomicInc), so launches
// that overlap on different streams never share a counter.
static constexpr unsigned B2RL_N_TICKETS = 256;
unsigned b2rl_next_ticket();

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (kernel, device)
template <auto KERNEL>
static cudaError_t b2rl_allow_smem(size_t bytes)
{
    static bool done[64];
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev < 0 || dev >= 64 || !done[dev]) {
        e = cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
        if (e != cudaSuccess) return e;
        if (dev >= 0 && dev < 64) done[dev] = true;
    }
    return cudaSuccess;
}

// Sampler arguments of a draw of n uniforms `u` (device) from the handle's trees: the
// shared-memory split (T, D), the handle's slot / priority outputs, the optional user
// outputs and the exact sampler's test hooks (env B2RL_V6_SLOW_EVERY / B2RL_V6_EPS_SCALE);
// no weights, no publication to other CTAs (sampler.cu, SampleArgs: tree_dev.cuh).
struct SampleArgs;
SampleArgs b2rl_sample_args(const b2rl_replay *h, const double *u, int n, int64_t *index_out,
                            double *prio_user);

// Preconditions of a sample of n draws in `mode` (b2rl_per_sample, b2rl_replay_step): the
// trees exist, 1 <= n <= max_batch and the live count, no sample awaits its priorities
// (collections/prioritized.py:98), and every host uniform u_host[i] lies in [0, 1) (u_host
// null: the uniforms are on the device).  `fn` names the caller in the messages.
int b2rl_check_sample(const b2rl_replay *h, int n, int mode, const double *u_host, const char *fn);

// Host uniforms u[0..n) to the device through a ring of B2RL_U_RING pinned slots, allocated on
// first use; *u_dev receives the device copy, valid for the next B2RL_U_RING uploads.
int b2rl_upload_u(b2rl_replay *h, const double *u, int n, cudaStream_t s, const double **u_dev);

// Write-back arguments for the n priorities of the last sample: in h->new_prio, or computed
// there from the TD errors `err` (priority_from_errors) when err is not null.
struct UpdateArgs;
UpdateArgs b2rl_update_args(const b2rl_replay *h, int n, const void *err, int err_is_f64,
                            double alpha, double eps, double emin, double emax);

// Apply a write-back registered with b2rl_per_defer_errors (no-op if none).
int b2rl_flush_pending(b2rl_replay *h, cudaStream_t s);

// Ancestors of up to 4 ring-slot ranges (<= 512 leaves in total) recomputed by the
// multi-CTA path kernel, then napp += bump_n and eviction down to capacity.
int b2rl_launch_repair_multi(b2rl_replay *h, int nranges, const long long *first_slot,
                             const long long *count, long long bump_n, cudaStream_t s);

// ---- gather: one piece of one observation part --------------------------------
// A part is cut in GATHER_SPLIT pieces so that the CTAs of the gathers are short
// (~17 KB of traffic) and the last, partially filled wave costs little.
#define GATHER_SPLIT 2

// Ring slot of the record with logical index i (0 = oldest live record).
__device__ __forceinline__ long long b2rl_logical_slot(const B2rlDevState *st, long long nslots,
                                                       long long i)
{
    return (st->npop + i) & (nslots - 1);
}

// Copies piece `piece` of the part `src` to output part `dst_part` (counted in
// parts from `out`), converting it to f32 in U8_TO_F32 mode.  Every thread of the
// 256-thread CTA turns one 32-bit word (4 pixels) into one 128-bit store, so both
// the loads and the stores are fully coalesced (k_gather, k_seq_gather).
__device__ __forceinline__ void b2rl_gather_part_piece(const uint8_t *src, uint8_t *out,
                                                       size_t dst_part, int part_bytes,
                                                       int piece, int obs_mode, float sc)
{
    if (obs_mode == B2RL_OBS_U8_TO_F32) {
        const int words = part_bytes / 4;
        const int per = (words + GATHER_SPLIT - 1) / GATHER_SPLIT;
        const int w0 = piece * per;
        const int w1 = min(words, w0 + per);
        const uint32_t *s4 = reinterpret_cast<const uint32_t *>(src);
        float4 *d4 = reinterpret_cast<float4 *>(out) + dst_part * words;
        constexpr int U = 4; // loads in flight per thread
        for (int base = w0 + threadIdx.x; base < w1; base += U * 256) {
            uint32_t v[U];
#pragma unroll
            for (int i = 0; i < U; i++)
                if (base + i * 256 < w1) v[i] = __ldg(s4 + base + i * 256);
#pragma unroll
            for (int i = 0; i < U; i++) {
                if (base + i * 256 >= w1) continue;
                float4 f;
                f.x = (float)(v[i] & 0xffu) * sc;
                f.y = (float)((v[i] >> 8) & 0xffu) * sc;
                f.z = (float)((v[i] >> 16) & 0xffu) * sc;
                f.w = (float)(v[i] >> 24) * sc;
                __stcs(d4 + base + i * 256, f);
            }
        }
    } else {
        const int vecs = part_bytes / 16;
        const int per = (vecs + GATHER_SPLIT - 1) / GATHER_SPLIT;
        const int w0 = piece * per;
        const int w1 = min(vecs, w0 + per);
        const uint4 *s16 = reinterpret_cast<const uint4 *>(src);
        uint4 *d16 = reinterpret_cast<uint4 *>(out) + dst_part * vecs;
        for (int w = w0 + threadIdx.x; w < w1; w += 256) __stcs(d16 + w, __ldg(s16 + w));
    }
}

// The records, outputs and options of a minibatch gather of n experiences, shared by
// k_gather (gather.cu) and the gather CTAs of the fused step (step.cu).
struct GatherArgs {
    const uint8_t *parts;
    const int32_t *state_parts, *next_parts;
    const uint8_t *action;
    const double *rewards;
    const uint8_t *len, *terminal;
    const int32_t *slots;      // slots of the last sample
    double gamma_pow[9];       // gamma**i, i <= n_step (<= 8), passed by value
    int n, stack, part_bytes, n_step, action_bytes;
    int obs_mode;
    float obs_scale;
    uint8_t *o_side[2]; // state, next_state (either may be null)
    uint8_t *o_action;
    float *o_reward, *o_terminal, *o_discount;
    double *o_step_rewards;
    uint8_t *o_len;
};

GatherArgs b2rl_gather_args(const b2rl_replay *h, int n, const double *gamma_pow_host,
                            int obs_mode, float obs_scale, const b2rl_batch_out *out);

// Scalars of experience k, stored at ring slot `slot`: n-step reward, discount, terminal,
// len, step rewards, action (pfrl/replay_buffer.py:183-206).
__device__ __forceinline__ void b2rl_gather_scalars(const GatherArgs &g, int k, long long slot)
{
    const int len = g.len[slot];
    if (g.o_reward) {
        // sum((gamma**i) * r_i) evaluated like CPython's float sum():
        // Neumaier-compensated accumulation (replay_buffer.py:183-190); the
        // compensation is added only when it is finite, so an infinite or
        // overflowed sum stays +-inf instead of becoming NaN (CPython also skips
        // c == 0, which changes nothing here: s starts at +0.0, never becomes -0.0)
        double s = 0.0, c = 0.0;
        for (int i = 0; i < len; i++) {
            const double x = __dmul_rn(g.gamma_pow[i], g.rewards[slot * g.n_step + i]);
            const double t = __dadd_rn(s, x);
            if (fabs(s) >= fabs(x))
                c = __dadd_rn(c, __dadd_rn(__dsub_rn(s, t), x));
            else
                c = __dadd_rn(c, __dadd_rn(__dsub_rn(x, t), s));
            s = t;
        }
        g.o_reward[k] = (float)(fabs(c) < INFINITY ? __dadd_rn(s, c) : s);
    }
    if (g.o_terminal) g.o_terminal[k] = g.terminal[slot] ? 1.0f : 0.0f;
    if (g.o_discount) g.o_discount[k] = (float)g.gamma_pow[len]; // gamma ** len(elem), :203
    if (g.o_len) g.o_len[k] = (uint8_t)len;
    if (g.o_step_rewards)
        for (int i = 0; i < g.n_step; i++)
            g.o_step_rewards[(size_t)k * g.n_step + i] =
                i < len ? g.rewards[slot * g.n_step + i] : 0.0;
    if (g.o_action) {
        const uint8_t *src = g.action + slot * g.action_bytes;
        uint8_t *dst = g.o_action + (size_t)k * g.action_bytes;
        for (int i = 0; i < g.action_bytes; i++) dst[i] = src[i];
    }
}

// ---- packed sequences (k_seq_gather, k_rollout_seq_gather) --------------------
// Step t of packed row `row`: the largest t in [0, Lmax) with row0(t) <= row, where
// row0(t) = sum_b min(len[b], t) is the packed row of step t of sequence 0
// (row0(0) = 0, row0(Lmax) = N).  Sequence b = row - row0(t).
template <class Row0>
__device__ __forceinline__ int b2rl_packed_step(int row, int Lmax, Row0 row0)
{
    int lo = 0, hi = Lmax;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (row0(mid) <= row) lo = mid;
        else hi = mid;
    }
    return lo;
}

// The recurrent states of each sequence's first record, written by the threads
// gid, gid + nthreads, ... of the grid: element e of [side][b][float f of the ring row]
// is float f of side `side` of ring row ring_row(b) (0.0 for a stored None), written
// into the leaf holding f, laid out [d0][B][inner] (concatenate_recurrent_states).
// Floats outside every leaf and leaves without an output for that side are skipped.
// `a` is the kernel's argument block (fields B and rs); reading B from it, not from a
// copy, keeps k_seq_gather's code as it was before the helper existed.
template <class Args, class RingRow>
__device__ __forceinline__ void b2rl_seq_states_write(const Args &a, long long gid,
                                                      long long nthreads, RingRow ring_row)
{
    const b2rl_seq_states &rs = a.rs;
    const int D = rs.row_floats;
    const long long total = 2LL * a.B * D;
    for (long long e = gid; e < total; e += nthreads) {
        const int side = (int)(e / ((long long)a.B * D));
        const int rem = (int)(e % ((long long)a.B * D));
        const int b = rem / D, f = rem % D;
        int leaf = -1;
        for (int i = 0; i < rs.n_leaves; i++)
            if (f >= rs.offset[i] && f < rs.offset[i] + rs.d0[i] * rs.inner[i]) leaf = i;
        if (leaf < 0) continue;
        float *out = side ? rs.out_next_state[leaf] : rs.out_state[leaf];
        if (!out) continue;
        const long long r = ring_row(b);
        const float v = rs.present[r * 2 + side] ? rs.ring[(r * 2 + side) * D + f] : 0.0f;
        const int g = f - rs.offset[leaf];
        const int inner = rs.inner[leaf];
        out[((size_t)(g / inner) * a.B + b) * inner + g % inner] = v;
    }
}

// Kernel launchers implemented in the other TUs.
// Recompute the ancestors of up to 4 contiguous leaf-node ranges [lo, hi]
// (inclusive heap indices at the leaf level; modified in place), then add
// bump_n to the device append counter and evict down to capacity.
int b2rl_launch_tree_fix(b2rl_replay *h, int nranges, long long *lo, long long *hi,
                         long long bump_n, cudaStream_t s);
