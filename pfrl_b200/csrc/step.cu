// step.cu -- the fused replay step: ONE persistent launch per minibatch.
//
//   [write-back of the previous sample's TD errors]   CTA 0, all warps
//   prioritized sample (exact or parallel) + IS weights  CTA 0
//   gather of state / next_state / scalars             CTAs 1..G, consuming
//                                                      the draws 32 at a time
//                                                      while CTA 0 is still
//                                                      drawing
//
// Replaces, in one launch, the reference's (pure Python)
//   pfrl/replay_buffers/prioritized.py:117-126   sample / update_errors
//   pfrl/collections/prioritized.py:56-116       _sample_indices_and_probabilities,
//                                                sample, set_last_priority
//   pfrl/replay_buffer.py:157-212                batch_experiences
//   pfrl/utils/batch_states.py:18-36             batch_states + H2D copy
// Ordering: the reference runs sample_k -> forward -> update_errors_k ->
// (appends) -> sample_k+1 (pfrl/agents/dqn.py:338-364, SURVEY 3.1).  The
// write-back folded into the head of launch k+1 is the one of sample k; an
// append in between flushes it first (b2rl_flush_pending), so max_priority and
// the trees are always what the reference would see.
//
// Gather CTAs stream whole parts (frames) global -> shared with cp.async.bulk
// (SASS UBLKCP) through an 8-stage mbarrier ring -- the loads cost no thread
// instructions and no registers -- and convert u8 -> f32 out of shared memory
// into 512-byte-per-warp coalesced .cs stores.
#include <math.h>
#include <stdlib.h>

#include "tree_dev.cuh"

#define TRY(x)                                                                 \
    do {                                                                       \
        int rc__ = (x);                                                        \
        if (rc__ != B2RL_OK) return rc__;                                      \
    } while (0)

static constexpr int GS = 8;            // stages of the part ring in shared memory
static constexpr int PIECE_MAX = 8192;  // parts larger than this are cut in pieces
static constexpr int STEP_THREADS = 512;

struct StepGather {
    const uint8_t *parts;
    const int32_t *state_parts, *next_parts;
    const uint8_t *action;
    const double *rewards;
    const uint8_t *len, *terminal;
    const int32_t *slots; // slots of the sample drawn by CTA 0 of this launch
    double gamma_pow[9];
    int n, stack, part_bytes, n_step, action_bytes;
    int obs_mode;
    float obs_scale;
    int pieces, piece_bytes, stage_stride;
    uint8_t *o_side[2]; // state, next_state (either may be null)
    uint8_t *o_action;
    float *o_reward, *o_terminal, *o_discount;
    double *o_step_rewards;
    uint8_t *o_len;
    const unsigned long long *ready;
    unsigned long long seq_base;
    int poll_ns;
};

struct StepArgs {
    SampleArgs s;
    UpdateArgs u;
    int upd_n; // > 0: write back the previous sample first
    unsigned long long *upd_sync; // [0] done stamp, [1] arrival counter
    // %globaltimer stamps of this launch (b2rl_step_times): [0] CTA 0 entry, [1] write-back
    // complete, [2] all draws published, [8 + c] exit of CTA c
    unsigned long long *times;
    StepGather g;
};

__device__ __forceinline__ unsigned long long global_ns()
{
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

extern __shared__ __align__(128) unsigned char smem_raw[];

// scalars of one experience: n-step reward, discount, terminal, action
// (pfrl/replay_buffer.py:183-206)
__device__ __forceinline__ void gather_scalars(const StepGather &g, int k, long long slot)
{
    const int len = g.len[slot];
    if (g.o_reward) {
        // sum((gamma**i) * r_i) evaluated like CPython's float sum():
        // Neumaier-compensated accumulation (replay_buffer.py:183-190)
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
        g.o_reward[k] = (float)__dadd_rn(s, c);
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

struct Unit {
    int k, sidx, part, piece;
};

__device__ __forceinline__ Unit decode_unit(const StepGather &g, int nsides, long long q)
{
    Unit u;
    u.piece = (int)(q % g.pieces);
    long long t = q / g.pieces;
    u.part = (int)(t % g.stack);
    t /= g.stack;
    u.sidx = (int)(t % nsides);
    u.k = (int)(t / nsides);
    return u;
}

// One gather CTA.  w = worker index in [0, G).
__device__ __forceinline__ void gather_worker(const StepGather &g, unsigned char *smem, int w, int G)
{
    const int tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    const int nwarps = blockDim.x >> 5;
    uint8_t *stage = smem;
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + (size_t)GS * g.stage_stride);
    uint64_t *empty = full + GS;
    int side_of[2];
    int nsides = 0;
    if (g.o_side[0]) side_of[nsides++] = 0;
    if (g.o_side[1]) side_of[nsides++] = 1;

    if (nsides == 0) {
        // scalars only: one thread per experience, strided over the workers
        for (long long k = (long long)w * blockDim.x + tid; k < g.n; k += (long long)G * blockDim.x) {
            while (ld_acquire_gpu(g.ready) <= g.seq_base + (unsigned long long)k)
                __nanosleep(g.poll_ns);
            gather_scalars(g, (int)k, __ldcg(g.slots + k));
        }
        return;
    }

    if (tid == 0) {
        for (int s = 0; s < GS; s++) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], nwarps - 1);
        }
        mbar_fence_init();
    }
    __syncthreads();

    const int upe = nsides * g.stack * g.pieces; // units per experience
    const long long total = (long long)g.n * upe;
    const int my_units = total > w ? (int)((total - w + G - 1) / G) : 0;

    if (warp == 0) {
        // ---------------- lookups + bulk-copy producer ----------------
        int base = 0, next = 0;
        bool done_l = false;
        unsigned long long src_l = 0;
        unsigned bytes_l = 0;
        unsigned long long r = 0;
        while (next < my_units) {
            const int i = base + lane;
            bool progressed = false;
            if (!done_l && i < my_units) {
                const Unit u = decode_unit(g, nsides, w + (long long)i * G);
                const unsigned long long need = g.seq_base + (unsigned long long)u.k;
                if (r <= need) r = ld_acquire_gpu(g.ready);
                if (r > need) {
                    const long long slot = __ldcg(g.slots + u.k);
                    const int side = side_of[u.sidx];
                    const int32_t ps =
                        (side ? g.next_parts : g.state_parts)[slot * g.stack + u.part];
                    const int off = u.piece * g.piece_bytes;
                    src_l = (unsigned long long)(g.parts + (size_t)ps * g.part_bytes + off);
                    bytes_l = (unsigned)min(g.piece_bytes, g.part_bytes - off);
                    if (u.sidx == 0 && u.part == 0 && u.piece == 0) gather_scalars(g, u.k, slot);
                    done_l = true;
                }
            }
            const unsigned mask = __ballot_sync(0xffffffffu, done_l);
            while (next < my_units && next < base + 32 && ((mask >> (next - base)) & 1u)) {
                const unsigned long long src = __shfl_sync(0xffffffffu, src_l, next - base);
                const unsigned bytes = __shfl_sync(0xffffffffu, bytes_l, next - base);
                if (lane == 0) {
                    const int s = next % GS;
                    if (next >= GS) mbar_wait(&empty[s], ((next / GS) - 1) & 1);
                    mbar_expect_tx(&full[s], bytes);
                    bulk_g2s(stage + (size_t)s * g.stage_stride, (const void *)src, bytes, &full[s]);
                }
                next++;
                progressed = true;
            }
            __syncwarp();
            if (next == base + 32) {
                base += 32;
                done_l = false;
            } else if (!progressed) {
                __nanosleep(g.poll_ns);
            }
        }
    } else {
        // ------------------------- consumers ---------------------------
        const int ct = tid - 32, nct = blockDim.x - 32;
        for (int i = 0; i < my_units; i++) {
            const int s = i % GS;
            const Unit u = decode_unit(g, nsides, w + (long long)i * G);
            const int off = u.piece * g.piece_bytes;
            const int bytes = min(g.piece_bytes, g.part_bytes - off);
            uint8_t *out = g.o_side[side_of[u.sidx]];
            const size_t obyte = ((size_t)u.k * g.stack + u.part) * g.part_bytes + off;
            const uint8_t *src = stage + (size_t)s * g.stage_stride;
            mbar_wait(&full[s], (i / GS) & 1);
            if (g.obs_mode == B2RL_OBS_U8_TO_F32) {
                const int words = bytes >> 2;
                const uint32_t *s4 = reinterpret_cast<const uint32_t *>(src);
                float4 *d4 = reinterpret_cast<float4 *>(out) + obyte / 4; // one f32 per byte
                const float sc = g.obs_scale;
                constexpr int U = 4;
                for (int b = ct; b < words; b += U * nct) {
                    uint32_t v[U];
#pragma unroll
                    for (int j = 0; j < U; j++)
                        if (b + j * nct < words) v[j] = s4[b + j * nct];
#pragma unroll
                    for (int j = 0; j < U; j++) {
                        if (b + j * nct >= words) continue;
                        float4 f;
                        f.x = (float)(v[j] & 0xffu) * sc;
                        f.y = (float)((v[j] >> 8) & 0xffu) * sc;
                        f.z = (float)((v[j] >> 16) & 0xffu) * sc;
                        f.w = (float)(v[j] >> 24) * sc;
                        __stcs(d4 + b + j * nct, f);
                    }
                }
            } else {
                const int vecs = bytes >> 4;
                const uint4 *s16 = reinterpret_cast<const uint4 *>(src);
                uint4 *d16 = reinterpret_cast<uint4 *>(out + obyte);
                for (int b = ct; b < vecs; b += nct) __stcs(d16 + b, s16[b]);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[s]);
        }
    }
}

// MODE: the SamplerKind of choose_sampler (tree_dev.cuh), D its template depth
template <int D, int MODE>
__global__ void __launch_bounds__(STEP_THREADS, 1) k_replay_step(const __grid_constant__ StepArgs a)
{
    if (blockIdx.x == 0 && threadIdx.x == 0) a.times[0] = global_ns();
    if (a.upd_n > 0) {
        // write-back of the previous sample: every CTA takes the subtrees it owns; the
        // sampler (CTA 0) waits for the one that finishes the top of the tree
        tree_update_multi(a.u, smem_raw, a.upd_sync, a.s.seq_base);
        if (blockIdx.x == 0) {
            if (threadIdx.x == 0)
                while (ld_acquire_gpu(a.upd_sync) != a.s.seq_base) __nanosleep(100);
            __syncthreads();
        }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) a.times[1] = global_ns();
    if (blockIdx.x == 0) {
        if constexpr (MODE == SAMPLER_V5)
            exact_deep<D>(a.s, reinterpret_cast<double *>(smem_raw));
        else if constexpr (MODE == SAMPLER_V6)
            exact_deep_v6<D>(a.s, reinterpret_cast<double *>(smem_raw));
        else if constexpr (MODE == SAMPLER_SMALL)
            exact_small(a.s, reinterpret_cast<double *>(smem_raw));
        else
            sample_parallel(a.s, reinterpret_cast<double *>(smem_raw));
        if (threadIdx.x == 0) a.times[2] = global_ns();
    } else {
        gather_worker(a.g, smem_raw, blockIdx.x - 1, gridDim.x - 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) a.times[8 + blockIdx.x] = global_ns();
}

template <int D, int MODE>
static cudaError_t launch_step_as(const StepArgs &a, int grid, size_t smem, cudaStream_t s)
{
    const cudaError_t e = b2rl_allow_smem<k_replay_step<D, MODE>>(227 * 1024);
    if (e != cudaSuccess) return e;
    k_replay_step<D, MODE><<<grid, STEP_THREADS, smem, s>>>(a);
    return cudaGetLastError();
}

static cudaError_t launch_step(const StepArgs &a, int mode, int grid, size_t smem_other,
                               cudaStream_t s)
{
    auto mx = [](size_t x, size_t y) { return x > y ? x : y; };
    const SamplerChoice c = choose_sampler(mode, a.s.levels, a.s.n);
    switch (c.kind) {
    case SAMPLER_PARALLEL:
        return launch_step_as<0, SAMPLER_PARALLEL>(a, grid, mx(smem_other, 1024), s);
    case SAMPLER_SMALL: {
        const size_t sm = sizeof(double) * ((size_t(1) << a.s.T) + 2);
        return launch_step_as<0, SAMPLER_SMALL>(a, grid, mx(smem_other, sm), s);
    }
    case SAMPLER_V6:
        return with_depth<5, 9>(c.D, [&](auto d) {
            constexpr int D = decltype(d)::value;
            return launch_step_as<D, SAMPLER_V6>(a, grid, mx(smem_other, exact_v6_smem_bytes<D>()), s);
        });
    default:
        return with_depth<1, 10>(c.D, [&](auto d) {
            constexpr int D = decltype(d)::value;
            return launch_step_as<D, SAMPLER_V5>(a, grid, mx(smem_other, exact_deep_smem_bytes<D>()), s);
        });
    }
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
static int step_resources(b2rl_replay *h)
{
    if (h->u_ring_dev) return B2RL_OK;
    const size_t ring = (size_t)B2RL_U_RING * h->cfg.max_batch * sizeof(double);
    B2RL_CUDA(cudaMallocHost((void **)&h->u_ring_pin, ring));
    B2RL_CUDA(cudaMalloc((void **)&h->u_ring_dev, ring));
    for (int i = 0; i < B2RL_U_RING; i++)
        B2RL_CUDA(cudaEventCreateWithFlags(&h->u_ev[i], cudaEventDisableTiming));
    int sm = 0;
    B2RL_CUDA(cudaDeviceGetAttribute(&sm, cudaDevAttrMultiProcessorCount, h->cfg.device));
    h->sm_count = sm;
    h->device_bytes += (int64_t)ring;
    return B2RL_OK;
}

extern "C" int b2rl_replay_step(b2rl_replay *h, const b2rl_step_args *p, void *stream)
{
    B2RL_REQUIRE(h && p, B2RL_ERR_INVALID, "null argument");
    B2RL_REQUIRE(h->cfg.prioritized, B2RL_ERR_INVALID, "buffer has no priority trees");
    const int n = p->n;
    B2RL_REQUIRE(n > 0 && n <= h->cfg.max_batch, B2RL_ERR_RANGE,
                 "step: n=%d out of 1..max_batch=%d", n, h->cfg.max_batch);
    B2RL_REQUIRE(n <= h->napp - h->npop, B2RL_ERR_RANGE,
                 "step: n=%d exceeds the %lld stored experiences", n,
                 (long long)(h->napp - h->npop));
    B2RL_REQUIRE(!h->wait_priority, B2RL_ERR_PROTOCOL,
                 "step: the previous sample's priorities were not set "
                 "(collections/prioritized.py:98)");
    B2RL_REQUIRE(p->mode == B2RL_SAMPLE_EXACT || p->mode == B2RL_SAMPLE_PARALLEL,
                 B2RL_ERR_INVALID, "unknown sample mode %d", p->mode);
    B2RL_REQUIRE(p->u && p->gamma_pow_host, B2RL_ERR_INVALID, "step: null u / gamma_pow");
    B2RL_REQUIRE(p->norm >= 0 && p->norm <= 2, B2RL_ERR_INVALID, "unknown normalisation %d",
                 p->norm);
    B2RL_REQUIRE(p->obs_mode == B2RL_OBS_RAW || p->obs_mode == B2RL_OBS_U8_TO_F32,
                 B2RL_ERR_INVALID, "unknown obs_mode %d", p->obs_mode);
    cudaStream_t s = (cudaStream_t)stream;
    B2RL_CUDA(cudaSetDevice(h->cfg.device));
    TRY(step_resources(h));
    const b2rl_replay_config &c = h->cfg;

    // a deferred write-back too large for the in-launch path goes first, alone
    if (h->pending && h->pend_n > UPD_MAX) TRY(b2rl_flush_pending(h, s));

    // uniforms: device pointer, or host values through a ring of pinned slots
    const double *u_dev = p->u;
    if (!p->u_on_device) {
        for (int i = 0; i < n; i++)
            B2RL_REQUIRE(p->u[i] >= 0.0 && p->u[i] < 1.0, B2RL_ERR_INVALID,
                         "step: u[%d]=%g not in [0,1)", i, p->u[i]);
        const int slot = (int)(h->u_head % B2RL_U_RING);
        if (h->u_head >= B2RL_U_RING) B2RL_CUDA(cudaEventSynchronize(h->u_ev[slot]));
        double *pin = h->u_ring_pin + (size_t)slot * c.max_batch;
        double *dev = h->u_ring_dev + (size_t)slot * c.max_batch;
        memcpy(pin, p->u, (size_t)n * 8);
        B2RL_CUDA(cudaMemcpyAsync(dev, pin, (size_t)n * 8, cudaMemcpyHostToDevice, s));
        B2RL_CUDA(cudaEventRecord(h->u_ev[slot], s));
        h->u_head++;
        u_dev = dev;
    }

    StepArgs a;
    memset(&a, 0, sizeof(a));
    h->step_seq++;
    const unsigned long long seq_base = (unsigned long long)h->step_seq << 32;
    // ---- sampler
    a.s = b2rl_sample_args(h, u_dev, n, p->index_dev, p->priority_dev);
    a.s.weight = p->weight_dev;
    a.s.prob = p->prob_dev;
    a.s.beta = p->beta;
    a.s.norm = p->norm;
    a.s.ready = h->ready_dev;
    a.s.seq_base = seq_base;
    {
        static int want = -1; // B2RL_V6_CYCLES=1: clock64 sums per pipeline segment of the sampler
        if (want < 0) {
            const char *e = getenv("B2RL_V6_CYCLES");
            want = (e && e[0] == '1') ? 1 : 0;
        }
        a.s.dbg_cycles = want ? (long long *)(h->times_dev + 8 + 256) : nullptr;
    }
    // ---- deferred write-back of the previous sample
    a.upd_n = 0;
    if (h->pending) {
        a.u.sum = h->sum;
        a.u.mn = h->mn;
        a.u.st = h->st;
        a.u.slots = h->last_slots;
        a.u.new_prio = h->new_prio;
        a.u.err = h->pend_err;
        a.u.err_is_f64 = h->pend_is_f64;
        a.u.alpha = h->pend_alpha;
        a.u.eps = h->pend_eps;
        a.u.emin = h->pend_emin;
        a.u.emax = h->pend_emax;
        a.u.winner = h->winner;
        a.u.n = h->pend_n;
        a.u.levels = h->levels;
        a.u.nslots = h->nslots;
        a.upd_n = h->pend_n;
        a.upd_sync = h->ready_dev + 1;
        a.u.stamps = h->times_dev + 3; // [3..7]: phases of the write-back
    }
    a.times = h->times_dev;
    // ---- gather
    StepGather &g = a.g;
    g.parts = h->parts;
    g.state_parts = h->state_parts;
    g.next_parts = h->next_parts;
    g.action = h->action;
    g.rewards = h->rewards;
    g.len = h->len;
    g.terminal = h->terminal;
    g.slots = h->last_slots;
    for (int i = 0; i <= c.n_step; i++) g.gamma_pow[i] = p->gamma_pow_host[i];
    g.n = n;
    g.stack = c.stack;
    g.part_bytes = c.part_bytes;
    g.n_step = c.n_step;
    g.action_bytes = c.action_bytes;
    g.obs_mode = p->obs_mode;
    g.obs_scale = p->obs_scale;
    g.pieces = (c.part_bytes + PIECE_MAX - 1) / PIECE_MAX;
    g.piece_bytes = (((c.part_bytes + g.pieces - 1) / g.pieces) + 15) & ~15;
    g.stage_stride = (g.piece_bytes + 127) & ~127;
    g.o_side[0] = (uint8_t *)p->out.state;
    g.o_side[1] = (uint8_t *)p->out.next_state;
    g.o_action = (uint8_t *)p->out.action;
    g.o_reward = p->out.reward;
    g.o_terminal = p->out.terminal;
    g.o_discount = p->out.discount;
    g.o_step_rewards = p->out.step_rewards;
    g.o_len = p->out.len;
    g.ready = h->ready_dev;
    g.seq_base = seq_base;
    g.poll_ns = p->mode == B2RL_SAMPLE_EXACT ? 400 : 100;

    const int nsides = (g.o_side[0] ? 1 : 0) + (g.o_side[1] ? 1 : 0);
    long long units = nsides ? (long long)n * nsides * c.stack * g.pieces : (n + STEP_THREADS - 1) / STEP_THREADS;
    int grid = h->sm_count;
    if (units + 1 < grid) grid = (int)units + 1;
    if (grid < 2) grid = 2;
    size_t smem = (size_t)GS * g.stage_stride + 2 * GS * sizeof(uint64_t);
    if (a.upd_n > 0) {
        const size_t us = update_multi_smem_bytes(h->levels);
        if (us > smem) smem = us;
    }
    h->last_step_grid = grid;
    B2RL_CUDA(launch_step(a, p->mode, grid, smem, s));
    h->pending = false;
    h->wait_priority = true;
    h->last_n = n;
    h->last_mode = p->mode;
    return B2RL_OK;
}

// Phase durations of the LAST fused step launch, from %globaltimer stamps the kernel
// leaves behind (synchronises the stream): out_ns[0] write-back, [1] sampling (first
// draw to last draw published), [2] gather tail (last draw published -> last CTA exits),
// [3] whole launch (CTA 0 entry -> last CTA exits).
extern "C" int b2rl_step_times(b2rl_replay *h, uint64_t *out_ns, void *stream)
{
    B2RL_REQUIRE(h && out_ns, B2RL_ERR_INVALID, "null argument");
    B2RL_REQUIRE(h->last_step_grid > 0, B2RL_ERR_PROTOCOL, "no fused step was launched yet");
    cudaStream_t s = (cudaStream_t)stream;
    B2RL_CUDA(cudaSetDevice(h->cfg.device));
    unsigned long long t[8 + 256];
    const int grid = h->last_step_grid < 248 ? h->last_step_grid : 248;
    B2RL_CUDA(cudaMemcpyAsync(t, h->times_dev, sizeof(unsigned long long) * (8 + grid),
                              cudaMemcpyDeviceToHost, s));
    B2RL_CUDA(cudaStreamSynchronize(s));
    unsigned long long last = 0;
    for (int c = 0; c < grid; c++)
        if (t[8 + c] > last) last = t[8 + c];
    out_ns[0] = t[1] - t[0];
    out_ns[1] = t[2] - t[1];
    out_ns[2] = last > t[2] ? last - t[2] : 0;
    out_ns[3] = last - t[0];

    // [4, 36): clock64 sums of the exact sampler's pipeline segments (B2RL_V6_CYCLES=1)
    B2RL_CUDA(cudaMemcpyAsync(out_ns + 4, h->times_dev + 8 + 256, sizeof(uint64_t) * 32,
                              cudaMemcpyDeviceToHost, s));
    B2RL_CUDA(cudaStreamSynchronize(s));
    // [31, 36): phases of the multi-CTA write-back, ns since CTA 0's entry (UpdateArgs::stamps)
    for (int i = 0; i < 5; i++) out_ns[31 + i] = t[3 + i] > t[0] ? t[3 + i] - t[0] : 0;
    if (getenv("B2RL_WB_FINE")) { // dev: finer stamps of CTA 0's subtree phase
        unsigned long long f[3];
        B2RL_CUDA(cudaMemcpy(f, h->times_dev + 200, sizeof f, cudaMemcpyDeviceToHost));
        for (int i = 0; i < 3; i++) out_ns[28 + i] = f[i] > t[0] ? f[i] - t[0] : 0;
    }
    return B2RL_OK;
}
