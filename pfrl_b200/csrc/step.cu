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

static constexpr int GS = 8;            // stages of the part ring in shared memory
static constexpr int PIECE_MAX = 8192;  // parts larger than this are cut in pieces
static constexpr int STEP_THREADS = 512;

struct StepArgs {
    SampleArgs s;
    UpdateArgs u;
    int upd_n; // > 0: write back the previous sample first
    unsigned long long *upd_sync; // [0] done stamp, [1] arrival counter
    // %globaltimer stamps of this launch (b2rl_step_times): [0] CTA 0 entry, [1] write-back
    // complete, [2] all draws published, [8 + c] exit of CTA c
    unsigned long long *times;
    // gather CTAs: the draws come from a.s (slots) as a.s.ready releases them; parts are
    // copied in `pieces` pieces of piece_bytes through stages of stage_stride bytes
    GatherArgs g;
    int pieces, piece_bytes, stage_stride;
    int poll_ns;
};

__device__ __forceinline__ unsigned long long global_ns()
{
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

extern __shared__ __align__(128) unsigned char smem_raw[];

struct Unit {
    int k, sidx, part, piece;
};

__device__ __forceinline__ Unit decode_unit(const StepArgs &a, int nsides, long long q)
{
    Unit u;
    u.piece = (int)(q % a.pieces);
    long long t = q / a.pieces;
    u.part = (int)(t % a.g.stack);
    t /= a.g.stack;
    u.sidx = (int)(t % nsides);
    u.k = (int)(t / nsides);
    return u;
}

// One gather CTA.  w = worker index in [0, G).
__device__ __forceinline__ void gather_worker(const StepArgs &a, unsigned char *smem, int w, int G)
{
    const GatherArgs &g = a.g;
    const int tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    const int nwarps = blockDim.x >> 5;
    uint8_t *stage = smem;
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + (size_t)GS * a.stage_stride);
    uint64_t *empty = full + GS;
    int side_of[2];
    int nsides = 0;
    if (g.o_side[0]) side_of[nsides++] = 0;
    if (g.o_side[1]) side_of[nsides++] = 1;

    if (nsides == 0) {
        // scalars only: one thread per experience, strided over the workers
        for (long long k = (long long)w * blockDim.x + tid; k < g.n; k += (long long)G * blockDim.x) {
            while (ld_acquire_gpu(a.s.ready) <= a.s.seq_base + (unsigned long long)k)
                __nanosleep(a.poll_ns);
            b2rl_gather_scalars(g, (int)k, __ldcg(g.slots + k));
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

    const int upe = nsides * g.stack * a.pieces; // units per experience
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
                const Unit u = decode_unit(a, nsides, w + (long long)i * G);
                const unsigned long long need = a.s.seq_base + (unsigned long long)u.k;
                if (r <= need) r = ld_acquire_gpu(a.s.ready);
                if (r > need) {
                    const long long slot = __ldcg(g.slots + u.k);
                    const int side = side_of[u.sidx];
                    const int32_t ps =
                        (side ? g.next_parts : g.state_parts)[slot * g.stack + u.part];
                    const int off = u.piece * a.piece_bytes;
                    src_l = (unsigned long long)(g.parts + (size_t)ps * g.part_bytes + off);
                    bytes_l = (unsigned)min(a.piece_bytes, g.part_bytes - off);
                    if (u.sidx == 0 && u.part == 0 && u.piece == 0) b2rl_gather_scalars(g, u.k, slot);
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
                    bulk_g2s(stage + (size_t)s * a.stage_stride, (const void *)src, bytes, &full[s]);
                }
                next++;
                progressed = true;
            }
            __syncwarp();
            if (next == base + 32) {
                base += 32;
                done_l = false;
            } else if (!progressed) {
                __nanosleep(a.poll_ns);
            }
        }
    } else {
        // ------------------------- consumers ---------------------------
        const int ct = tid - 32, nct = blockDim.x - 32;
        for (int i = 0; i < my_units; i++) {
            const int s = i % GS;
            const Unit u = decode_unit(a, nsides, w + (long long)i * G);
            const int off = u.piece * a.piece_bytes;
            const int bytes = min(a.piece_bytes, g.part_bytes - off);
            uint8_t *out = g.o_side[side_of[u.sidx]];
            const size_t obyte = ((size_t)u.k * g.stack + u.part) * g.part_bytes + off;
            const uint8_t *src = stage + (size_t)s * a.stage_stride;
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
        gather_worker(a, smem_raw, blockIdx.x - 1, gridDim.x - 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) a.times[8 + blockIdx.x] = global_ns();
}

static cudaError_t launch_step(const StepArgs &a, int mode, int grid, size_t smem_other,
                               cudaStream_t s)
{
    const SamplerChoice c = choose_sampler(mode, a.s.levels, a.s.n);
    const size_t sm = sampler_smem_bytes(c, a.s);
    const size_t smem = sm > smem_other ? sm : smem_other;
    return with_sampler(c, [&](auto d, auto kind) {
        constexpr int D = decltype(d)::value, MODE = decltype(kind)::value;
        const cudaError_t e = b2rl_allow_smem<k_replay_step<D, MODE>>(227 * 1024);
        if (e != cudaSuccess) return e;
        k_replay_step<D, MODE><<<grid, STEP_THREADS, smem, s>>>(a);
        return cudaGetLastError();
    });
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
extern "C" int b2rl_replay_step(b2rl_replay *h, const b2rl_step_args *p, void *stream)
{
    B2RL_REQUIRE(h && p, B2RL_ERR_INVALID, "null argument");
    B2RL_REQUIRE(p->u && p->gamma_pow_host, B2RL_ERR_INVALID, "step: null u / gamma_pow");
    const int n = p->n;
    TRY(b2rl_check_sample(h, n, p->mode, p->u_on_device ? nullptr : p->u, "step"));
    B2RL_REQUIRE(p->norm >= 0 && p->norm <= 2, B2RL_ERR_INVALID, "unknown normalisation %d",
                 p->norm);
    B2RL_REQUIRE(p->obs_mode == B2RL_OBS_RAW || p->obs_mode == B2RL_OBS_U8_TO_F32,
                 B2RL_ERR_INVALID, "unknown obs_mode %d", p->obs_mode);
    cudaStream_t s = (cudaStream_t)stream;
    B2RL_CUDA(cudaSetDevice(h->cfg.device));
    if (!h->sm_count)
        B2RL_CUDA(cudaDeviceGetAttribute(&h->sm_count, cudaDevAttrMultiProcessorCount, h->cfg.device));
    const b2rl_replay_config &c = h->cfg;

    // a deferred write-back too large for the in-launch path goes first, alone
    if (h->pending && h->pend_n > UPD_MAX) TRY(b2rl_flush_pending(h, s));

    // uniforms: device pointer, or host values through the ring of pinned slots
    const double *u_dev = p->u;
    if (!p->u_on_device) TRY(b2rl_upload_u(h, p->u, n, s, &u_dev));

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
        a.u = b2rl_update_args(h, h->pend_n, h->pend_err, h->pend_is_f64, h->pend_alpha,
                               h->pend_eps, h->pend_emin, h->pend_emax);
        a.u.stamps = h->times_dev + 3; // [3..7]: phases of the write-back
        a.upd_n = h->pend_n;
        a.upd_sync = h->ready_dev + 1;
    }
    a.times = h->times_dev;
    // ---- gather
    a.g = b2rl_gather_args(h, n, p->gamma_pow_host, p->obs_mode, p->obs_scale, &p->out);
    a.pieces = (c.part_bytes + PIECE_MAX - 1) / PIECE_MAX;
    a.piece_bytes = (((c.part_bytes + a.pieces - 1) / a.pieces) + 15) & ~15;
    a.stage_stride = (a.piece_bytes + 127) & ~127;
    a.poll_ns = p->mode == B2RL_SAMPLE_EXACT ? 400 : 100;

    const int nsides = (a.g.o_side[0] ? 1 : 0) + (a.g.o_side[1] ? 1 : 0);
    long long units = nsides ? (long long)n * nsides * c.stack * a.pieces : (n + STEP_THREADS - 1) / STEP_THREADS;
    int grid = h->sm_count;
    if (units + 1 < grid) grid = (int)units + 1;
    if (grid < 2) grid = 2;
    size_t smem = (size_t)GS * a.stage_stride + 2 * GS * sizeof(uint64_t);
    if (a.upd_n > 0) {
        const size_t us = update_multi_smem_bytes(h->levels);
        if (us > smem) smem = us;
    }
    h->last_step_grid = grid;
    B2RL_CUDA(launch_step(a, p->mode, grid, smem, s));
    h->pending = false;
    h->wait_priority = true;
    h->last_n = n;
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
