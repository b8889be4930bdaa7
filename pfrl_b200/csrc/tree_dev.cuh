// tree_dev.cuh -- device-side building blocks on the dense fp64 heaps, shared
// by the stand-alone kernels (sampler.cu) and the fused replay step (step.cu):
//
//   exact_deep<D>()        bit-exact sequential sampler (main warp + two scout
//                          warps + a publisher warp)
//   exact_deep_v6<D>()     bit-exact sampler deciding on approximate tables
//   sample_parallel()      all descents concurrently on the frozen tree
//   tree_update_multi()    priority write-back for <= 512 leaves: sorted
//                          paths, siblings prefetched in ONE round trip, the
//                          level loop runs on shared memory only
//
// Reference semantics (pure Python, pfrl/collections/prioritized.py):
//   :245-258 _find, :294-312 prioritized_sample, :107-116 set_last_priority,
//   :140-180 _reduce / _write; pfrl/replay_buffers/prioritized.py:47-66
//   priority_from_errors / weights_from_probabilities.
#pragma once
#include <math.h>

#include <type_traits>

#include "b2rl_internal.cuh"

static constexpr int TOP_LEVELS = 14; // heap levels 0..13 -> 16383 nodes = 128 KB
static constexpr int V6_T = 13;       // v6 keeps heap levels 0..12 in shared memory

struct SampleArgs {
    double *sum;
    const double *mn;
    B2rlDevState *st;
    const double *u;
    int n;
    int levels;      // leaves are at heap level `levels`
    long long nslots;
    int T;           // levels held in shared memory (nodes [1, 2^T))
    int D;           // levels below the shared part (0: leaves are in shared)
    int32_t *slots_out;
    double *prio_out;
    long long *index_out; // optional
    double *prio_user;    // optional
    // importance weights computed by the sampler itself (fused step); weight
    // and prob may be null (replay_buffers/prioritized.py:57-66)
    float *weight;
    double *prob;
    double beta;
    int norm;
    // publication of completed draws to other CTAs (fused step), or null:
    // *ready = seq_base | (number of draws whose outputs are visible)
    unsigned long long *ready;
    unsigned long long seq_base;
    // v6 test hooks (env B2RL_V6_SLOW_EVERY / B2RL_V6_EPS_SCALE): force the exact slow
    // path on every k-th draw / widen the decision margin; results must not change
    int dbg_slow_every;
    double dbg_eps_scale;
    long long *dbg_cycles; // optional [32]: clock64 sums per pipeline segment (tools/v6_cycles.py)
};

// The sampler that serves a draw of n from a tree with leaves at heap level `levels`; the
// values double as the MODE of the fused k_replay_step<D, MODE> (step.cu).
enum SamplerKind { SAMPLER_V5 = 0, SAMPLER_SMALL = 1, SAMPLER_PARALLEL = 2, SAMPLER_V6 = 3 };

struct SamplerChoice {
    SamplerKind kind;
    int D; // template depth of exact_deep<D> / exact_deep_v6<D>; 0 for the others
};

// parallel mode -> sample_parallel; a tree that fits the TOP_LEVELS shared-memory levels
// (SampleArgs::D == 0) -> exact_small; levels 17..21 with n <= 60000 -> v6 with D = levels - 12
// (it stages 5..9 levels per draw, and its conflict table keeps draw ids in u16); every other
// exact draw -> v5 with D = levels - 13.
inline SamplerChoice choose_sampler(int mode, int levels, int n)
{
    if (mode == B2RL_SAMPLE_PARALLEL) return {SAMPLER_PARALLEL, 0};
    if (levels < TOP_LEVELS) return {SAMPLER_SMALL, 0};
    if (levels >= 17 && levels <= 21 && n <= 60000) return {SAMPLER_V6, levels - (V6_T - 1)};
    return {SAMPLER_V5, levels - (TOP_LEVELS - 1)};
}

// f(std::integral_constant<int, d>{}) for a runtime d in [LO, HI]: turns the depth of a
// SamplerChoice into the template argument of the kernel that serves it.
template <int LO, int HI, typename F>
cudaError_t with_depth(int d, F &&f)
{
    if constexpr (LO > HI)
        return cudaErrorInvalidValue;
    else
        return d == LO ? f(std::integral_constant<int, LO>{}) : with_depth<LO + 1, HI>(d, f);
}

// ---------------------------------------------------------------------------
// small PTX helpers
// ---------------------------------------------------------------------------
// L2 residency: the sum tree (32 MB at 1M capacity) is re-read by every draw
// while the gather streams ~140 MB per minibatch through the same L2.  Tree
// accesses carry an evict_last policy (the gather's stores are .cs).
__device__ __forceinline__ uint64_t policy_evict_last()
{
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}

__device__ __forceinline__ double2 ld_tree_pair(const double2 *ptr, uint64_t pol)
{
    double2 v;
    asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v2.f64 {%0, %1}, [%2], %3;"
                 : "=d"(v.x), "=d"(v.y)
                 : "l"(ptr), "l"(pol));
    return v;
}

__device__ __forceinline__ void st_tree(double *ptr, double v, uint64_t pol)
{
    asm volatile("st.global.L2::cache_hint.f64 [%0], %1, %2;" ::"l"(ptr), "d"(v), "l"(pol)
                 : "memory");
}

__device__ __forceinline__ uint32_t smem_u32(const void *p)
{
    return (uint32_t)__cvta_generic_to_shared(p);
}

__device__ __forceinline__ void mbar_init(uint64_t *bar, int count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}

__device__ __forceinline__ void mbar_fence_init()
{
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
                 "r"(bytes)
                 : "memory");
}

__device__ __forceinline__ void mbar_arrive(uint64_t *bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t phase)
{
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(phase)
        : "memory");
    return ok != 0;
}

__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t phase)
{
    while (!mbar_try_wait(bar, phase)) {
    }
}

// cp.async.bulk (SASS UBLKCP): global -> shared, completion on an mbarrier
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src, uint32_t bytes,
                                         uint64_t *bar)
{
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
            "r"(smem_u32(dst_smem)),
        "l"(src), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}

__device__ __forceinline__ void bulk_s2g(void *dst, const void *src_smem, uint32_t bytes)
{
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst),
                 "r"(smem_u32(src_smem)), "r"(bytes)
                 : "memory");
}

__device__ __forceinline__ int ld_acquire_smem(const int *p)
{
    int v;
    asm volatile("ld.acquire.cta.shared.b32 %0, [%1];" : "=r"(v) : "r"(smem_u32(p)) : "memory");
    return v;
}

__device__ __forceinline__ void st_release_smem(int *p, int v)
{
    asm volatile("st.release.cta.shared.b32 [%0], %1;" ::"r"(smem_u32(p)), "r"(v) : "memory");
}

__device__ __forceinline__ unsigned long long ld_acquire_gpu(const unsigned long long *p)
{
    unsigned long long v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}

__device__ __forceinline__ void st_release_gpu(unsigned long long *p, unsigned long long v)
{
    asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// ---------------------------------------------------------------------------
// importance-sampling weight of one draw (replay_buffers/prioritized.py:57-66,
// probabilities of collections/prioritized.py:79-82 with uniform_ratio == 0)
// ---------------------------------------------------------------------------
__device__ __forceinline__ float is_weight(double prob, double denom, double len, double beta,
                                           int norm)
{
    const double base = (norm == B2RL_NORM_NONE) ? len * prob : prob / denom;
    return (float)pow(base, -beta);
}

// ---------------------------------------------------------------------------
// speculative lane-parallel descent (see sampler.cu header comment)
//
// The conditional subtraction `if (right) x -= left` is ONE fused multiply-add
// with a lane-constant multiplier: fma(-1, left, x) rounds x - left once,
// exactly like __dsub_rn; fma(-0, left, x) = x + (-0) = x because tree values
// are finite and >= 0.  The arithmetic of the winning lane is therefore bit
// for bit the reference's (the bit-identity suite checks it).
// ---------------------------------------------------------------------------
template <int R>
__device__ __forceinline__ void spec_round(const double *val, int &node, double &pos, int lane)
{
    static_assert(R >= 1 && R <= 5, "one round covers at most 5 levels");
    const int li = lane & ((1 << R) - 1);
    double left[R];
#pragma unroll
    for (int j = 0; j < R; j++) {
        const int nj = (node << j) + (li >> (R - j));
        left[j] = val[2 * nj];
    }
    double x = pos;
    bool ok = true;
#pragma unroll
    for (int j = 0; j < R; j++) {
        const bool right = (li >> (R - 1 - j)) & 1;
        const bool lt = x < left[j];
        ok = ok && (lt != right);
        x = __fma_rn(right ? -1.0 : -0.0, left[j], x);
    }
    unsigned m = __ballot_sync(0xffffffffu, ok);
    if constexpr (R < 5) m &= (1u << (1 << R)) - 1u;
    const int win = __ffs(m) - 1;
    pos = __shfl_sync(0xffffffffu, x, win);
    node = (node << R) + win;
}

template <int L>
__device__ __forceinline__ void spec_descend(const double *val, int &node, double &pos, int lane)
{
    if constexpr (L > 0) {
        constexpr int R = L >= 5 ? 5 : L;
        spec_round<R>(val, node, pos, lane);
        spec_descend<L - R>(val, node, pos, lane);
    }
}

// ---------------------------------------------------------------------------
// EXACT sampler for deep trees (levels >= TOP_LEVELS).  Called by ALL threads
// of the CTA (it uses __syncthreads); warps >= 4 only take part in the
// barriers.
//   warp 0 (main)      walks the draws in order, exactly as the reference does
//   warps 1, 2 (scouts) run a couple of draws ahead on the not-yet-final tree,
//                      predict which level-13 node a future draw will pick and
//                      stage that node's lower levels in shared memory, so the
//                      main warp's only global round trip per draw is usually
//                      done when it gets there (measured: ~99 % of the draws)
//   warp 3 (publisher) moves finished draws to global memory 32 at a time,
//                      computes their importance weights and (fused step)
//                      releases them to the gather CTAs
// The prediction is only a prefetch hint: the main warp uses the staged copy
// iff the predicted node equals the node its own exact descent reached AND no
// draw in flight when the copy was taken could have changed that subtree
// (release/acquire on `main_done` + "node != previous node").  The arithmetic
// of the main warp is the reference's, so indices stay bit-identical.
// Shared memory: [top 2^14 f64][sub_own 2^(D+1)][sub_pref 3 x 2^(D+1)]
// [o_prio ring][2 f64][o_slot ring][flags][mbarrier].
// ---------------------------------------------------------------------------
static constexpr int EX_RING = 64;    // finished draws waiting for the publisher
static constexpr int EX_NSCOUT = 2;
static constexpr int EX_LAG = 2;
static constexpr int EX_NBUF = EX_LAG + 1;

template <int D>
__host__ __device__ constexpr size_t exact_deep_smem_bytes()
{
    return sizeof(double) * ((size_t(1) << TOP_LEVELS) + (size_t(2) << D) * (1 + EX_NBUF) +
                             EX_RING + 2) +
           sizeof(int) * (EX_RING + 16) + 16;
}

template <int D>
__device__ __forceinline__ void exact_deep(const SampleArgs &a, double *smem_d)
{
    constexpr int T = TOP_LEVELS;
    constexpr int TOPN = 1 << T;
    constexpr int SUBN = 2 << D;
    constexpr int PAIRS = (1 << D) - 1; // child pairs below the chosen top node
    constexpr int NIT = (PAIRS + 31) / 32;
    constexpr int CHUNK = 32;
    constexpr int NSCOUT = EX_NSCOUT, LAG = EX_LAG, NBUF = EX_NBUF, RING = EX_RING;
    constexpr int F_READY = 0, F_NODE = 4, F_DONE = 8, F_PUB = 9;
    double *top = smem_d;
    double *sub_own = smem_d + TOPN;
    double *sub_pref = sub_own + SUBN;              // [NBUF][SUBN]
    double *o_prio = sub_pref + NBUF * SUBN;        // [RING]
    double *s_stat = o_prio + RING;                 // total, min-root
    int *o_slot = reinterpret_cast<int *>(s_stat + 2); // [RING]
    int *flags = o_slot + RING; // ready_seq[NBUF] @0, pred_node[NBUF] @4, main_done @8, pub_done @9
    uint64_t *bar = reinterpret_cast<uint64_t *>(flags + 16);
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;

    if (threadIdx.x == 0) {
        for (int i = 0; i < 16; i++) flags[i] = -1;
        flags[F_DONE] = 0;
        flags[F_PUB] = 0;
        mbar_init(bar, 1);
        mbar_fence_init();
        // earlier generic-proxy writes to the tree by this CTA (fused write-back)
        // must be visible to the bulk copy engine
        asm volatile("fence.proxy.async;" ::: "memory");
        mbar_expect_tx(bar, TOPN * 8);
#pragma unroll
        for (int c = 0; c < 4; c++)
            bulk_g2s(top + c * (TOPN / 4), a.sum + c * (TOPN / 4), TOPN * 2, bar);
    }
    __syncthreads();
    if (warp < 4) mbar_wait(bar, 0);

    const long long mask = a.nslots - 1;
    const long long npop = a.st->npop;
    const int older = ((npop & mask) >= (a.nslots >> 1)) ? 3 : 2;
    const uint64_t pol = policy_evict_last();
    const double2 *sum2 = reinterpret_cast<const double2 *>(a.sum);

    if (warp >= 1 && warp <= NSCOUT) {
        // ------------------------------ scouts -------------------------------
        for (int k = warp; k < a.n; k += NSCOUT) {
            const double uk = a.u[k];
            // draws 0..k-1-LAG must be complete (their stores visible) before we read
            while (ld_acquire_smem(&flags[F_DONE]) < k - LAG) __nanosleep(64);
            double pos = uk * top[1]; // approximate: up to LAG draws still in flight
            int node = older;
            {
                const double left = top[older];
                if (!(pos < left)) { pos -= left; node = older ^ 1; }
            }
            spec_descend<T - 2>(top, node, pos, lane);
            double *dst = sub_pref + (k % NBUF) * SUBN;
            const unsigned unode = (unsigned)node;
            double2 tmp[NIT];
#pragma unroll
            for (int it = 0; it < NIT; it++) {
                int q = lane + 32 * it;
                q = q < 1 ? 1 : (q > PAIRS ? PAIRS : q);
                const int dq = 31 - __clz(q);
                tmp[it] = ld_tree_pair(sum2 + ((unode << dq) + (unsigned)(q - (1 << dq))), pol);
            }
#pragma unroll
            for (int it = 0; it < NIT; it++) {
                int q = lane + 32 * it;
                q = q < 1 ? 1 : (q > PAIRS ? PAIRS : q);
                reinterpret_cast<double2 *>(dst)[q] = tmp[it];
            }
            __syncwarp();
            if (lane == 0) {
                flags[F_NODE + (k % NBUF)] = node;
                st_release_smem(&flags[F_READY + (k % NBUF)], k);
            }
            __syncwarp();
        }
    } else if (warp == 0) {
        // ------------------------------- main --------------------------------
        if (lane == 0) {
            const double total = top[1]; // priority_sums.sum(), :58
            const double mroot = a.mn[1]; // priority_mins.min(), :59
            a.st->last_total = total;
            a.st->last_min = mroot;
            a.st->last_n = a.n;
            s_stat[0] = total;
            s_stat[1] = mroot;
        }
        int prev_node[LAG];
#pragma unroll
        for (int i = 0; i < LAG; i++) prev_node[i] = -1;
        int hits = 0, late = 0;
        for (int k0 = 0; k0 < a.n; k0 += CHUNK) {
            const double u_lane = (k0 + lane < a.n) ? a.u[k0 + lane] : 0.0;
            const int kend = (a.n - k0 < CHUNK) ? a.n - k0 : CHUNK;
            // ring space: the publisher must have drained the chunk RING draws back
            while (ld_acquire_smem(&flags[F_PUB]) < k0 + CHUNK - RING) __nanosleep(32);
            for (int kk = 0; kk < kend; kk++) {
                const int k = k0 + kk;
                const double uk = __shfl_sync(0xffffffffu, u_lane, kk);
                // np.random.uniform(0.0, root) = 0.0 + (root - 0.0) * u, :302
                double pos = __dmul_rn(top[1], uk);
                int node = older;
                {
                    const double left = top[older];
                    if (!(pos < left)) {
                        pos = __dsub_rn(pos, left);
                        node = older ^ 1;
                    }
                }
                spec_descend<T - 2>(top, node, pos, lane); // level 1 -> T-1
                const unsigned unode = (unsigned)node;
                // ---- the D levels under `node`: staged by the scout, or fetched here
                const double *sub;
                const int ready_seq = ld_acquire_smem(&flags[F_READY + (k % NBUF)]);
                bool staged = ready_seq == k && flags[F_NODE + (k % NBUF)] == node;
                if (ready_seq != k) late++;
#pragma unroll
                for (int i = 0; i < LAG; i++) staged = staged && node != prev_node[i];
                if (staged) {
                    sub = sub_pref + (k % NBUF) * SUBN;
                    hits++;
                } else {
                    double2 tmp[NIT];
#pragma unroll
                    for (int it = 0; it < NIT; it++) {
                        int q = lane + 32 * it;
                        q = q < 1 ? 1 : (q > PAIRS ? PAIRS : q);
                        const int dq = 31 - __clz(q);
                        tmp[it] =
                            ld_tree_pair(sum2 + ((unode << dq) + (unsigned)(q - (1 << dq))), pol);
                    }
#pragma unroll
                    for (int it = 0; it < NIT; it++) {
                        int q = lane + 32 * it;
                        q = q < 1 ? 1 : (q > PAIRS ? PAIRS : q);
                        reinterpret_cast<double2 *>(sub_own)[q] = tmp[it];
                    }
                    __syncwarp();
                    sub = sub_own;
                }
                int rel = 1;
                spec_descend<D>(sub, rel, pos, lane);
                const unsigned leafnode = (unode << D) + (unsigned)(rel - (1 << D));
                const double prio = sub[rel];
                // ---- _write(ix, 0.0): re-reduce the path, siblings first (:303)
                double sib[D + T - 1];
#pragma unroll
                for (int j = 0; j < D; j++) sib[j] = sub[(rel >> j) ^ 1];
#pragma unroll
                for (int j = 0; j < T - 1; j++) sib[D + j] = top[(node >> j) ^ 1];
                double v = 0.0;
                if (lane == 0) st_tree(a.sum + leafnode, 0.0, pol);
#pragma unroll
                for (int j = 0; j < D; j++) {
                    v = __dadd_rn(v, sib[j]);
                    if (lane == 0) {
                        if (j + 1 < D) {
                            const int dp = D - j - 1; // depth of the relative parent
                            const unsigned p = (unsigned)(rel >> (j + 1));
                            st_tree(a.sum + ((unode << dp) + (p - (1u << dp))), v, pol);
                        } else {
                            top[node] = v;
                        }
                    }
                }
#pragma unroll
                for (int j = 0; j < T - 1; j++) {
                    v = __dadd_rn(v, sib[D + j]);
                    if (lane == 0) top[node >> (j + 1)] = v;
                }
                if (lane == 0) {
                    o_slot[k % RING] = (int)(leafnode - (unsigned)a.nslots);
                    o_prio[k % RING] = prio;
                    // publish "draws 0..k are complete" (global + shared stores above)
                    st_release_smem(&flags[F_DONE], k + 1);
                }
#pragma unroll
                for (int i = LAG - 1; i > 0; i--) prev_node[i] = prev_node[i - 1];
                prev_node[0] = node;
                __syncwarp();
            }
        }
        if (lane == 0) a.st->pad = hits | (late << 16); // scout diagnostics: hits, not-ready
    } else if (warp == 3) {
        // ----------------------------- publisher -----------------------------
        double total = 0.0, mroot = 0.0, bmin = INFINITY;
        const double len = (double)(a.st->napp - npop);
        for (int k0 = 0; k0 < a.n; k0 += CHUNK) {
            const int kend = (a.n - k0 < CHUNK) ? a.n : k0 + CHUNK;
            while (ld_acquire_smem(&flags[F_DONE]) < kend) __nanosleep(200);
            if (k0 == 0) {
                total = s_stat[0];
                mroot = s_stat[1];
            }
            const int k = k0 + lane;
            if (k < kend) {
                const long long slot = o_slot[k % RING];
                const double prio = o_prio[k % RING];
                a.slots_out[k] = (int32_t)slot;
                a.prio_out[k] = prio;
                if (a.index_out) a.index_out[k] = (slot - npop) & mask;
                if (a.prio_user) a.prio_user[k] = prio;
                const double p = prio / total;
                if (a.prob) a.prob[k] = p;
                bmin = fmin(bmin, p);
                if (a.weight && a.norm != B2RL_NORM_BATCH)
                    a.weight[k] = is_weight(p, mroot / total, len, a.beta, a.norm);
            }
            __syncwarp();
            if (lane == 0) {
                if (a.ready) st_release_gpu(a.ready, a.seq_base | (unsigned long long)kend);
                st_release_smem(&flags[F_PUB], kend);
            }
            __syncwarp();
        }
        if (a.weight && a.norm == B2RL_NORM_BATCH) {
            // np.min(probabilities) over the batch, replay_buffers/prioritized.py:60
            for (int o = 16; o > 0; o >>= 1) bmin = fmin(bmin, __shfl_xor_sync(0xffffffffu, bmin, o));
            for (int k = lane; k < a.n; k += 32)
                a.weight[k] = is_weight(a.prio_out[k] / total, bmin, len, a.beta, a.norm);
        }
    }
    __syncthreads();
    // publish the shared-memory levels (zeroed state) back to HBM: bulk store
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
        for (int c = 0; c < 4; c++)
            bulk_s2g(a.sum + c * (TOPN / 4), top + c * (TOPN / 4), TOPN * 2);
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    }
}

// ---------------------------------------------------------------------------
// EXACT sampler, whole tree in shared memory (levels < TOP_LEVELS).  Called by
// all threads of the CTA; warp 0 walks the draws.
// ---------------------------------------------------------------------------
__device__ __forceinline__ void exact_small(const SampleArgs &a, double *smem_d)
{
    double *top = smem_d;
    double *sub = smem_d + (1 << a.T);
    const int topn = 1 << a.T;
    const int tid = threadIdx.x;
    for (int i = 1 + tid; i < topn; i += blockDim.x) top[i] = a.sum[i];
    __syncthreads();

    if (tid < 32) {
        const int lane = tid;
        const long long mask = a.nslots - 1;
        const long long npop = a.st->npop;
        // The reference's root visits its OLDER half first
        // (collections/prioritized.py:255-258 with the bounds of :229-241).
        const int older = ((npop & mask) >= (a.nslots >> 1)) ? 3 : 2;
        const double total = top[1]; // priority_sums.sum(), :58
        const double mroot = a.mn[1]; // priority_mins.min(), :59
        const double len = (double)(a.st->napp - npop);
        if (lane == 0) {
            a.st->last_total = total;
            a.st->last_min = mroot;
            a.st->last_n = a.n;
        }
        double bmin = INFINITY;
        double unext = a.n > 0 ? a.u[0] : 0.0;
        for (int k = 0; k < a.n; k++) {
            const double uk = unext;
            if (k + 1 < a.n) unext = a.u[k + 1];
            // np.random.uniform(0.0, root) = 0.0 + (root - 0.0) * u, :302
            double pos = __dmul_rn(top[1], uk);
            // _find, :245-258
            int node = older;
            {
                const double left = top[older];
                if (!(pos < left)) {
                    pos = __dsub_rn(pos, left);
                    node = older ^ 1;
                }
            }
            for (int lv = 1; lv < a.T - 1; lv++) {
                const double left = top[2 * node];
                if (pos < left) {
                    node = 2 * node;
                } else {
                    pos = __dsub_rn(pos, left);
                    node = 2 * node + 1;
                }
            }
            long long leafnode;
            double prio;
            if (a.D > 0) {
                // one round trip: all D levels under `node`
                for (int j = 1; j <= a.D; j++) {
                    const int cnt = 1 << j;
                    const double *src = a.sum + ((long long)node << j);
                    for (int i = lane; i < cnt; i += 32) sub[cnt + i] = src[i];
                }
                __syncwarp();
                int rel = 1;
                for (int j = 0; j < a.D; j++) {
                    const double left = sub[2 * rel];
                    if (pos < left) {
                        rel = 2 * rel;
                    } else {
                        pos = __dsub_rn(pos, left);
                        rel = 2 * rel + 1;
                    }
                }
                leafnode = ((long long)node << a.D) + (rel - (1 << a.D));
                prio = sub[rel];
                // _write(ix, 0.0): zero the leaf, re-reduce the path, :303
                sub[rel] = 0.0;
                if (lane == 0) a.sum[leafnode] = 0.0;
                int dj = a.D - 1;
                for (int p = rel >> 1; p >= 2; p >>= 1, dj--) {
                    const double v = __dadd_rn(sub[2 * p], sub[2 * p + 1]);
                    sub[p] = v;
                    if (lane == 0) a.sum[((long long)node << dj) + (p - (1 << dj))] = v;
                }
                top[node] = __dadd_rn(sub[2], sub[3]);
            } else {
                leafnode = node;
                prio = top[node];
                top[node] = 0.0;
            }
            for (int p = node >> 1; p >= 1; p >>= 1)
                top[p] = __dadd_rn(top[2 * p], top[2 * p + 1]);
            if (lane == 0) {
                const long long slot = leafnode - a.nslots;
                a.slots_out[k] = (int32_t)slot;
                a.prio_out[k] = prio;
                if (a.index_out) a.index_out[k] = (slot - npop) & mask;
                if (a.prio_user) a.prio_user[k] = prio;
                const double p = prio / total;
                if (a.prob) a.prob[k] = p;
                bmin = fmin(bmin, p);
                if (a.weight && a.norm != B2RL_NORM_BATCH)
                    a.weight[k] = is_weight(p, mroot / total, len, a.beta, a.norm);
                if (a.ready && ((k & 31) == 31 || k == a.n - 1))
                    st_release_gpu(a.ready, a.seq_base | (unsigned long long)(k + 1));
            }
            __syncwarp();
        }
        if (lane == 0 && a.weight && a.norm == B2RL_NORM_BATCH)
            for (int k = 0; k < a.n; k++)
                a.weight[k] = is_weight(a.prio_out[k] / total, bmin, len, a.beta, a.norm);
    }
    __syncthreads();
    // publish the shared-memory levels (zeroed state) back to HBM
    for (int i = 1 + tid; i < topn; i += blockDim.x) a.sum[i] = top[i];
}

// ---------------------------------------------------------------------------
// PARALLEL mode: every draw descends the frozen tree on its own thread (with
// replacement).  Three levels per global round trip: the 8 great-grandchildren
// of a node are 64 contiguous bytes, and because every heap node is exactly
// fl(left + right) of its children the two levels in between are recomputed
// bit for bit from them -- the decisions are those of a level-by-level walk.
// Called by all threads of the CTA.  red: >= 32 doubles of shared memory.
// ---------------------------------------------------------------------------
__device__ __forceinline__ void sample_parallel(const SampleArgs &a, double *red)
{
    const long long mask = a.nslots - 1;
    const long long npop = a.st->npop;
    const double root = a.sum[1];
    const double mroot = a.mn[1];
    const double len = (double)(a.st->napp - npop);
    const int older = ((npop & mask) >= (a.nslots >> 1)) ? 3 : 2;
    const double older_v = a.sum[older];
    double bmin = INFINITY;
    for (int k = threadIdx.x; k < a.n; k += blockDim.x) {
        double pos = __dmul_rn(root, a.u[k]);
        long long node = older;
        if (!(pos < older_v)) {
            pos = __dsub_rn(pos, older_v);
            node = older ^ 1;
        }
        int rem = a.levels - 1;
        while (rem >= 3) {
            const double2 *g = reinterpret_cast<const double2 *>(a.sum + 8 * node);
            const double2 g01 = g[0], g23 = g[1], g45 = g[2], g67 = g[3];
            const double c0 = __dadd_rn(g01.x, g01.y), c1 = __dadd_rn(g23.x, g23.y);
            const double c2 = __dadd_rn(g45.x, g45.y);
            const double l0 = __dadd_rn(c0, c1);
            int b1 = 0, b2 = 0, b3 = 0;
            if (!(pos < l0)) { pos = __dsub_rn(pos, l0); b1 = 1; }
            const double l1 = b1 ? c2 : c0;
            if (!(pos < l1)) { pos = __dsub_rn(pos, l1); b2 = 1; }
            const double l2 = b1 ? (b2 ? g67.x : g45.x) : (b2 ? g23.x : g01.x);
            if (!(pos < l2)) { pos = __dsub_rn(pos, l2); b3 = 1; }
            node = 8 * node + 4 * b1 + 2 * b2 + b3;
            rem -= 3;
        }
        for (; rem > 0; rem--) {
            const double left = a.sum[2 * node];
            if (pos < left) {
                node = 2 * node;
            } else {
                pos = __dsub_rn(pos, left);
                node = 2 * node + 1;
            }
        }
        const double prio = a.sum[node];
        const long long slot = node - a.nslots;
        a.slots_out[k] = (int32_t)slot;
        a.prio_out[k] = prio;
        if (a.index_out) a.index_out[k] = (slot - npop) & mask;
        if (a.prio_user) a.prio_user[k] = prio;
        const double p = prio / root;
        if (a.prob) a.prob[k] = p;
        bmin = fmin(bmin, p);
        if (a.weight && a.norm != B2RL_NORM_BATCH)
            a.weight[k] = is_weight(p, mroot / root, len, a.beta, a.norm);
    }
    if (threadIdx.x == 0) {
        a.st->last_total = root;
        a.st->last_min = mroot;
        a.st->last_n = a.n;
    }
    if (a.weight && a.norm == B2RL_NORM_BATCH) {
        for (int o = 16; o > 0; o >>= 1) bmin = fmin(bmin, __shfl_xor_sync(0xffffffffu, bmin, o));
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = bmin;
        __syncthreads();
        bmin = INFINITY;
        for (int w = 0; w < (int)(blockDim.x >> 5); w++) bmin = fmin(bmin, red[w]);
        for (int k = threadIdx.x; k < a.n; k += blockDim.x)
            a.weight[k] = is_weight(a.prio_out[k] / root, bmin, len, a.beta, a.norm);
    }
    __syncthreads();
    if (threadIdx.x == 0 && a.ready) {
        __threadfence();
        st_release_gpu(a.ready, a.seq_base | (unsigned long long)a.n);
    }
}

// ---------------------------------------------------------------------------
// Priority write-back (set_last_priority, collections/prioritized.py:107-116,
// with priority_from_errors of replay_buffers/prioritized.py:47-55 in front
// when TD errors are given): tree_update_multi below for up to UPD_MAX leaves,
// the level-synchronous k_update (sampler.cu) for larger batches.
// ---------------------------------------------------------------------------
static constexpr int UPD_MAX = 512;

struct UpdateArgs {
    double *sum, *mn;
    B2rlDevState *st;
    const int32_t *slots;
    double *new_prio;       // [n] priorities (input, or scratch for the error form)
    const void *err;        // optional TD errors
    int err_is_f64;
    double alpha, eps, emin, emax;
    int32_t *winner;        // scratch of the level-synchronous kernel (n > UPD_MAX)
    int n, levels;
    long long nslots;
    // "repair" mode (append / eviction): the n touched leaves are the ring-slot ranges
    // below and already hold their values; only their ancestors are recomputed, then the
    // append / pop counters advance (collections/prioritized.py:207-242)
    int nranges;            // 0: normal write-back
    int r_first[4], r_count[4];
    long long bump_n, capacity;
    // measurement aid (b2rl_step_times [4..8]): %globaltimer stamps of the multi-CTA
    // write-back -- [0] CTA 0 collected its entries, [1] CTA 0 stored its subtree,
    // [2] CTA 0 has its arrival ticket, [3] last CTA holds the subtree roots,
    // [4] last CTA released the completion flag.  NULL: none.
    unsigned long long *stamps;
};

__device__ __forceinline__ void upd_stamp(const UpdateArgs &a, int slot)
{
    if (a.stamps) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        a.stamps[slot] = t;
    }
}

// (min(hi, max(lo, d)) + eps) ** alpha.  emin > emax: no clipping; an infinite bound is an
// absent one (DeviceReplayStore passes None as -inf / +inf), so a NaN error is clipped only by
// a finite bound, as Python's max / min do: max(lo, nan) == lo, min(hi, nan) == hi.  One edge
// differs: an explicit error_min = -inf with a NaN error gives NaN here, -inf in Python (the
// priority is then NaN or complex there, which set_last_priority rejects either way).
__device__ __forceinline__ double error_to_priority(double d, double alpha, double eps,
                                                    double emin, double emax)
{
    if (emin <= emax) {
        if (emin != -INFINITY) d = fmax(d, emin);
        if (emax != INFINITY) d = fmin(d, emax);
    }
    d += eps;
    // sqrt is correctly rounded; CUDA's pow(d, 1.0) can be 1 ulp off d, libm's is exact
    return (alpha == 0.5) ? sqrt(d) : (alpha == 1.0) ? d : pow(d, alpha);
}

__device__ __forceinline__ double priority_from_error(const UpdateArgs &a, int k)
{
    // priority_from_errors, replay_buffers/prioritized.py:47-55
    double d = a.err_is_f64 ? ((const double *)a.err)[k] : (double)((const float *)a.err)[k];
    return error_to_priority(d, a.alpha, a.eps, a.emin, a.emax);
}

// The top `topl` <= 10 levels (<= 1023 nodes) recomputed from level `topl` in shared
// memory (cheap barriers) instead of `topl` more global round trips: every node is a
// pure function of its children, so recomputing all of them is exact.  Used by the
// level-synchronous write-back (k_update) and append repair (k_tree_fix_small).
// Called by all threads of the CTA.
__device__ __forceinline__ void rebuild_top_levels(double *sum, double *mn, int topl)
{
    __shared__ double s_sum[2048], s_min[2048];
    const int tid = threadIdx.x, nt = blockDim.x;
    const int base = 1 << topl;
    for (int i = tid; i < base; i += nt) {
        s_sum[base + i] = sum[base + i];
        s_min[base + i] = mn[base + i];
    }
    __syncthreads();
    for (int lv = topl - 1; lv >= 0; lv--) {
        const int w = 1 << lv;
        for (int i = tid; i < w; i += nt) {
            const int node = w + i;
            s_sum[node] = s_sum[2 * node] + s_sum[2 * node + 1];
            s_min[node] = fmin(s_min[2 * node], s_min[2 * node + 1]);
        }
        __syncthreads();
    }
    for (int i = 1 + tid; i < base; i += nt) {
        sum[i] = s_sum[i];
        mn[i] = s_min[i];
    }
}

// ---------------------------------------------------------------------------
// Multi-CTA write-back of up to UPD_MAX leaves.
//
// A level-synchronous walk over global memory costs one L2 round trip per
// level (21 at 1 M capacity: 29 us for 512 leaves in round 1).  The sorted-path
// algorithm instead sorts the updated leaves, resolves duplicates (the
// reference writes in order, so the LAST occurrence wins), and fetches EVERY
// sibling any path can need up front in one round trip; the level loop then
// runs on shared memory only.  Sorted order makes the merge logic local: the
// paths below one node form a contiguous run of entries, the first entry of a
// run is its leader and carries the node's new value; two runs merge when they
// are the two children of one parent.  Every parent is computed as
// fl(left + right) / min(left, right) of its two children's final values,
// exactly what the reference's bottom-up _write produces after the whole batch.
//
// On one CTA that algorithm is bound by the SM's L1TEX: the ~21 x 512 x 2
// scattered 8-byte sibling loads are ~20 k wavefronts, ~2 cycles each (42 us
// measured).  So the heap splits into 2^sl independent subtrees below level sl
// (sl = min(7, levels)): CTA c runs the sorted-path algorithm on the updated
// leaves that fall into subtree c (typically 4 of 512) -- all subtrees in
// parallel on different SMs -- and the LAST CTA to arrive (atomic ticket)
// recomputes the 2^sl - 1 nodes above from the subtree roots (every node is a
// pure function of its children, so recomputing untouched ones changes
// nothing).  sync[0] = "write-back of launch `seq` complete" (release/acquire),
// sync[1] = arrival counter (self-resetting atomicInc).
// Called by all threads of every CTA of the grid; n <= UPD_MAX.
// ---------------------------------------------------------------------------
__host__ __device__ inline int update_split_level(int levels) { return levels < 7 ? levels : 7; }

__host__ __device__ inline size_t update_multi_smem_bytes(int levels)
{
    const int lb = levels - update_split_level(levels);
    return (size_t)UPD_MAX * (5 * 4 + 3 * 8) + 64 * 8 + (size_t)lb * UPD_MAX * 16 + 2 * 256 * 8;
}

__device__ __forceinline__ void tree_update_multi(const UpdateArgs &a, unsigned char *smem_raw,
                                                  unsigned long long *sync,
                                                  unsigned long long seq)
{
    const int tid = threadIdx.x, nt = blockDim.x;
    const int lane = tid & 31, warp = tid >> 5, nw = nt >> 5;
    const int sl = update_split_level(a.levels);
    const int lb = a.levels - sl;           // levels inside one subtree
    const int NS = 1 << sl;
    double *prio_k = reinterpret_cast<double *>(smem_raw);     // [UPD_MAX] by draw index
    double *vs = prio_k + UPD_MAX;                             // [UPD_MAX] by sorted entry
    double *vm = vs + UPD_MAX;
    double *red = vm + UPD_MAX;                                // [64]
    double *sib_s = red + 64;                                  // [lb][UPD_MAX]
    double *sib_m = sib_s + (size_t)lb * UPD_MAX;
    double *t_sum = sib_m + (size_t)lb * UPD_MAX;              // [256] top phase
    double *t_min = t_sum + 256;
    unsigned *keys = reinterpret_cast<unsigned *>(t_min + 256); // [UPD_MAX] unsorted
    unsigned *skeys = keys + UPD_MAX;                          // [UPD_MAX] sorted
    int *leaf = reinterpret_cast<int *>(skeys + UPD_MAX);      // [UPD_MAX] slot inside the ring
    int *runlen = leaf + UPD_MAX;
    int *lead = runlen + UPD_MAX;
    int *ctr = reinterpret_cast<int *>(red) + 64;              // [0] count, [1] last flag, [2..] group counts
    double mx = 0.0;

    for (int st = blockIdx.x; st < NS; st += gridDim.x) {
        if (tid == 0) ctr[0] = 0;
        __syncthreads();
        // ---- collect the draws whose leaf lies in subtree `st`
        for (int k = tid; k < a.n; k += nt) {
            int slot;
            if (a.nranges > 0) {
                int r = 0, off = k;
                while (off >= a.r_count[r]) off -= a.r_count[r++];
                slot = a.r_first[r] + off;
            } else {
                slot = a.slots[k];
            }
            if ((slot >> lb) != st) continue;
            if (a.nranges == 0) {
                const double p = a.err ? priority_from_error(a, k) : a.new_prio[k];
                if (a.err) a.new_prio[k] = p;
                prio_k[k] = p;
                mx = fmax(mx, p); // max_priority sees every value, :114
            }
            const int pos = atomicAdd(&ctr[0], 1);
            keys[pos] = ((unsigned)(slot & ((1 << lb) - 1)) << 16) | (unsigned)k;
        }
        __syncthreads();
        const int cnt = ctr[0];
        if (blockIdx.x == 0 && tid == 0 && st == 0) upd_stamp(a, 0);
        if (cnt == 0) continue; // uniform
        // A subtree usually gets a handful of the 512 leaves: one warp then does the rest
        // with warp barriers only (no 512-thread barrier per level); a crowded subtree
        // takes the whole CTA.
        const bool solo = cnt <= 32;
        const int wt = solo ? lane : tid;        // worker index / count inside the team
        const int wn = solo ? 32 : nt;
        const int ww = solo ? 0 : warp, wnw = solo ? 1 : nw;
        const bool member = !solo || warp == 0;
#define TEAM_SYNC()            \
    do {                       \
        if (solo)              \
            __syncwarp();      \
        else                   \
            __syncthreads();   \
    } while (0)
        if (member) {
            // ---- rank sort by (slot, draw index); keys are distinct
            for (int i = wt; i < cnt; i += wn) {
                const unsigned key = keys[i];
                int rank = 0;
                for (int j = 0; j < cnt; j++) rank += keys[j] < key;
                skeys[rank] = key;
            }
            TEAM_SYNC();
            // ---- unique leaves (last occurrence of a slot wins), compaction
            const int ngroups = (cnt + 31) >> 5;
            for (int g = ww; g < ngroups; g += wnw) {
                const int i = g * 32 + lane;
                const bool w = i < cnt && (i == cnt - 1 || (skeys[i + 1] >> 16) != (skeys[i] >> 16));
                const unsigned b = __ballot_sync(0xffffffffu, w);
                if (lane == 0) ctr[2 + g] = __popc(b);
            }
            TEAM_SYNC();
            int m = 0;
            for (int g = 0; g < ngroups; g++) m += ctr[2 + g];
            for (int g = ww; g < ngroups; g += wnw) {
                const int i = g * 32 + lane;
                const bool w = i < cnt && (i == cnt - 1 || (skeys[i + 1] >> 16) != (skeys[i] >> 16));
                const unsigned b = __ballot_sync(0xffffffffu, w);
                int base = 0;
                for (int q = 0; q < g; q++) base += ctr[2 + q];
                if (w) {
                    const int pos = base + __popc(b & ((1u << lane) - 1u));
                    const int lf = (st << lb) | (int)(skeys[i] >> 16);
                    leaf[pos] = lf;
                    if (a.nranges > 0) { // repair: the leaves are already in place
                        vs[pos] = a.sum[a.nslots + lf];
                        vm[pos] = a.mn[a.nslots + lf];
                    } else {
                        const double p = prio_k[skeys[i] & 0xffffu];
                        vs[pos] = p;
                        vm[pos] = p;
                    }
                    runlen[pos] = 1;
                    lead[pos] = 1;
                }
            }
            TEAM_SYNC();
            if (blockIdx.x == 0 && wt == 0) upd_stamp(a, 197);
            // ---- leaves out, every sibling of every path inside the subtree in
            if (a.nranges == 0)
                for (int i = wt; i < m; i += wn) {
                    const long long ln = a.nslots + leaf[i];
                    a.sum[ln] = vs[i];
                    a.mn[ln] = vm[i];
                }
            for (int idx = wt; idx < m * lb; idx += wn) {
                const int i = idx % m, s = idx / m;
                const long long node = (a.nslots + leaf[i]) >> s;
                sib_s[(size_t)s * UPD_MAX + i] = a.sum[node ^ 1];
                sib_m[(size_t)s * UPD_MAX + i] = a.mn[node ^ 1];
            }
            TEAM_SYNC();
            if (blockIdx.x == 0 && wt == 0) upd_stamp(a, 198);
            // ---- level loop on shared memory: at level s a leader whose node is a left child
            // merges the run of its right sibling if that run exists, or else combines with the
            // prefetched sibling; a right child whose left sibling leads a run was merged by that
            // leader and stops leading.  The node values go to
            // global memory AFTER the loop, in one batch, so that no global store sits in front
            // of a level's barrier; the results are parked in the sibling slots (level s, entry i)
            // they were computed from, -1 marks the entries that wrote nothing at that level
            // (node sums are never negative).  Measured (b2rl_step_times, B2RL_WB_FINE=1): the
            // loop still costs ~0.4 us per level -- a chain of dependent shared-memory loads
            // behind the previous level's stores -- 5.5 of the write-back's 19 us.
            for (int s = 0; s < lb; s++) {
                for (int i = wt; i < m; i += wn) {
                    const size_t slot = (size_t)s * UPD_MAX + i;
                    if (!lead[i]) {
                        sib_s[slot] = -1.0;
                        continue;
                    }
                    const long long node = (a.nslots + leaf[i]) >> s;
                    double ns, nm;
                    if ((node & 1) == 0) {
                        const int j = i + runlen[i];
                        if (j < m && ((a.nslots + leaf[j]) >> s) == node + 1) {
                            ns = __dadd_rn(vs[i], vs[j]);
                            nm = fmin(vm[i], vm[j]);
                            runlen[i] += runlen[j];
                        } else {
                            ns = __dadd_rn(vs[i], sib_s[slot]);
                            nm = fmin(vm[i], sib_m[slot]);
                        }
                    } else {
                        if (i > 0 && ((a.nslots + leaf[i - 1]) >> s) == node - 1) {
                            lead[i] = 0;
                            sib_s[slot] = -1.0;
                            continue;
                        }
                        ns = __dadd_rn(sib_s[slot], vs[i]);
                        nm = fmin(sib_m[slot], vm[i]);
                    }
                    vs[i] = ns;
                    vm[i] = nm;
                    sib_s[slot] = ns;
                    sib_m[slot] = nm;
                }
                TEAM_SYNC();
            }
            for (int idx = wt; idx < m * lb; idx += wn) {
                const int i = idx % m, s = idx / m;
                const double ns = sib_s[(size_t)s * UPD_MAX + i];
                if (ns < 0.0) continue;
                const long long parent = (a.nslots + leaf[i]) >> (s + 1);
                a.sum[parent] = ns;
                a.mn[parent] = sib_m[(size_t)s * UPD_MAX + i];
            }
            if (blockIdx.x == 0 && wt == 0) upd_stamp(a, 199);
        }
#undef TEAM_SYNC
        __syncthreads(); // the team rejoins the CTA (uniform: cnt is the same for all)
    }
    // ---- max_priority (positive doubles order like their bit patterns), arrival
    if (blockIdx.x == 0 && tid == 0) upd_stamp(a, 1);
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    __threadfence(); // this thread's node stores before the CTA's arrival ticket
    __syncthreads();
    if (lane == 0) red[warp] = mx;
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < nw; w++) mx = fmax(mx, red[w]);
        if (mx > 0.0)
            atomicMax(reinterpret_cast<unsigned long long *>(&a.st->max_priority),
                      (unsigned long long)__double_as_longlong(mx));
        __threadfence();
        const unsigned prev = atomicInc(reinterpret_cast<unsigned *>(sync + 1), gridDim.x - 1);
        ctr[1] = (prev == gridDim.x - 1);
        if (blockIdx.x == 0) upd_stamp(a, 2);
    }
    __syncthreads();
    if (ctr[1]) {
        // ---- last CTA: the sl levels above the subtree roots
        __threadfence();
        for (int i = tid; i < NS; i += nt) {
            t_sum[NS + i] = __ldcg(a.sum + NS + i);
            t_min[NS + i] = __ldcg(a.mn + NS + i);
        }
        __syncthreads();
        if (tid == 0) upd_stamp(a, 3);
        for (int lv = sl - 1; lv >= 0; lv--) {
            const int w = 1 << lv;
            for (int i = tid; i < w; i += nt) {
                const int node = w + i;
                t_sum[node] = __dadd_rn(t_sum[2 * node], t_sum[2 * node + 1]);
                t_min[node] = fmin(t_min[2 * node], t_min[2 * node + 1]);
            }
            __syncthreads();
        }
        for (int i = 1 + tid; i < NS; i += nt) {
            a.sum[i] = t_sum[i];
            a.mn[i] = t_min[i];
        }
        if (tid == 0) {
            if (a.nranges == 0) {
                a.st->last_n = 0;
            } else if (a.bump_n > 0) {
                long long napp = a.st->napp + a.bump_n;
                long long npop = a.st->npop;
                if (napp - npop > a.capacity) npop = napp - a.capacity;
                a.st->napp = napp;
                a.st->npop = npop;
            }
        }
        __threadfence();
        __syncthreads();
        if (tid == 0) st_release_gpu(sync, seq);
        if (tid == 0) upd_stamp(a, 4);
    }
}

#ifndef B2RL_V6_PROFILE
#define B2RL_V6_PROFILE 0 // 1: clock64 sums per pipeline segment (b2rl_step_times [4..35])
#endif
#if B2RL_V6_PROFILE
#define V6_CLK() clock64()
#else
#define V6_CLK() 0ll
#endif

// ===========================================================================
// EXACT sampler v6: decisions on approximate prefix tables, proofs by margin,
// the exact re-reduction trails on its own warp.
//
// The reference's draw k is a dependent chain: pos = u_k * root_k, 21 compare /
// subtract steps down, then `_write(ix, 0.0)` re-reduces 21 nodes bottom-up
// (each fl(left + right)) to give root_k+1 -- and only then can draw k+1 start
// (collections/prioritized.py:245-258, 294-312, 140-180).  v5 walks exactly
// that chain on one warp (~0.75 us per draw: ~400 dependent instructions).
//
// What the caller needs from draw k is only the LEAF (its index and priority);
// `pos` is thrown away.  The leaf is determined by the signs of the comparisons
// `pos_j < left_j`, and a sign can be proven without the exact operands: the
// positions that lead to a given node form an interval [prefix, prefix + mass)
// of the descent order, so if approximations of prefix and mass with error
// < EPS put pos farther than EPS inside the interval, every comparison on the
// way has the reference's outcome.  So:
//
//   * top 13 levels -> three approximate tables over the 4096 level-12 nodes in
//     descent order (the reference visits the OLDER half of the ring first):
//     M[o] mass, P_lo[o] prefix inside its block of 64, P_hi[b] prefix of the
//     blocks.  After a draw of priority p at node o they are updated by plain
//     subtractions, all entries at once (lanes): M[o], P_lo[e > o in the
//     block], P_hi[b' > block].  Errors: each entry sees <= n roundings of
//     <= 2^-53 root, the initial sums <= 80; EPS = (n + 64) 2^-46 root is > 40x
//     everything a decision depends on (DESIGN.md has the budget).
//   * bottom 9 levels -> the scout that stages the predicted node's subtree
//     (exact values, one global round trip, ~4 draws ahead) also lays down the
//     running sums Q[0..512] of its 512 leaves.
//   * the main warp decides draw k with
//         pos12 = u_k * rootA - P_hi[o >> 6] - P_lo[o]   (must be in (EPS, M[o] - EPS))
//         two 32-way compares of pos12 against Q         (leaf i; pos12 farther
//                                                         than EPS from Q[i], Q[i+1])
//     and no draw still in flight in the exact pipeline touched that subtree.
//     Any doubt (late or wrong scout, margin, conflict) -> SLOW PATH: wait until
//     the exact tree has caught up and run the reference's arithmetic on it (the
//     v5 code).  Never wrong, only slow; the count is reported
//     (b2rl_per_info.scout_hits: fast | slow << 16).
//   * the ascent warp applies draw k to the EXACT tree (shared-memory top +
//     global bottom) with the reference's bottom-up adds, one draw after the
//     other, a few draws behind.  The tree that goes back to HBM and every
//     priority returned are exact.
//   * four scout warps; a publisher warp moves results out.
// tools/v6_model.py is a CPU model of the decision logic (adversarial trees:
// ties, 1e-30..1e+30 dynamic range, u on boundaries, mispredictions).
// ===========================================================================
static constexpr int V6_NSCOUT = 4;
static constexpr int V6_LAG = 4;
static constexpr int V6_NBUF = 6;
static constexpr int V6_Q = 16;
static constexpr int V6_NTOP = 1 << (V6_T - 1);  // 4096 level-12 nodes
// Warp roles.  The issue arbiter of an SM sub-partition (warp id % 4) prefers its
// highest eligible warp id, so the latency-critical main warp gets a sub-partition to
// itself and all four scouts share another one.
static constexpr int V6_W_MAIN = 3, V6_W_ASC = 1, V6_W_PUB = 2; // scouts: warps 0, 4, 8, 12
static constexpr int V6_THREADS = 512;

// One staged subtree: [the 2^(D+1) nodes below a level-12 node, relative heap order: node r
// has children 2r, 2r+1, leaves at r >= 2^D][QB: exclusive running sums of the 32 nodes five
// levels down + their total].  The nodes arrive by cp.async.bulk (one copy per level, the
// level's slice is contiguous in the heap): the copy engine goes global -> shared without
// touching the SM's L1TEX pipe, which the main warp's shared-memory loads depend on (LDG
// staging with 32 KB in flight behind a 13 KB L1 made every LDS of the SM wait: ncu showed
// 330-cycle shared loads).
__host__ __device__ constexpr size_t v6_buf_doubles(int D)
{
    return (size_t(2) << D) + 40;
}

template <int D>
__host__ __device__ constexpr size_t exact_v6_smem_bytes()
{
    // etop, M, P_lo, P_hi(64) + rootA + stat(2) + pad, sub_own, NBUF x staged buffer, o_prio
    return sizeof(double) * ((size_t(1) << V6_T) + 2 * V6_NTOP + 80 + (size_t(2) << D) +
                             V6_NBUF * v6_buf_doubles(D) + 2 * EX_RING) +
           sizeof(int) * 32 + sizeof(unsigned short) * V6_NTOP + 16 + 8 * V6_NBUF;
}

// One speculative round of R levels on approximate `pos` (see spec_round): the lane whose
// comparisons are all consistent wins; `safe` is kept only if every comparison of that lane
// is farther than eps from equality.
template <int R>
__device__ __forceinline__ void spec_round_margin(const double *val, int &node, double &pos,
                                                  bool &safe, double eps, int lane)
{
    if constexpr (R > 0) {
        const int li = lane & ((1 << R) - 1);
        double left[R];
#pragma unroll
        for (int j = 0; j < R; j++) {
            const int nj = (node << j) + (li >> (R - j));
            left[j] = val[2 * nj];
        }
        double x = pos;
        bool ok = true, far = true;
#pragma unroll
        for (int j = 0; j < R; j++) {
            const bool right = (li >> (R - 1 - j)) & 1;
            const double d = x - left[j];
            ok = ok && ((d < 0.0) != right);
            far = far && (fabs(d) > eps);
            x = right ? d : x;
        }
        unsigned m = __ballot_sync(0xffffffffu, ok && far);
        if constexpr (R < 5) m &= (1u << (1 << R)) - 1u;
        safe = safe && m != 0;
        node = (node << R) + (m ? __ffs(m) - 1 : 0);
    }
}

template <int D>
__device__ __forceinline__ void exact_deep_v6(const SampleArgs &a, double *smem_d)
{
    constexpr int T = V6_T;
    constexpr int TOPN = 1 << T;
    constexpr int NTOP = V6_NTOP;
    constexpr int SUBN = 2 << D;
    constexpr int NLEAF = 1 << D;               // leaves under one level-12 node
    constexpr int BUFN = (int)v6_buf_doubles(D);
    constexpr int O_QB = SUBN;                  // [33] running sums of the depth-5 nodes
    constexpr int R2 = D - 5;                   // levels below the 32-way split
    constexpr int PAIRS = (1 << D) - 1;         // child pairs of a whole subtree (slow path)
    constexpr int NIT = (PAIRS + 31) / 32;
    constexpr int CHUNK = 32;
    constexpr int NSCOUT = V6_NSCOUT, LAG = V6_LAG, NBUF = V6_NBUF, RING = EX_RING;
    constexpr int Q = V6_Q;
    // F_ASC:  draws whose exact update is VISIBLE (global stores fenced), published in
    //         batches -- the fence waits for the L2 acknowledgement of the ascent's global
    //         stores and a MEMBAR holds up the SM's shared-memory pipe for everybody, so it
    //         must not be paid per draw;
    // F_ASCR: draws the ascent warp has finished READING the inputs of (relaxed, per draw):
    //         staged buffers and queue slots can be reused.
    constexpr int F_MAIN = 24, F_ASC = 25, F_PUB = 26, F_ASCR = 27;
    constexpr int ASC_BATCH = 4;
    static_assert(D >= 5 && D <= 9, "v6 stages 5..9 levels per draw");
    double *etop = smem_d;                      // exact top, levels 0..12
    double *mtab = etop + TOPN;                 // [NTOP] approximate node mass, descent order
    double *plo = mtab + NTOP;                  // [NTOP] approximate prefix inside a block of 64
    double *phi = plo + NTOP;                   // [64]   approximate prefix of the blocks
    double *s_misc = phi + 64;                  // [8]: rootA, total, min-root
    // [NBUF] one word per staged buffer: draw << 32 | F_ASC seen << 12 | node (descent order)
    unsigned long long *ready64 = reinterpret_cast<unsigned long long *>(s_misc + 8);
    double *sub_own = s_misc + 16;
    double *sub_pref = sub_own + SUBN;          // [NBUF][BUFN]
    // one 16-byte entry per decided draw, read by the ascent warp and by the publisher:
    // {ring slot of the leaf, staged buffer (NBUF = sub_own), priority}
    struct DrawEnt {
        int slot, buf;
        double prio;
    };
    DrawEnt *ring = reinterpret_cast<DrawEnt *>(sub_pref + NBUF * BUFN); // [RING]
    int *flags = reinterpret_cast<int *>(ring + RING);                   // [32]
    uint64_t *bar = reinterpret_cast<uint64_t *>(flags + 32); // [1 + NBUF]: top copy, staged buffers
    // 1 + index of the last draw of this launch that chose node o (0 = none): the conflict
    // test "did a draw still in flight touch this subtree" is one load, no vote
    unsigned short *lastd = reinterpret_cast<unsigned short *>(bar + 2 + NBUF);
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;

    if (threadIdx.x == 0) {
        for (int i = 0; i < 32; i++) flags[i] = -1;
        flags[F_MAIN] = 0;
        flags[F_ASC] = 0;
        flags[F_ASCR] = 0;
        flags[F_PUB] = 0;
        mbar_init(bar, 1);
        for (int i = 0; i < NBUF; i++) mbar_init(bar + 2 + i, 1);
        mbar_fence_init();
        asm volatile("fence.proxy.async;" ::: "memory");
        mbar_expect_tx(bar, TOPN * 8);
#pragma unroll
        for (int c = 0; c < 4; c++)
            bulk_g2s(etop + c * (TOPN / 4), a.sum + c * (TOPN / 4), TOPN * 2, bar);
    }
    __syncthreads();
    mbar_wait(bar, 0);

    const long long mask = a.nslots - 1;
    const long long npop = a.st->npop;
    const int older = ((npop & mask) >= (a.nslots >> 1)) ? 3 : 2;
    const int oflip = older == 2 ? 0 : NTOP / 2; // descent order o <-> node 4096 + (o ^ oflip)
    // ---- the approximate tables, from the exact top
    for (int o = threadIdx.x; o < NTOP; o += blockDim.x) {
        mtab[o] = etop[NTOP + (o ^ oflip)];
        lastd[o] = 0;
    }
    if (threadIdx.x < 8) ready64[threadIdx.x] = ~0ull;
    __syncthreads();
    if (threadIdx.x < 64) {
        double run = 0.0;
        const int b = threadIdx.x;
        for (int i = 0; i < 64; i++) {
            plo[64 * b + i] = run;
            run += mtab[64 * b + i];
        }
    } else if (threadIdx.x == 64) {
        double run = 0.0;
        for (int b = 0; b < 64; b++) {
            phi[b] = run;
            run += etop[64 + (b ^ (oflip >> 6))]; // level-6 nodes = sums of 64 level-12 nodes
        }
    }
    __syncthreads();

    const uint64_t pol = policy_evict_last();
    const double2 *sum2 = reinterpret_cast<const double2 *>(a.sum);
    const double root0 = etop[1];
    if (threadIdx.x == 0) s_misc[0] = root0;
    // decision margin (see the header comment / DESIGN.md)
    const double eps = root0 * (double)(a.n + 64) * 1.4210854715202004e-14 /* 2^-46 */ *
                       (a.dbg_eps_scale > 0.0 ? a.dbg_eps_scale : 1.0);
    __syncthreads();

    if ((warp & 3) == 0 && (warp >> 2) < NSCOUT) {
        // ------------------------------ scouts -------------------------------
        const double pbar = root0 / (double)(a.st->napp - npop); // expected mass per draw
        long long c_wait = 0, c_fetch = 0, c_rest = 0;
        for (int k = warp >> 2; k < a.n; k += NSCOUT) {
            const long long tc0 = V6_CLK();
            const double uk = a.u[k];
            const int b = k % NBUF;
            int m;
            while ((m = ld_acquire_smem(&flags[F_MAIN])) < k - LAG ||
                   ld_acquire_smem(&flags[F_ASCR]) < k - NBUF + 1)
                __nanosleep(32);
            const long long tc1 = V6_CLK();
            // ---- prediction (any error only costs a slow draw): search the tables
            double pos = uk * (s_misc[0] - (double)(k - m) * pbar);
            int blk = __popc(__ballot_sync(0xffffffffu, pos >= phi[lane])) +
                      __popc(__ballot_sync(0xffffffffu, pos >= phi[lane + 32])) - 1;
            blk = blk < 0 ? 0 : blk;
            pos -= phi[blk];
            int w = __popc(__ballot_sync(0xffffffffu, pos >= plo[64 * blk + lane])) +
                    __popc(__ballot_sync(0xffffffffu, pos >= plo[64 * blk + lane + 32])) - 1;
            w = w < 0 ? 0 : w;
            const int ord = 64 * blk + w;
            const unsigned unode = (unsigned)(NTOP + (ord ^ oflip));
            const int seen = ld_acquire_smem(&flags[F_ASC]);
            double *dst = sub_pref + b * BUFN;
            // ---- one bulk copy per level: the 2^j nodes j levels below `unode` are contiguous
            uint64_t *sb = bar + 2 + b;
            if (lane == 0) {
                mbar_expect_tx(sb, (uint32_t)((SUBN - 2) * 8));
#pragma unroll
                for (int j = 1; j <= D; j++)
                    bulk_g2s(dst + (1 << j), a.sum + ((size_t)unode << j), (uint32_t)(8u << j), sb);
            }
            const long long tc2 = V6_CLK();
            while (!mbar_try_wait(sb, (uint32_t)((k / NBUF) & 1))) {
            }
            // ---- running sums of the 32 nodes five levels down (warp scan)
            {
                const double bs = dst[32 + lane];
                double incl = bs;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const double up = __shfl_up_sync(0xffffffffu, incl, o);
                    if (lane >= o) incl += up;
                }
                dst[O_QB + lane] = incl - bs;
                if (lane == 31) dst[O_QB + 32] = incl;
            }
            __syncwarp();
            if (lane == 0) {
                const unsigned long long wv = ((unsigned long long)(unsigned)k << 32) |
                                              ((unsigned long long)(unsigned)seen << 12) |
                                              (unsigned long long)ord;
                asm volatile("st.release.cta.shared.b64 [%0], %1;" ::"r"(smem_u32(&ready64[b])),
                             "l"(wv)
                             : "memory");
            }
            __syncwarp();
            const long long tc3 = V6_CLK();
            c_wait += tc1 - tc0;
            c_fetch += tc2 - tc1;   // prediction + issue of the loads + store of the internal levels
            c_rest += tc3 - tc2;    // leaf loads arrive, running sums, stores, release
        }
        if (a.dbg_cycles && lane == 0 && warp == 0) {
            a.dbg_cycles[8] = c_wait;
            a.dbg_cycles[9] = c_fetch;
            a.dbg_cycles[10] = c_rest;
        }
    } else if (warp == V6_W_MAIN) {
        // ------------------------------- main --------------------------------
        if (lane == 0) {
            const double mroot = a.mn[1]; // priority_mins.min(), :59
            a.st->last_total = root0;     // priority_sums.sum(), :58
            a.st->last_min = mroot;
            a.st->last_n = a.n;
            s_misc[1] = root0;
            s_misc[2] = mroot;
        }
        // The loop is software-pipelined around one measured fact: a shared-memory LOAD
        // issued behind this warp's own STOREs waits 100-200 cycles for them to drain
        // (ncu: three such load -> DADD pairs were 45 % of the draw).  So every draw issues
        // ALL its loads first -- including the ones the NEXT draw needs -- and its stores
        // last.  The next draw's table entries are therefore read before this draw's update
        // is stored; the one missing update is applied in registers (ord_prev, p_prev).
        double rootA = root0;
        int nfast = 0, nslow = 0;
        // prefetched state of the draw about to be decided
        int pf_rs = -1, pf_o = 0, pf_seen = 0, pf_last = 0;
        double pf_pre = 0.0, pf_mass = 0.0, pf_qb = 0.0;
        bool pf_stale = false;      // read before the previous draw's stores
        int ord_prev = -1;
        double p_prev = 0.0;
        long long c_ready = 0, c_decide = 0, c_queue = 0, c_loads = 0, c_stores = 0;
        auto prefetch = [&](int k) {
            const int b = k % NBUF;
            // plain (volatile) load of the ready word: an acquire would park this warp until
            // the load returns; the loads below are performed after it in the SM's in-order
            // shared-memory pipe, behind the scout's release, which is all the ordering needed
            unsigned long long wv;
            asm volatile("ld.volatile.shared.b64 %0, [%1];"
                         : "=l"(wv)
                         : "r"(smem_u32(&ready64[b]))
                         : "memory");
            pf_rs = (int)(wv >> 32);
            pf_o = (int)(wv & (NTOP - 1));          // garbage unless pf_rs == k, but in range
            pf_seen = (int)((wv >> 12) & 0xfffffu);
            pf_pre = phi[pf_o >> 6] + plo[pf_o];
            pf_mass = mtab[pf_o];
            pf_last = lastd[pf_o];
            pf_qb = sub_pref[b * BUFN + O_QB + lane];
        };
        if (a.n > 0) prefetch(0);
        for (int k0 = 0; k0 < a.n; k0 += CHUNK) {
            const double u_lane = (k0 + lane < a.n) ? a.u[k0 + lane] : 0.0;
            const int kend = (a.n - k0 < CHUNK) ? a.n - k0 : CHUNK;
            while (ld_acquire_smem(&flags[F_PUB]) < k0 + CHUNK - RING) __nanosleep(32);
            for (int kk = 0; kk < kend; kk++) {
                const int k = k0 + kk;
                const long long tm0 = V6_CLK();
                const double uk = __shfl_sync(0xffffffffu, u_lane, kk);
                const int b = k % NBUF;
                int ord = 0, rel = 1;
                double prio = 0.0;
                bool fast = false;
                // ---- the scout's staging of draw k: prefetched, or wait for it (bounded)
                if (pf_rs != k) {
                    for (int spin = 0; spin < 48; spin++) {
                        unsigned long long wv;
                        asm volatile("ld.acquire.cta.shared.b64 %0, [%1];"
                                     : "=l"(wv)
                                     : "r"(smem_u32(&ready64[b]))
                                     : "memory");
                        if ((int)(wv >> 32) == k) break;
                    }
                    prefetch(k);
                    pf_stale = false;
                }
                // this draw's prefetched state moves to locals; the NEXT draw's loads start now,
                // behind no store of this warp, and overlap the whole decision below
                const int c_rs = pf_rs, c_o = pf_o, c_seen = pf_seen, c_last = pf_last;
                const double c_pre = pf_pre, c_mass = pf_mass, c_qb = pf_qb;
                const bool c_stale = pf_stale;
                if (k + 1 < a.n) {
                    prefetch(k + 1);
                    pf_stale = true;
                }
                const long long tm1 = V6_CLK();
                if (c_rs == k && !(a.dbg_slow_every > 0 && k % a.dbg_slow_every == 0)) {
                    const int o = c_o;
                    // a draw not yet applied to the exact tree when the copy was taken chose
                    // the same node?  (draw j is recorded as j + 1; the previous draw may
                    // still be missing from the table when the entry was read)
                    const bool conflict = c_last > c_seen || (c_stale && ord_prev == o) ||
                                          k - c_seen > 60000;
                    // position inside the node: u * root minus everything before it
                    double pre = c_pre;
                    if (c_stale && ord_prev < o) pre -= p_prev; // the update not yet in the tables
                    const double pos = rootA * uk - pre;
                    const double mass = (c_stale && ord_prev == o) ? c_mass - p_prev : c_mass;
                    const double *sub = sub_pref + b * BUFN;
                    bool safe = !conflict && pos > eps && pos < mass - eps;
                    // 32-way compare against the running sums of the nodes five levels down,
                    // then ONE speculative round over the remaining levels
                    int blk = __popc(__ballot_sync(0xffffffffu, pos >= c_qb)) - 1;
                    blk = blk < 0 ? 0 : blk;
                    const double lo = sub[O_QB + blk], hi = sub[O_QB + blk + 1];
                    double x = pos - lo;
                    safe = safe && (x > eps) && (hi - pos > eps);
                    int r = 32 + blk;
                    spec_round_margin<R2>(sub, r, x, safe, eps, lane);
                    const double pr = sub[r];
                    if (safe) {
                        fast = true;
                        ord = o;
                        rel = r;
                        prio = pr;
                        nfast++;
                    }
                }
                int node;
                if (!fast) {
                    // ---- slow path: the reference's arithmetic on the exact tree
                    nslow++;
                    while (ld_acquire_smem(&flags[F_ASC]) < k) {
                    }
                    // the ascent warp keeps level 12 exact; levels 11..0 = fl(left + right)
                    for (int lv = T - 2; lv >= 0; lv--) {
                        const int wdt = 1 << lv;
                        for (int i = lane; i < wdt; i += 32)
                            etop[wdt + i] = __dadd_rn(etop[2 * (wdt + i)], etop[2 * (wdt + i) + 1]);
                        __syncwarp();
                    }
                    double pos = __dmul_rn(etop[1], uk); // np.random.uniform(0.0, root), :302
                    node = older;
                    {
                        const double left = etop[older];
                        if (!(pos < left)) {
                            pos = __dsub_rn(pos, left);
                            node = older ^ 1;
                        }
                    }
                    spec_descend<T - 2>(etop, node, pos, lane); // level 1 -> 12
                    const unsigned unode = (unsigned)node;
#pragma unroll
                    for (int it = 0; it < NIT; it++) {
                        int q = lane + 32 * it;
                        q = q < 1 ? 1 : (q > PAIRS ? PAIRS : q);
                        const int dq = 31 - __clz(q);
                        reinterpret_cast<double2 *>(sub_own)[q] =
                            ld_tree_pair(sum2 + ((unode << dq) + (unsigned)(q - (1 << dq))), pol);
                    }
                    __syncwarp();
                    rel = 1;
                    spec_descend<D>(sub_own, rel, pos, lane);
                    prio = sub_own[rel];
                    ord = (node - NTOP) ^ oflip;
                } else {
                    node = NTOP + (ord ^ oflip);
                }
                const long long tm2 = V6_CLK();
                // room in the ascent queue: Q entries, checked every fourth draw
                if ((k & 3) == 0)
                    while (ld_acquire_smem(&flags[F_ASCR]) < k - Q + 4) {
                    }
                const long long tm3 = V6_CLK();
                rootA = rootA - prio;
                // ---- loads first: this draw's table entries
                const int base = ord & ~63, within = ord & 63, bk = ord >> 6;
                const double t_m = mtab[ord];
                const double t_l0 = plo[base + lane], t_l1 = plo[base + lane + 32];
                const double t_h0 = phi[lane], t_h1 = phi[lane + 32];
                // ---- then the stores: ascent queue, publisher ring, approximate tables
                const long long tm4 = V6_CLK();
                if (lane == 0) {
                    const unsigned leafnode = ((unsigned)node << D) + (unsigned)(rel - (1 << D));
                    DrawEnt e;
                    e.slot = (int)(leafnode - (unsigned)a.nslots);
                    e.buf = fast ? b : NBUF;
                    e.prio = prio;
                    *reinterpret_cast<int4 *>(&ring[k % RING]) = *reinterpret_cast<int4 *>(&e);
                    lastd[ord] = (unsigned short)(k + 1);
                    mtab[ord] = t_m - prio;
                    if ((k & 3) == 3) s_misc[0] = rootA; // the scouts' estimate tolerates the lag
                }
                if (lane > within) plo[base + lane] = t_l0 - prio;
                if (lane + 32 > within) plo[base + lane + 32] = t_l1 - prio;
                if (lane > bk) phi[lane] = t_h0 - prio;
                if (lane + 32 > bk) phi[lane + 32] = t_h1 - prio;
                ord_prev = ord;
                p_prev = prio;
                __syncwarp();
                // consumers read what LANE 0 stored above (queue, ring) after this flag; one
                // thread's shared-memory stores are performed in order, so a plain store does
                // what st.release did without the MEMBAR
                if (lane == 0)
                    asm volatile("st.volatile.shared.b32 [%0], %1;" ::"r"(smem_u32(&flags[F_MAIN])),
                                 "r"(k + 1)
                                 : "memory");
                const long long tm5 = V6_CLK();
                c_ready += tm1 - tm0;
                c_decide += tm2 - tm1;
                c_queue += tm3 - tm2;
                c_loads += tm4 - tm3;
                c_stores += tm5 - tm4;
            }
        }
        if (a.dbg_cycles && lane == 0) {
            a.dbg_cycles[0] = c_ready;
            a.dbg_cycles[1] = c_decide;
            a.dbg_cycles[2] = c_queue;
            a.dbg_cycles[3] = c_loads;
            a.dbg_cycles[4] = c_stores;
        }
        if (lane == 0) a.st->pad = (nfast & 0xffff) | (nslow << 16); // fast draws, slow draws
    } else if (warp == V6_W_ASC) {
        // --------------- ascent: _write(ix, 0.0) on the exact tree ---------------
        long long c_await = 0, c_awork = 0;
        for (int k = 0; k < a.n; k++) {
            const long long ta0 = V6_CLK();
            while (ld_acquire_smem(&flags[F_MAIN]) <= k) __nanosleep(20);
            const long long ta1 = V6_CLK();
            const int4 ev = *reinterpret_cast<const int4 *>(&ring[k % RING]);
            const unsigned lfn = (unsigned)a.nslots + (unsigned)ev.x; // heap index of the leaf
            const int node = (int)(lfn >> D);
            const int rel = NLEAF + (int)(lfn & (NLEAF - 1));
            const int bid = ev.y;
            const double *sub = bid < NBUF ? sub_pref + bid * BUFN : sub_own;
            const unsigned unode = (unsigned)node;
            // Only the D levels below the shared-memory top are re-reduced per draw.  Every
            // node above is fl(left + right) of its children at all times, so levels 11..0 of
            // the exact top are a pure function of level 12: they are recomputed once when
            // the batch ends (and before a slow-path draw needs them) -- half the chain,
            // half the instructions of the warp that bounds the pipeline.
            double sib[D];
#pragma unroll
            for (int j = 0; j < D; j++) sib[j] = sub[(rel >> j) ^ 1];
            const unsigned leafnode = (unode << D) + (unsigned)(rel - (1 << D));
            double v = 0.0;
            if (lane == 0) st_tree(a.sum + leafnode, 0.0, pol);
#pragma unroll
            for (int j = 0; j < D; j++) {
                v = __dadd_rn(v, sib[j]);
                if (lane == 0) {
                    if (j + 1 < D)
                        st_tree(a.sum + (leafnode >> (j + 1)), v, pol); // heap parent chain
                    else
                        etop[node] = v;
                }
            }
            __syncwarp();
            if (lane == 0) {
                // inputs consumed: a plain store ordered after the loads that fed the chain
                *reinterpret_cast<volatile int *>(&flags[F_ASCR]) = k + 1;
                // visibility of the global stores: every ASC_BATCH draws, and whenever
                // the main warp has nothing more queued (it may be waiting for us)
                if ((k + 1) % ASC_BATCH == 0 || k + 1 == a.n ||
                    *reinterpret_cast<volatile int *>(&flags[F_MAIN]) == k + 1) {
                    // the scouts read the bottom levels with the bulk-copy engine (async proxy)
                    asm volatile("fence.proxy.async;" ::: "memory");
                    st_release_smem(&flags[F_ASC], k + 1);
                }
            }
            __syncwarp();
            c_await += ta1 - ta0;
            c_awork += V6_CLK() - ta1;
        }
        if (a.dbg_cycles && lane == 0) {
            a.dbg_cycles[16] = c_await;
            a.dbg_cycles[17] = c_awork;
        }
    } else if (warp == V6_W_PUB) {
        // ----------------------------- publisher -----------------------------
        double total = 0.0, mroot = 0.0, bmin = INFINITY;
        const double len = (double)(a.st->napp - npop);
        for (int k0 = 0; k0 < a.n; k0 += CHUNK) {
            const int kend = (a.n - k0 < CHUNK) ? a.n : k0 + CHUNK;
            while (ld_acquire_smem(&flags[F_MAIN]) < kend) __nanosleep(200);
            if (k0 == 0) {
                total = s_misc[1];
                mroot = s_misc[2];
            }
            const int k = k0 + lane;
            if (k < kend) {
                const long long slot = ring[k % RING].slot;
                const double prio = ring[k % RING].prio;
                a.slots_out[k] = (int32_t)slot;
                a.prio_out[k] = prio;
                if (a.index_out) a.index_out[k] = (slot - npop) & mask;
                if (a.prio_user) a.prio_user[k] = prio;
                const double p = prio / total;
                if (a.prob) a.prob[k] = p;
                bmin = fmin(bmin, p);
                if (a.weight && a.norm != B2RL_NORM_BATCH)
                    a.weight[k] = is_weight(p, mroot / total, len, a.beta, a.norm);
            }
            __syncwarp();
            if (lane == 0) {
                if (a.ready) st_release_gpu(a.ready, a.seq_base | (unsigned long long)kend);
                st_release_smem(&flags[F_PUB], kend);
            }
            __syncwarp();
        }
        if (a.weight && a.norm == B2RL_NORM_BATCH) {
            for (int o = 16; o > 0; o >>= 1) bmin = fmin(bmin, __shfl_xor_sync(0xffffffffu, bmin, o));
            for (int k = lane; k < a.n; k += 32)
                a.weight[k] = is_weight(a.prio_out[k] / total, bmin, len, a.beta, a.norm);
        }
    }
    __syncthreads();
    // levels 11..0 of the exact top from level 12 (see the ascent warp)
    for (int lv = T - 2; lv >= 0; lv--) {
        const int wdt = 1 << lv;
        for (int i = threadIdx.x; i < wdt; i += blockDim.x)
            etop[wdt + i] = __dadd_rn(etop[2 * (wdt + i)], etop[2 * (wdt + i) + 1]);
        __syncthreads();
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
        for (int c = 0; c < 4; c++)
            bulk_s2g(a.sum + c * (TOPN / 4), etop + c * (TOPN / 4), TOPN * 2);
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    }
}
