// sampler.cu -- prioritized sampling, IS weights and priority write-back on
// the dense fp64 heaps.
//
// Replaces (reference, pure Python):
//   pfrl/collections/prioritized.py:56-116   _sample_indices_and_probabilities,
//                                            sample, set_last_priority
//   pfrl/collections/prioritized.py:245-258  _find
//   pfrl/collections/prioritized.py:294-312  SumTreeQueue.prioritized_sample
//   pfrl/replay_buffers/prioritized.py:47-66 priority_from_errors,
//                                            weights_from_probabilities
//
// EXACT mode reproduces the reference's sampled indices bit for bit: the
// draws are a dependent chain (draw k sees the root after the k-1 earlier
// hits were zeroed and their paths re-reduced), so one warp walks them in
// order.  What makes it fast is where the chain's operands live: the top
// TOP_LEVELS levels of the sum tree are staged in shared memory for the
// whole launch, and the remaining levels under the chosen top node are
// fetched by the 32 lanes in ONE round trip (each level's slice of a subtree
// is contiguous in the heap), so a draw costs one global latency, not one per
// level.
#include <math.h>
#include <stdlib.h>

#include "tree_dev.cuh"

extern __shared__ __align__(128) unsigned char smem_raw[];

__global__ void __launch_bounds__(256, 1) k_sample_exact(SampleArgs a)
{
    exact_small(a, reinterpret_cast<double *>(smem_raw));
}

// main warp + two scouts + publisher (tree_dev.cuh)
template <int D>
__global__ void __launch_bounds__(128, 1) k_sample_exact_deep(SampleArgs a)
{
    exact_deep<D>(a, reinterpret_cast<double *>(smem_raw));
}

// v6 (tree_dev.cuh): decisions on an approximate top, exact re-reduction on a trailing warp
template <int D>
__global__ void __launch_bounds__(V6_THREADS, 1) k_sample_exact_v6(SampleArgs a)
{
    exact_deep_v6<D>(a, reinterpret_cast<double *>(smem_raw));
}

__global__ void __launch_bounds__(512, 1) k_sample_parallel(SampleArgs a)
{
    sample_parallel(a, reinterpret_cast<double *>(smem_raw));
}

static cudaError_t launch_sample(const SampleArgs &a, int mode, cudaStream_t s)
{
    const SamplerChoice c = choose_sampler(mode, a.levels, a.n);
    const size_t smem = sampler_smem_bytes(c, a);
    return with_sampler(c, [&](auto d, auto kind) {
        constexpr int D = decltype(d)::value, KIND = decltype(kind)::value;
        if constexpr (KIND == SAMPLER_V6) {
            const cudaError_t e = b2rl_allow_smem<k_sample_exact_v6<D>>(smem);
            if (e != cudaSuccess) return e;
            k_sample_exact_v6<D><<<1, V6_THREADS, smem, s>>>(a);
        } else if constexpr (KIND == SAMPLER_V5) {
            const cudaError_t e = b2rl_allow_smem<k_sample_exact_deep<D>>(smem);
            if (e != cudaSuccess) return e;
            k_sample_exact_deep<D><<<1, 128, smem, s>>>(a);
        } else if constexpr (KIND == SAMPLER_SMALL) {
            const cudaError_t e = b2rl_allow_smem<k_sample_exact>(200 * 1024);
            if (e != cudaSuccess) return e;
            k_sample_exact<<<1, 256, smem, s>>>(a);
        } else {
            k_sample_parallel<<<1, 512, smem, s>>>(a);
        }
        return cudaGetLastError();
    });
}

static int v6_slow_every()
{
    static int cached = -1;
    if (cached < 0) {
        const char *e = getenv("B2RL_V6_SLOW_EVERY");
        cached = e ? atoi(e) : 0;
        if (cached < 0) cached = 0;
    }
    return cached;
}

static double v6_eps_scale()
{
    static double cached = -1.0;
    if (cached < 0.0) {
        const char *e = getenv("B2RL_V6_EPS_SCALE");
        cached = e ? atof(e) : 0.0;
        if (cached < 0.0) cached = 0.0;
    }
    return cached;
}

SampleArgs b2rl_sample_args(const b2rl_replay *h, const double *u, int n, int64_t *index_out,
                            double *prio_user)
{
    SampleArgs a{};
    a.sum = h->sum;
    a.mn = h->mn;
    a.st = h->st;
    a.u = u;
    a.n = n;
    a.levels = h->levels;
    a.nslots = h->nslots;
    a.T = h->levels + 1 < TOP_LEVELS ? h->levels + 1 : TOP_LEVELS;
    a.D = h->levels - (a.T - 1);
    a.slots_out = h->last_slots;
    a.prio_out = h->last_prio;
    a.index_out = (long long *)index_out;
    a.prio_user = prio_user;
    a.norm = B2RL_NORM_NONE;
    a.dbg_slow_every = v6_slow_every();
    a.dbg_eps_scale = v6_eps_scale();
    return a;
}

int b2rl_check_sample(const b2rl_replay *h, int n, int mode, const double *u_host, const char *fn)
{
    B2RL_REQUIRE(h->cfg.prioritized, B2RL_ERR_INVALID, "buffer has no priority trees");
    B2RL_REQUIRE(n > 0 && n <= h->cfg.max_batch, B2RL_ERR_RANGE, "%s: n=%d out of 1..max_batch=%d",
                 fn, n, h->cfg.max_batch);
    B2RL_REQUIRE(n <= h->napp - h->npop, B2RL_ERR_RANGE,
                 "%s: n=%d exceeds the %lld stored experiences", fn, n,
                 (long long)(h->napp - h->npop));
    B2RL_REQUIRE(!h->wait_priority, B2RL_ERR_PROTOCOL,
                 "%s: called again before the previous sample's priorities were set "
                 "(collections/prioritized.py:98)", fn);
    B2RL_REQUIRE(mode == B2RL_SAMPLE_EXACT || mode == B2RL_SAMPLE_PARALLEL, B2RL_ERR_INVALID,
                 "unknown sample mode %d", mode);
    if (u_host)
        for (int i = 0; i < n; i++)
            B2RL_REQUIRE(u_host[i] >= 0.0 && u_host[i] < 1.0, B2RL_ERR_INVALID,
                         "%s: u[%d]=%g not in [0,1)", fn, i, u_host[i]);
    return B2RL_OK;
}

int b2rl_upload_u(b2rl_replay *h, const double *u, int n, cudaStream_t s, const double **u_dev)
{
    const int mb = h->cfg.max_batch;
    if (!h->u_ring_dev) {
        const size_t ring = (size_t)B2RL_U_RING * mb * sizeof(double);
        B2RL_CUDA(cudaMallocHost((void **)&h->u_ring_pin, ring));
        B2RL_CUDA(cudaMalloc((void **)&h->u_ring_dev, ring));
        for (int i = 0; i < B2RL_U_RING; i++)
            B2RL_CUDA(cudaEventCreateWithFlags(&h->u_ev[i], cudaEventDisableTiming));
        h->device_bytes += (int64_t)ring;
    }
    // the slot's previous copy (B2RL_U_RING uploads ago) must have left its pinned source
    const int slot = (int)(h->u_head % B2RL_U_RING);
    if (h->u_head >= B2RL_U_RING) B2RL_CUDA(cudaEventSynchronize(h->u_ev[slot]));
    double *pin = h->u_ring_pin + (size_t)slot * mb;
    double *dev = h->u_ring_dev + (size_t)slot * mb;
    memcpy(pin, u, (size_t)n * 8);
    B2RL_CUDA(cudaMemcpyAsync(dev, pin, (size_t)n * 8, cudaMemcpyHostToDevice, s));
    B2RL_CUDA(cudaEventRecord(h->u_ev[slot], s));
    h->u_head++;
    *u_dev = dev;
    return B2RL_OK;
}

extern "C" int b2rl_per_sample(b2rl_replay *h, const double *u_host, int32_t n, int mode,
                               int64_t *index_dev, double *priority_dev, void *stream)
{
    B2RL_REQUIRE(h && u_host, B2RL_ERR_INVALID, "null argument");
    TRY(b2rl_check_sample(h, n, mode, u_host, "sample"));
    cudaStream_t s = (cudaStream_t)stream;
    B2RL_CUDA(cudaSetDevice(h->cfg.device));
    TRY(b2rl_flush_pending(h, s));
    const double *u_dev;
    TRY(b2rl_upload_u(h, u_host, n, s, &u_dev));

    // weights are a separate call on this path (b2rl_per_weights)
    B2RL_CUDA(launch_sample(b2rl_sample_args(h, u_dev, n, index_dev, priority_dev), mode, s));
    h->wait_priority = true;
    h->last_n = n;
    return B2RL_OK;
}

// ---------------------------------------------------------------------------
// importance-sampling weights
// ---------------------------------------------------------------------------
// The last sample's probabilities and weights from its priorities (a.prio_out) and the
// sum-tree and min-tree roots its sampler recorded in a.st.
__global__ void __launch_bounds__(1024) k_weights(SampleArgs a)
{
    __shared__ double red[32];
    __shared__ double s_min;
    const double total = a.st->last_total;
    double denom;
    if (a.norm == B2RL_NORM_BATCH) {
        // np.min(probabilities), replay_buffers/prioritized.py:60
        double m = INFINITY;
        for (int k = threadIdx.x; k < a.n; k += blockDim.x) m = fmin(m, a.prio_out[k] / total);
        for (int o = 16; o > 0; o >>= 1) m = fmin(m, __shfl_xor_sync(0xffffffffu, m, o));
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
        __syncthreads();
        if (threadIdx.x < 32) {
            m = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : INFINITY;
            for (int o = 16; o > 0; o >>= 1) m = fmin(m, __shfl_xor_sync(0xffffffffu, m, o));
            if (threadIdx.x == 0) s_min = m;
        }
        __syncthreads();
        denom = s_min;
    } else if (a.norm == B2RL_NORM_MEMORY) {
        denom = a.st->last_min / total; // collections/prioritized.py:60
    } else {
        denom = 0.0;
    }
    const double len = (double)(a.st->napp - a.st->npop);
    for (int k = threadIdx.x; k < a.n; k += blockDim.x) {
        const double p = a.prio_out[k] / total; // :79-82 with uniform_ratio == 0
        if (a.prob) a.prob[k] = p;
        if (a.weight) a.weight[k] = is_weight(p, denom, len, a.beta, a.norm); // :62 / :64
    }
}

extern "C" int b2rl_per_weights(b2rl_replay *h, double beta, int norm, float *weight_dev,
                                double *prob_dev, void *stream)
{
    B2RL_REQUIRE(h, B2RL_ERR_INVALID, "null handle");
    B2RL_REQUIRE(h->wait_priority && h->last_n > 0, B2RL_ERR_PROTOCOL,
                 "weights requested without a pending sample");
    B2RL_REQUIRE(norm >= 0 && norm <= 2, B2RL_ERR_INVALID, "unknown normalisation %d", norm);
    B2RL_CUDA(cudaSetDevice(h->cfg.device));
    SampleArgs a = b2rl_sample_args(h, nullptr, h->last_n, nullptr, nullptr);
    a.weight = weight_dev;
    a.prob = prob_dev;
    a.beta = beta;
    a.norm = norm;
    k_weights<<<1, 1024, 0, (cudaStream_t)stream>>>(a);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}

// ---------------------------------------------------------------------------
// priority write-back
// ---------------------------------------------------------------------------
// UpdateArgs, tree_update_multi(): tree_dev.cuh.  n <= UPD_MAX takes the sorted-path
// kernel (one global round trip); larger batches the level-synchronous one below.
// One CTA per subtree below level 7, the last one to arrive finishes the top.
__global__ void __launch_bounds__(256) k_update_multi(UpdateArgs a, unsigned long long *sync,
                                                      unsigned long long seq)
{
    tree_update_multi(a, smem_raw, sync, seq);
}

static int launch_update_multi(b2rl_replay *h, const UpdateArgs &a, cudaStream_t s)
{
    B2RL_CUDA(b2rl_allow_smem<k_update_multi>(227 * 1024)); // once per device: the maximum
    const int grid = 1 << update_split_level(h->levels);
    k_update_multi<<<grid, 256, update_multi_smem_bytes(h->levels), s>>>(
        a, h->ready_dev + 1, (unsigned long long)h->step_seq << 32);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}

__global__ void __launch_bounds__(1024) k_update(UpdateArgs a)
{
    __shared__ double red[32];
    const int tid = threadIdx.x, nt = blockDim.x;
    if (a.err)
        for (int k = tid; k < a.n; k += nt) a.new_prio[k] = priority_from_error(a, k);
    // duplicates: the reference writes in order, so the LAST occurrence wins
    for (int k = tid; k < a.n; k += nt) atomicMax(&a.winner[a.slots[k]], k);
    __syncthreads();
    double mx = 0.0;
    for (int k = tid; k < a.n; k += nt) {
        const double p = a.new_prio[k];
        mx = fmax(mx, p); // max_priority sees every value, :114
        const long long leaf = a.nslots + a.slots[k];
        if (a.winner[a.slots[k]] == k) {
            a.sum[leaf] = p;
            a.mn[leaf] = p;
        }
    }
    __syncthreads();
    // lower levels: one node per updated leaf and level, block barrier per level.
    // The leaf index stays in a register (n <= 4 * blockDim), so a level costs
    // one round trip for the four child loads instead of two dependent ones.
    const int topl = a.levels < 10 ? a.levels : 10; // levels < topl are redone in shared memory
    if (a.n <= 4 * nt) {
        long long leaf[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int k = tid + j * nt;
            leaf[j] = k < a.n ? a.nslots + a.slots[k] : -1;
        }
        for (int lv = a.levels - 1; lv >= topl; lv--) {
            const int sh = a.levels - lv;
#pragma unroll
            for (int j = 0; j < 4; j++) {
                if (leaf[j] < 0) continue;
                const long long node = leaf[j] >> sh;
                const double2 sc = *reinterpret_cast<const double2 *>(a.sum + 2 * node);
                const double2 mc = *reinterpret_cast<const double2 *>(a.mn + 2 * node);
                a.sum[node] = sc.x + sc.y;
                a.mn[node] = fmin(mc.x, mc.y);
            }
            __syncthreads();
        }
    } else {
        for (int lv = a.levels - 1; lv >= topl; lv--) {
            const int sh = a.levels - lv;
            for (int k = tid; k < a.n; k += nt) {
                const long long node = (a.nslots + a.slots[k]) >> sh;
                a.sum[node] = a.sum[2 * node] + a.sum[2 * node + 1];
                a.mn[node] = fmin(a.mn[2 * node], a.mn[2 * node + 1]);
            }
            __syncthreads();
        }
    }
    rebuild_top_levels(a.sum, a.mn, topl);
    for (int k = tid; k < a.n; k += nt) a.winner[a.slots[k]] = -1;
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((tid & 31) == 0) red[tid >> 5] = mx;
    __syncthreads();
    if (tid < 32) {
        mx = tid < (nt >> 5) ? red[tid] : 0.0;
        for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        if (tid == 0) {
            if (mx > a.st->max_priority) a.st->max_priority = mx;
            a.st->last_n = 0;
        }
    }
}

UpdateArgs b2rl_update_args(const b2rl_replay *h, int n, const void *err, int err_is_f64,
                            double alpha, double eps, double emin, double emax)
{
    UpdateArgs a{};
    a.sum = h->sum;
    a.mn = h->mn;
    a.st = h->st;
    a.slots = h->last_slots;
    a.new_prio = h->new_prio;
    a.err = err;
    a.err_is_f64 = err_is_f64;
    a.alpha = alpha;
    a.eps = eps;
    a.emin = emin;
    a.emax = emax;
    a.winner = h->winner;
    a.n = n;
    a.levels = h->levels;
    a.nslots = h->nslots;
    a.capacity = h->cfg.capacity;
    return a;
}

static int launch_update(b2rl_replay *h, int32_t n, const void *err, int err_is_f64, double alpha,
                         double eps, double emin, double emax, cudaStream_t s)
{
    const UpdateArgs a = b2rl_update_args(h, n, err, err_is_f64, alpha, eps, emin, emax);
    if (n <= UPD_MAX) {
        TRY(launch_update_multi(h, a, s));
    } else {
        k_update<<<1, 1024, 0, s>>>(a);
        B2RL_CUDA(cudaGetLastError());
    }
    h->wait_priority = false;
    h->last_n = 0;
    return B2RL_OK;
}

static int check_update(b2rl_replay *h, int32_t n)
{
    B2RL_REQUIRE(h, B2RL_ERR_INVALID, "null handle");
    B2RL_REQUIRE(h->wait_priority, B2RL_ERR_PROTOCOL,
                 "priorities set without a pending sample (collections/prioritized.py:108)");
    B2RL_REQUIRE(n == h->last_n, B2RL_ERR_RANGE,
                 "got %d priorities for a sample of %d (collections/prioritized.py:110)", n,
                 h->last_n);
    return B2RL_OK;
}

extern "C" int b2rl_per_update_priorities(b2rl_replay *h, const double *priority, int on_device,
                                          int32_t n, void *stream)
{
    TRY(check_update(h, n));
    B2RL_REQUIRE(priority, B2RL_ERR_INVALID, "null priorities");
    cudaStream_t s = (cudaStream_t)stream;
    B2RL_CUDA(cudaSetDevice(h->cfg.device));
    if (on_device) {
        B2RL_CUDA(cudaMemcpyAsync(h->new_prio, priority, (size_t)n * 8, cudaMemcpyDeviceToDevice, s));
    } else {
        for (int i = 0; i < n; i++)
            B2RL_REQUIRE(priority[i] > 0.0, B2RL_ERR_INVALID,
                         "priority[%d]=%g must be > 0 (collections/prioritized.py:109)", i,
                         priority[i]);
        TRY(b2rl_stage_acquire(h, (size_t)n * 8));
        memcpy(h->pin, priority, (size_t)n * 8);
        B2RL_CUDA(cudaMemcpyAsync(h->new_prio, h->pin, (size_t)n * 8, cudaMemcpyHostToDevice, s));
        TRY(b2rl_stage_release(h, s));
    }
    return launch_update(h, n, nullptr, 0, 0, 0, 0, 0, s);
}

extern "C" int b2rl_per_update_errors(b2rl_replay *h, const void *err_dev, int err_is_f64,
                                      int32_t n, double alpha, double eps, double error_min,
                                      double error_max, void *stream)
{
    TRY(check_update(h, n));
    B2RL_REQUIRE(err_dev, B2RL_ERR_INVALID, "null errors");
    B2RL_CUDA(cudaSetDevice(h->cfg.device));
    return launch_update(h, n, err_dev, err_is_f64, alpha, eps, error_min, error_max,
                         (cudaStream_t)stream);
}

// Ancestor repair after a small append: same multi-CTA kernel, "repair" mode.
int b2rl_launch_repair_multi(b2rl_replay *h, int nranges, const long long *first_slot,
                             const long long *count, long long bump_n, cudaStream_t s)
{
    UpdateArgs a = b2rl_update_args(h, 0, nullptr, 0, 0, 0, 0, 0);
    a.nranges = nranges;
    int total = 0;
    for (int r = 0; r < nranges; r++) {
        a.r_first[r] = (int)first_slot[r];
        a.r_count[r] = (int)count[r];
        total += (int)count[r];
    }
    a.n = total;
    a.bump_n = bump_n;
    return launch_update_multi(h, a, s);
}

// Register the write-back of launch_update's arguments without launching it: the trees are
// updated at the head of the next fused step launch (step.cu) or by the next call that reads
// or writes them, whichever comes first.
static void defer_update(b2rl_replay *h, int32_t n, const void *err, int err_is_f64, double alpha,
                         double eps, double emin, double emax)
{
    h->pending = true;
    h->pend_err = err;
    h->pend_is_f64 = err_is_f64;
    h->pend_n = n;
    h->pend_alpha = alpha;
    h->pend_eps = eps;
    h->pend_emin = emin;
    h->pend_emax = emax;
    h->wait_priority = false; // the sample is answered; the write-back is owed
    h->last_n = 0;
}

// Deferred form: register the TD errors of the last sample (defer_update).  err_dev must stay
// alive (and unchanged) until the write-back runs.
extern "C" int b2rl_per_defer_errors(b2rl_replay *h, const void *err_dev, int err_is_f64,
                                     int32_t n, double alpha, double eps, double error_min,
                                     double error_max)
{
    TRY(check_update(h, n));
    B2RL_REQUIRE(err_dev, B2RL_ERR_INVALID, "null errors");
    defer_update(h, n, err_dev, err_is_f64, alpha, eps, error_min, error_max);
    return B2RL_OK;
}

// ---------------------------------------------------------------------------
// Host TD errors (the reference's update_errors(list of Python floats),
// replay_buffers/prioritized.py:47-55,125-126): the priorities are computed HERE on the host
// with libm's pow -- the function behind CPython's float ** -- in the reference's operation
// order (max(lo, d), min(hi, d), + eps, ** alpha), so they are bit-identical to the reference's
// list comprehension; then staged to the device and either written back now or folded into
// the next fused step like b2rl_per_defer_errors.
// ---------------------------------------------------------------------------
extern "C" int b2rl_host_priority_from_errors(const double *err, int32_t n, double alpha,
                                              double eps, int has_min, double error_min,
                                              int has_max, double error_max, double *out)
{
    B2RL_REQUIRE(err && out && n >= 0, B2RL_ERR_INVALID, "host_priority_from_errors: bad argument");
    for (int32_t i = 0; i < n; i++) {
        double d = err[i];
        if (has_min) d = (d > error_min) ? d : error_min; // max(lo, d): lo unless d is larger
        if (has_max) d = (d < error_max) ? d : error_max; // min(hi, d)
        out[i] = pow(d + eps, alpha);
    }
    return B2RL_OK;
}

extern "C" int b2rl_per_update_host_errors(b2rl_replay *h, const double *err_host, int32_t n,
                                           double alpha, double eps, int has_min,
                                           double error_min, int has_max, double error_max,
                                           int defer, void *stream)
{
    TRY(check_update(h, n));
    B2RL_REQUIRE(err_host, B2RL_ERR_INVALID, "null errors");
    cudaStream_t s = (cudaStream_t)stream;
    B2RL_CUDA(cudaSetDevice(h->cfg.device));
    TRY(b2rl_stage_acquire(h, (size_t)n * 8));
    double *prio = reinterpret_cast<double *>(h->pin);
    TRY(b2rl_host_priority_from_errors(err_host, n, alpha, eps, has_min, error_min, has_max,
                                       error_max, prio));
    for (int i = 0; i < n; i++)
        B2RL_REQUIRE(prio[i] > 0.0, B2RL_ERR_INVALID,
                     "priority[%d]=%g must be > 0 (collections/prioritized.py:109)", i, prio[i]);
    B2RL_CUDA(cudaMemcpyAsync(h->new_prio, h->pin, (size_t)n * 8, cudaMemcpyHostToDevice, s));
    TRY(b2rl_stage_release(h, s));
    if (!defer) return launch_update(h, n, nullptr, 0, 0, 0, 0, 0, s);
    defer_update(h, n, nullptr, 0, 0, 0, 0, 0); // the priorities are already in new_prio
    return B2RL_OK;
}

int b2rl_flush_pending(b2rl_replay *h, cudaStream_t s)
{
    if (!h->pending) return B2RL_OK;
    h->pending = false;
    return launch_update(h, h->pend_n, h->pend_err, h->pend_is_f64, h->pend_alpha, h->pend_eps,
                         h->pend_emin, h->pend_emax, s);
}

extern "C" int b2rl_per_flush(b2rl_replay *h, void *stream)
{
    B2RL_REQUIRE(h, B2RL_ERR_INVALID, "null handle");
    B2RL_CUDA(cudaSetDevice(h->cfg.device));
    return b2rl_flush_pending(h, (cudaStream_t)stream);
}

// ---------------------------------------------------------------------------
// introspection
// ---------------------------------------------------------------------------
extern "C" int b2rl_per_get_info(b2rl_replay *h, b2rl_per_info *out, void *stream)
{
    B2RL_REQUIRE(h && out, B2RL_ERR_INVALID, "null argument");
    cudaStream_t s = (cudaStream_t)stream;
    B2RL_CUDA(cudaSetDevice(h->cfg.device));
    TRY(b2rl_flush_pending(h, s));
    B2rlDevState st;
    B2RL_CUDA(cudaMemcpyAsync(&st, h->st, sizeof(st), cudaMemcpyDeviceToHost, s));
    double roots[2] = {0.0, INFINITY};
    if (h->cfg.prioritized) {
        B2RL_CUDA(cudaMemcpyAsync(&roots[0], h->sum + 1, 8, cudaMemcpyDeviceToHost, s));
        B2RL_CUDA(cudaMemcpyAsync(&roots[1], h->mn + 1, 8, cudaMemcpyDeviceToHost, s));
    }
    B2RL_CUDA(cudaStreamSynchronize(s));
    out->total = roots[0];
    out->min = roots[1];
    out->max_priority = st.max_priority;
    out->napp = st.napp;
    out->npop = st.npop;
    out->scout_hits = st.pad;
    out->reserved = 0;
    return B2RL_OK;
}

// Checkpoint restore: PrioritizedBuffer is pickled whole, max_priority included
// (pfrl/replay_buffers/replay_buffer.py:85-94, collections/prioritized.py:32).
extern "C" int b2rl_per_set_max_priority(b2rl_replay *h, double max_priority, void *stream)
{
    B2RL_REQUIRE(h, B2RL_ERR_INVALID, "null argument");
    B2RL_REQUIRE(h->cfg.prioritized, B2RL_ERR_INVALID, "buffer has no priority trees");
    B2RL_REQUIRE(max_priority > 0.0 && max_priority < INFINITY, B2RL_ERR_RANGE,
                 "set_max_priority: value must be positive and finite");
    cudaStream_t s = (cudaStream_t)stream;
    B2RL_CUDA(cudaSetDevice(h->cfg.device));
    TRY(b2rl_flush_pending(h, s));
    B2RL_CUDA(cudaMemcpyAsync(&h->st->max_priority, &max_priority, sizeof(double),
                              cudaMemcpyHostToDevice, s));
    B2RL_CUDA(cudaStreamSynchronize(s)); // the source is a stack variable
    return B2RL_OK;
}

extern "C" int b2rl_per_read_priorities(b2rl_replay *h, int64_t first, int64_t n, double *out,
                                        void *stream)
{
    B2RL_REQUIRE(h && out, B2RL_ERR_INVALID, "null argument");
    B2RL_REQUIRE(h->cfg.prioritized, B2RL_ERR_INVALID, "buffer has no priority trees");
    B2RL_REQUIRE(first >= 0 && n >= 0 && first + n <= h->napp - h->npop, B2RL_ERR_RANGE,
                 "read_priorities: range out of bounds");
    cudaStream_t s = (cudaStream_t)stream;
    B2RL_CUDA(cudaSetDevice(h->cfg.device));
    TRY(b2rl_flush_pending(h, s));
    const int64_t mask = h->nslots - 1;
    int64_t done = 0;
    while (done < n) {
        int64_t slot = (h->npop + first + done) & mask;
        int64_t run = n - done < h->nslots - slot ? n - done : h->nslots - slot;
        B2RL_CUDA(cudaMemcpyAsync(out + done, h->sum + h->nslots + slot, (size_t)run * 8,
                                  cudaMemcpyDeviceToHost, s));
        done += run;
    }
    B2RL_CUDA(cudaStreamSynchronize(s));
    return B2RL_OK;
}

extern "C" int b2rl_per_read_tree(b2rl_replay *h, int which, int64_t first_node, int64_t n,
                                  double *out, void *stream)
{
    B2RL_REQUIRE(h && out, B2RL_ERR_INVALID, "null argument");
    B2RL_REQUIRE(h->cfg.prioritized, B2RL_ERR_INVALID, "buffer has no priority trees");
    B2RL_REQUIRE(which == 0 || which == 1, B2RL_ERR_INVALID,
                 "read_tree: which=%d must be 0 (sum) or 1 (min)", which);
    B2RL_REQUIRE(first_node >= 0 && n >= 0 && first_node + n <= 2 * h->nslots, B2RL_ERR_RANGE,
                 "read_tree: nodes [%lld, %lld) outside the heap [0, %lld)", (long long)first_node,
                 (long long)(first_node + n), (long long)(2 * h->nslots));
    cudaStream_t s = (cudaStream_t)stream;
    B2RL_CUDA(cudaSetDevice(h->cfg.device));
    TRY(b2rl_flush_pending(h, s));
    if (n > 0)
        B2RL_CUDA(cudaMemcpyAsync(out, (which ? h->mn : h->sum) + first_node, (size_t)n * 8,
                                  cudaMemcpyDeviceToHost, s));
    B2RL_CUDA(cudaStreamSynchronize(s));
    return B2RL_OK;
}
