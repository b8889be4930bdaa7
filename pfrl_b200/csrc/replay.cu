// replay.cu -- handle lifetime, part ring, experience append (+ eviction) and
// the level-synchronous tree repair used by append.
//
// Replaces (reference, pure Python):
//   pfrl/collections/prioritized.py:39-54   PrioritizedBuffer.append/popleft
//   pfrl/collections/prioritized.py:154-242 _write / TreeQueue.append/popleft
//   pfrl/collections/random_access_queue.py:80-98
//
// Data layout in HBM (see DESIGN.md): a ring of 2P leaf/record slots
// (P = pow2 >= capacity, slot = absolute index mod 2P) and two dense fp64
// heaps over those leaves.  Every heap node is a pure function of the leaves
// below it (`left + right`, `min(left, right)`, empty = 0.0 / +inf), which is
// bit-identical to the reference's sliding-window nested-list tree; so a
// batch of appends/evictions is: write the leaves, then recompute the touched
// ancestors level by level.
#include <math.h>
#include <stdarg.h>
#include <stdlib.h>

#include <algorithm>
#include <atomic>
#include <new>

#include "tree_dev.cuh"

// ---------------------------------------------------------------------------
static thread_local char g_err[512] = "";

void b2rl_set_error(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

unsigned b2rl_next_ticket()
{
    static std::atomic<unsigned> t{0};
    return t.fetch_add(1, std::memory_order_relaxed) % B2RL_N_TICKETS;
}

extern "C" const char *b2rl_last_error(void) { return g_err; }
extern "C" const char *b2rl_version(void) { return "b2rl 0.1 sm_90a"; }

// ---------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------
__global__ void k_fill_f64(double *p, long long n, double v)
{
    long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    long long stride = (long long)gridDim.x * blockDim.x;
    for (; i < n; i += stride) p[i] = v;
}

__global__ void k_fill_i32(int32_t *p, long long n, int32_t v)
{
    long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    long long stride = (long long)gridDim.x * blockDim.x;
    for (; i < n; i += stride) p[i] = v;
}

__global__ void k_init_state(B2rlDevState *st)
{
    st->napp = 0;
    st->npop = 0;
    st->max_priority = 1.0; // initial_max_priority, collections/prioritized.py:26
    st->last_total = 0.0;
    st->last_min = INFINITY;
    st->last_n = 0;
    st->pad = 0;
}

struct AppendArgs {
    // destination
    int32_t *state_parts, *next_parts;
    uint8_t *action;
    double *rewards;
    uint8_t *len, *terminal;
    double *sum, *mn;
    const B2rlDevState *st;
    // source (device-visible)
    const int32_t *s_state, *s_next;
    const uint8_t *s_action;
    const double *s_rewards;
    const uint8_t *s_len, *s_term;
    const double *s_prio; // may be null
    long long n, capacity, nslots;
    int stack, n_step, action_bytes, prioritized;
};

// One thread per new experience (payload + leaf), one thread per evicted leaf.
__global__ void k_append_write(AppendArgs a)
{
    const long long napp = a.st->napp, npop = a.st->npop;
    const long long mask = a.nslots - 1;
    long long evict = (napp - npop + a.n) - a.capacity;
    if (evict < 0) evict = 0;
    long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (j < a.n) {
        const long long slot = (napp + j) & mask;
        for (int p = 0; p < a.stack; p++) {
            a.state_parts[slot * a.stack + p] = a.s_state[j * a.stack + p];
            a.next_parts[slot * a.stack + p] = a.s_next[j * a.stack + p];
        }
        for (int b = 0; b < a.action_bytes; b++)
            a.action[slot * a.action_bytes + b] = a.s_action[j * a.action_bytes + b];
        for (int r = 0; r < a.n_step; r++)
            a.rewards[slot * a.n_step + r] = a.s_rewards[j * a.n_step + r];
        a.len[slot] = a.s_len[j];
        a.terminal[slot] = a.s_term[j];
        if (a.prioritized) {
            // priority None -> current max_priority (collections/prioritized.py:42-44)
            const double pr = a.s_prio ? a.s_prio[j] : a.st->max_priority;
            a.sum[a.nslots + slot] = pr;
            a.mn[a.nslots + slot] = pr;
        }
    }
    if (a.prioritized && j < evict) {
        // popleft: _write(0, None) (collections/prioritized.py:227)
        const long long slot = (npop + j) & mask;
        a.sum[a.nslots + slot] = 0.0;
        a.mn[a.nslots + slot] = INFINITY;
    }
}

// Recompute every node of one heap level in [lo, hi] (inclusive) from its
// children.  Multi-CTA, used while the touched range is wide (bulk loads).
__global__ void k_tree_level(double *sum, double *mn, long long lo, long long hi)
{
    long long n = lo + blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (n <= hi) {
        const double2 s = *reinterpret_cast<const double2 *>(sum + 2 * n);
        const double2 m = *reinterpret_cast<const double2 *>(mn + 2 * n);
        sum[n] = s.x + s.y;
        mn[n] = fmin(m.x, m.y);
    }
}

struct FixArgs {
    double *sum, *mn;
    B2rlDevState *st;
    long long lo[4], hi[4]; // node ranges (inclusive) at the level ABOVE which we start
    int nranges;
    int start_level; // level of lo/hi; parents at start_level-1 are recomputed first
    int levels;      // leaves live at heap level `levels`
    long long bump_n; // counters: napp += bump_n; npop = max(npop, napp - capacity)
    long long capacity;
};

// Single CTA: walk the remaining levels with a block barrier between levels,
// then bump the counters.
__global__ void __launch_bounds__(1024) k_tree_fix_small(FixArgs a)
{
    long long lo[4], hi[4];
    for (int r = 0; r < a.nranges; r++) { lo[r] = a.lo[r]; hi[r] = a.hi[r]; }
    // narrow ranges, level by level (global round trip + barrier each) ...
    const int topl = a.levels < 10 ? a.levels : 10;
    int level = a.start_level;
    for (; level > topl; level--) {
        for (int r = 0; r < a.nranges; r++) {
            lo[r] >>= 1;
            hi[r] >>= 1;
            for (long long n = lo[r] + threadIdx.x; n <= hi[r]; n += blockDim.x) {
                a.sum[n] = a.sum[2 * n] + a.sum[2 * n + 1];
                a.mn[n] = fmin(a.mn[2 * n], a.mn[2 * n + 1]);
            }
        }
        __syncthreads();
    }
    // ... then the top `topl` levels entirely in shared memory
    if (a.nranges > 0) rebuild_top_levels(a.sum, a.mn, topl);
    if (threadIdx.x == 0 && a.bump_n > 0) {
        long long napp = a.st->napp + a.bump_n;
        long long npop = a.st->npop;
        if (napp - npop > a.capacity) npop = napp - a.capacity;
        a.st->napp = napp;
        a.st->npop = npop;
    }
}

// ---------------------------------------------------------------------------
// staging
// ---------------------------------------------------------------------------
int b2rl_stage_acquire(b2rl_replay *h, size_t bytes)
{
    if (h->stage_busy) {
        B2RL_CUDA(cudaEventSynchronize(h->stage_ev));
        h->stage_busy = false;
    }
    if (bytes > h->stage_bytes) {
        size_t nb = std::max(bytes, h->stage_bytes * 2);
        nb = (nb + 4095) & ~size_t(4095);
        if (h->pin) cudaFreeHost(h->pin);
        if (h->stage) cudaFree(h->stage);
        h->pin = nullptr;
        h->stage = nullptr;
        h->stage_bytes = 0;
        B2RL_CUDA(cudaMallocHost((void **)&h->pin, nb));
        B2RL_CUDA(cudaMalloc((void **)&h->stage, nb));
        h->stage_bytes = nb;
    }
    return B2RL_OK;
}

int b2rl_stage_release(b2rl_replay *h, cudaStream_t s)
{
    B2RL_CUDA(cudaEventRecord(h->stage_ev, s));
    h->stage_busy = true;
    return B2RL_OK;
}

// ---------------------------------------------------------------------------
// create / destroy
// ---------------------------------------------------------------------------
template <typename T>
static int dev_alloc(b2rl_replay *h, T **p, size_t count)
{
    size_t bytes = count * sizeof(T);
    if (bytes == 0) bytes = 16;
    B2RL_CUDA(cudaMalloc((void **)p, bytes));
    h->device_bytes += (int64_t)bytes;
    return B2RL_OK;
}

static int create_impl(b2rl_replay *h)
{
    const b2rl_replay_config &c = h->cfg;
    B2RL_CUDA(cudaSetDevice(c.device));
    TRY(dev_alloc(h, &h->parts, (size_t)c.part_capacity * c.part_bytes));
    TRY(dev_alloc(h, &h->state_parts, (size_t)h->nslots * c.stack));
    TRY(dev_alloc(h, &h->next_parts, (size_t)h->nslots * c.stack));
    TRY(dev_alloc(h, &h->action, (size_t)h->nslots * c.action_bytes));
    TRY(dev_alloc(h, &h->rewards, (size_t)h->nslots * c.n_step));
    TRY(dev_alloc(h, &h->len, (size_t)h->nslots));
    TRY(dev_alloc(h, &h->terminal, (size_t)h->nslots));
    TRY(dev_alloc(h, &h->st, 1));
    TRY(dev_alloc(h, &h->last_slots, (size_t)c.max_batch));
    TRY(dev_alloc(h, &h->last_prio, (size_t)c.max_batch));
    TRY(dev_alloc(h, &h->new_prio, (size_t)c.max_batch));
    B2RL_CUDA(cudaMemset(h->len, 0, (size_t)h->nslots));
    B2RL_CUDA(cudaMemset(h->terminal, 0, (size_t)h->nslots));
    k_init_state<<<1, 1>>>(h->st);
    if (c.prioritized) {
        TRY(dev_alloc(h, &h->sum, (size_t)2 * h->nslots));
        TRY(dev_alloc(h, &h->mn, (size_t)2 * h->nslots));
        TRY(dev_alloc(h, &h->winner, (size_t)h->nslots));
        B2RL_CUDA(cudaMemset(h->sum, 0, sizeof(double) * 2 * (size_t)h->nslots));
        k_fill_f64<<<1024, 256>>>(h->mn, 2 * h->nslots, INFINITY);
        k_fill_i32<<<1024, 256>>>(h->winner, h->nslots, -1);
    }
    // [0] draws-ready counter of the fused step, [1] write-back-done stamp, [2] arrival counter
    B2RL_CUDA(cudaMalloc((void **)&h->ready_dev, 128));
    B2RL_CUDA(cudaMemset(h->ready_dev, 0, 128));
    B2RL_CUDA(cudaMalloc((void **)&h->times_dev, 8 * (8 + 256 + 32)));
    B2RL_CUDA(cudaMemset(h->times_dev, 0, 8 * (8 + 256 + 32)));
    h->device_bytes += 128 + 8 * (8 + 256 + 32);
    B2RL_CUDA(cudaEventCreateWithFlags(&h->stage_ev, cudaEventDisableTiming));
    B2RL_CUDA(cudaGetLastError());
    B2RL_CUDA(cudaDeviceSynchronize());
    return B2RL_OK;
}

extern "C" int b2rl_replay_create(const b2rl_replay_config *cfg, b2rl_replay **out)
{
    B2RL_REQUIRE(cfg && out, B2RL_ERR_INVALID, "null argument");
    B2RL_REQUIRE(cfg->capacity > 0 && cfg->capacity <= (int64_t(1) << 30),
                 B2RL_ERR_INVALID, "capacity must be in 1..2^30");
    B2RL_REQUIRE(cfg->stack >= 1 && cfg->stack <= 8, B2RL_ERR_INVALID, "stack must be 1..8");
    B2RL_REQUIRE(cfg->n_step >= 1 && cfg->n_step <= 8, B2RL_ERR_INVALID, "n_step must be 1..8");
    B2RL_REQUIRE(cfg->part_bytes > 0 && cfg->part_bytes % 16 == 0, B2RL_ERR_INVALID,
                 "part_bytes must be a positive multiple of 16");
    B2RL_REQUIRE(cfg->part_capacity > 0, B2RL_ERR_INVALID, "part_capacity must be > 0");
    B2RL_REQUIRE(cfg->action_bytes > 0 && cfg->action_bytes <= 256, B2RL_ERR_INVALID,
                 "action_bytes must be 1..256");
    B2RL_REQUIRE(cfg->max_batch > 0 && cfg->max_batch <= 65536, B2RL_ERR_INVALID,
                 "max_batch must be 1..65536");
    if (cfg->prioritized)
        B2RL_REQUIRE(cfg->capacity <= (int64_t(1) << 22), B2RL_ERR_INVALID,
                     "prioritized capacity is limited to 2^22 experiences in this build");
    b2rl_replay *h = new (std::nothrow) b2rl_replay();
    B2RL_REQUIRE(h, B2RL_ERR_NOMEM, "out of host memory");
    memset(h, 0, sizeof(*h));
    h->cfg = *cfg;
    int64_t P = 1;
    while (P < cfg->capacity) P <<= 1;
    h->P = P;
    h->nslots = 2 * P;
    h->levels = b2rl_ilog2(h->nslots);
    int rc = create_impl(h);
    if (rc != B2RL_OK) {
        b2rl_replay_destroy(h);
        return rc;
    }
    *out = h;
    return B2RL_OK;
}

extern "C" int b2rl_replay_destroy(b2rl_replay *h)
{
    if (!h) return B2RL_OK;
    cudaSetDevice(h->cfg.device);
    cudaDeviceSynchronize();
    void *ptrs[] = {h->parts, h->state_parts, h->next_parts, h->action, h->rewards,
                    h->len, h->terminal, h->sum, h->mn, h->st, h->last_slots,
                    h->last_prio, h->new_prio, h->winner, h->stage};
    for (void *p : ptrs)
        if (p) cudaFree(p);
    if (h->pin) cudaFreeHost(h->pin);
    if (h->stage_ev) cudaEventDestroy(h->stage_ev);
    if (h->ready_dev) cudaFree(h->ready_dev);
    if (h->times_dev) cudaFree(h->times_dev);
    if (h->u_ring_dev) cudaFree(h->u_ring_dev);
    if (h->u_ring_pin) cudaFreeHost(h->u_ring_pin);
    for (int i = 0; i < B2RL_U_RING; i++)
        if (h->u_ev[i]) cudaEventDestroy(h->u_ev[i]);
    delete h;
    return B2RL_OK;
}

extern "C" int64_t b2rl_replay_len(const b2rl_replay *h) { return h->napp - h->npop; }
extern "C" int64_t b2rl_replay_napp(const b2rl_replay *h) { return h->napp; }
extern "C" int64_t b2rl_replay_npop(const b2rl_replay *h) { return h->npop; }
extern "C" int64_t b2rl_replay_device_bytes(const b2rl_replay *h) { return h->device_bytes; }

// ---------------------------------------------------------------------------
// parts
// ---------------------------------------------------------------------------
extern "C" int b2rl_replay_put_parts(b2rl_replay *h, const void *src, int src_on_device,
                                     int64_t n, int32_t *slots_out_host, void *stream)
{
    B2RL_REQUIRE(h && src && n >= 0, B2RL_ERR_INVALID, "bad argument");
    B2RL_REQUIRE(n <= h->cfg.part_capacity, B2RL_ERR_RANGE,
                 "put_parts: %lld parts exceed the ring (%lld)", (long long)n,
                 (long long)h->cfg.part_capacity);
    if (n == 0) return B2RL_OK;
    cudaStream_t s = (cudaStream_t)stream;
    B2RL_CUDA(cudaSetDevice(h->cfg.device));
    const size_t pb = (size_t)h->cfg.part_bytes;
    const int64_t cap = h->cfg.part_capacity;
    const uint8_t *from = (const uint8_t *)src;
    if (!src_on_device) {
        TRY(b2rl_stage_acquire(h, (size_t)n * pb));
        memcpy(h->pin, src, (size_t)n * pb);
        from = h->pin;
    }
    int64_t first = h->part_head % cap;
    int64_t run1 = std::min<int64_t>(n, cap - first);
    cudaMemcpyKind kind = src_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    B2RL_CUDA(cudaMemcpyAsync(h->parts + (size_t)first * pb, from, (size_t)run1 * pb, kind, s));
    if (run1 < n)
        B2RL_CUDA(cudaMemcpyAsync(h->parts, from + (size_t)run1 * pb, (size_t)(n - run1) * pb,
                                  kind, s));
    if (!src_on_device) TRY(b2rl_stage_release(h, s));
    if (slots_out_host)
        for (int64_t i = 0; i < n; i++) slots_out_host[i] = (int32_t)((h->part_head + i) % cap);
    h->part_head += n;
    return B2RL_OK;
}

// ---------------------------------------------------------------------------
// tree repair over up to 4 contiguous leaf-node ranges
// ---------------------------------------------------------------------------
int b2rl_launch_tree_fix(b2rl_replay *h, int nranges, long long *lo, long long *hi,
                         long long bump_n, cudaStream_t s)
{
    if (h->cfg.prioritized && nranges > 0) {
        // small appends (one vector-env step): path-wise repair on up to 128 SMs instead
        // of a level-synchronous walk on one (42 us -> a few us)
        long long total = 0, first[4], cnt[4];
        for (int r = 0; r < nranges; r++) {
            first[r] = lo[r] - h->nslots;
            cnt[r] = hi[r] - lo[r] + 1;
            total += cnt[r];
        }
        if (total <= UPD_MAX) return b2rl_launch_repair_multi(h, nranges, first, cnt, bump_n, s);
    }
    int level = h->levels; // lo/hi are leaf-level node indices
    if (h->cfg.prioritized) {
        // wide phase: one multi-CTA launch per level and range
        for (;;) {
            long long widest = 0;
            for (int r = 0; r < nranges; r++) widest = std::max(widest, hi[r] - lo[r] + 1);
            if (widest <= 16384 || level == 0) break;
            for (int r = 0; r < nranges; r++) {
                lo[r] >>= 1;
                hi[r] >>= 1;
                long long cnt = hi[r] - lo[r] + 1;
                k_tree_level<<<(unsigned)((cnt + 255) / 256), 256, 0, s>>>(h->sum, h->mn, lo[r], hi[r]);
            }
            level--;
        }
    } else {
        nranges = 0;
    }
    FixArgs a;
    a.sum = h->sum;
    a.mn = h->mn;
    a.st = h->st;
    a.nranges = nranges;
    for (int r = 0; r < nranges; r++) { a.lo[r] = lo[r]; a.hi[r] = hi[r]; }
    a.start_level = nranges ? level : 0;
    a.levels = h->levels;
    a.bump_n = bump_n;
    a.capacity = h->cfg.capacity;
    k_tree_fix_small<<<1, 1024, 0, s>>>(a);
    B2RL_CUDA(cudaGetLastError());
    return B2RL_OK;
}

// split the slot interval [first, first+count) of the ring into <= 2 node ranges
static int ring_ranges(const b2rl_replay *h, long long first_abs, long long count,
                       long long *lo, long long *hi)
{
    if (count <= 0) return 0;
    const long long ns = h->nslots;
    long long s0 = first_abs & (ns - 1);
    if (count >= ns) { lo[0] = ns; hi[0] = 2 * ns - 1; return 1; }
    long long run1 = std::min(count, ns - s0);
    lo[0] = ns + s0;
    hi[0] = ns + s0 + run1 - 1;
    if (run1 == count) return 1;
    lo[1] = ns;
    hi[1] = ns + (count - run1) - 1;
    return 2;
}

extern "C" int b2rl_replay_append(b2rl_replay *h, const b2rl_experiences *e, int64_t n,
                                  int on_device, void *stream)
{
    B2RL_REQUIRE(h && e, B2RL_ERR_INVALID, "null argument");
    B2RL_REQUIRE(n >= 0 && n <= h->cfg.capacity, B2RL_ERR_RANGE,
                 "append: n=%lld must be in 0..capacity", (long long)n);
    if (n == 0) return B2RL_OK;
    B2RL_REQUIRE(e->state_parts && e->next_parts && e->action && e->rewards && e->len &&
                     e->terminal, B2RL_ERR_INVALID, "append: null array");
    cudaStream_t s = (cudaStream_t)stream;
    B2RL_CUDA(cudaSetDevice(h->cfg.device));
    const b2rl_replay_config &c = h->cfg;
    // a deferred write-back precedes the append: the new leaves take the
    // max_priority it may raise (collections/prioritized.py:42-44,114)
    TRY(b2rl_flush_pending(h, s));

    AppendArgs a;
    a.state_parts = h->state_parts;
    a.next_parts = h->next_parts;
    a.action = h->action;
    a.rewards = h->rewards;
    a.len = h->len;
    a.terminal = h->terminal;
    a.sum = h->sum;
    a.mn = h->mn;
    a.st = h->st;
    a.n = n;
    a.capacity = c.capacity;
    a.nslots = h->nslots;
    a.stack = c.stack;
    a.n_step = c.n_step;
    a.action_bytes = c.action_bytes;
    a.prioritized = c.prioritized;

    if (on_device) {
        a.s_state = e->state_parts;
        a.s_next = e->next_parts;
        a.s_action = (const uint8_t *)e->action;
        a.s_rewards = e->rewards;
        a.s_len = e->len;
        a.s_term = e->terminal;
        a.s_prio = e->priority;
    } else {
        // pack the arrays into the pinned buffer, one async copy
        auto al = [](size_t x) { return (x + 15) & ~size_t(15); };
        size_t o_state = 0;
        size_t o_next = o_state + al((size_t)n * c.stack * 4);
        size_t o_act = o_next + al((size_t)n * c.stack * 4);
        size_t o_rew = o_act + al((size_t)n * c.action_bytes);
        size_t o_len = o_rew + al((size_t)n * c.n_step * 8);
        size_t o_term = o_len + al((size_t)n);
        size_t o_prio = o_term + al((size_t)n);
        size_t total = o_prio + al((size_t)n * 8);
        TRY(b2rl_stage_acquire(h, total));
        memcpy(h->pin + o_state, e->state_parts, (size_t)n * c.stack * 4);
        memcpy(h->pin + o_next, e->next_parts, (size_t)n * c.stack * 4);
        memcpy(h->pin + o_act, e->action, (size_t)n * c.action_bytes);
        memcpy(h->pin + o_rew, e->rewards, (size_t)n * c.n_step * 8);
        memcpy(h->pin + o_len, e->len, (size_t)n);
        memcpy(h->pin + o_term, e->terminal, (size_t)n);
        if (e->priority) {
            for (int64_t i = 0; i < n; i++)
                B2RL_REQUIRE(e->priority[i] > 0.0, B2RL_ERR_INVALID,
                             "append: priority must be > 0");
            memcpy(h->pin + o_prio, e->priority, (size_t)n * 8);
        }
        B2RL_CUDA(cudaMemcpyAsync(h->stage, h->pin, total, cudaMemcpyHostToDevice, s));
        a.s_state = (const int32_t *)(h->stage + o_state);
        a.s_next = (const int32_t *)(h->stage + o_next);
        a.s_action = h->stage + o_act;
        a.s_rewards = (const double *)(h->stage + o_rew);
        a.s_len = h->stage + o_len;
        a.s_term = h->stage + o_term;
        a.s_prio = e->priority ? (const double *)(h->stage + o_prio) : nullptr;
    }
    k_append_write<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(a);
    B2RL_CUDA(cudaGetLastError());

    // ranges touched: appended leaves and evicted leaves (host mirrors)
    long long evict = (h->napp - h->npop + n) - c.capacity;
    if (evict < 0) evict = 0;
    long long lo[4], hi[4];
    int nr = ring_ranges(h, h->napp, n, lo, hi);
    nr += ring_ranges(h, h->npop, evict, lo + nr, hi + nr);
    TRY(b2rl_launch_tree_fix(h, nr, lo, hi, n, s));
    if (!on_device) TRY(b2rl_stage_release(h, s));
    h->napp += n;
    h->npop += evict;
    return B2RL_OK;
}
