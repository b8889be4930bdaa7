/*
 * b2rl.h -- C ABI of libb2rl.so, the H100 (sm_90a) replay / loss hot path
 * that sits behind pfrl_b200's PFRL-compatible Python classes.
 *
 * The reference (pfnet/pfrl) is pure Python and has no FFI of its own; each
 * entry point below names the reference code it replaces (file:line relative
 * to the reference root).  INTEGRATION.md shows the ctypes binding a
 * maintainer would add on the reference side.
 *
 * Conventions
 *  - every function returns 0 on success, a negative b2rl_status on error;
 *    b2rl_last_error() returns a thread-local message for the last failure.
 *  - no exceptions, no Python / torch types: plain pointers and sizes.
 *  - "dev" pointers are device pointers owned by the caller (e.g. torch
 *    tensors); they must stay alive until `stream` has passed the call.
 *    "host" pointers are read synchronously before the call returns.
 *  - `stream` is a cudaStream_t passed as void* (NULL = legacy default
 *    stream).  All work is enqueued asynchronously on it; the library never
 *    synchronises the device unless the function says so.
 *  - a handle is not thread-safe (same single-caller discipline as the
 *    reference's replay buffers).
 */
#ifndef B2RL_H
#define B2RL_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
    B2RL_OK = 0,
    B2RL_ERR_INVALID = -1,  /* bad argument */
    B2RL_ERR_CUDA = -2,     /* CUDA runtime error (see b2rl_last_error) */
    B2RL_ERR_PROTOCOL = -3, /* sample / update ordering violated
                               (asserts at collections/prioritized.py:98,108) */
    B2RL_ERR_RANGE = -4,    /* index / size out of range */
    B2RL_ERR_NOMEM = -5
} b2rl_status;

const char *b2rl_last_error(void);
/* Library / build identification, e.g. "b2rl 0.1 sm_90a". */
const char *b2rl_version(void);

/* ------------------------------------------------------------------------
 * Replay store: HBM ring of observation parts ("frames") + per-experience
 * records + (optionally) fp64 sum / min segment trees.
 *
 * Replaces: pfrl/replay_buffers/replay_buffer.py:24-80 (storage of n-step
 * experiences), pfrl/collections/random_access_queue.py:6-101,
 * pfrl/collections/prioritized.py:21-323 (PrioritizedBuffer, SumTreeQueue,
 * MinTreeQueue).
 *
 * An *observation* is `stack` parts of `part_bytes` bytes each (Atari:
 * 4 frames of 84*84 uint8; vector obs: 1 part of 4*dim bytes).  Parts are
 * shared between observations exactly like the reference's LazyFrames share
 * frame arrays (pfrl/wrappers/atari_wrappers.py:251-272).
 * An *experience* is what the reference stores as one replay element: the
 * list of 1..n_step consecutive transitions (replay_buffer.py:52-62).  Its
 * record holds: part slots of the first transition's state and of the last
 * transition's next_state, the first action, the per-step rewards, the
 * number of steps and the "any terminal" flag -- everything
 * batch_experiences (pfrl/replay_buffer.py:157-212) reads.
 * ---------------------------------------------------------------------- */
typedef struct b2rl_replay b2rl_replay;

typedef struct {
    int64_t capacity;      /* max live experiences (> 0)                     */
    int64_t part_capacity; /* slots in the part ring (>= parts kept alive)   */
    int32_t part_bytes;    /* bytes per part; multiple of 16                 */
    int32_t stack;         /* parts per observation (1..8)                   */
    int32_t n_step;        /* max transitions per experience (1..8)          */
    int32_t action_bytes;  /* bytes per action (int64 -> 8, f32[6] -> 24)    */
    int32_t prioritized;   /* 1: keep sum/min trees                          */
    int32_t device;        /* CUDA device ordinal                            */
    int32_t max_batch;     /* largest sample/update batch (<= 65536)         */
    int32_t reserved;
} b2rl_replay_config;

int b2rl_replay_create(const b2rl_replay_config *cfg, b2rl_replay **out);
int b2rl_replay_destroy(b2rl_replay *h);

/* Host mirrors of the counters (no device sync): live experiences, absolute
 * append / pop counters (collections/prioritized.py TreeQueue.length and the
 * popleft count). */
int64_t b2rl_replay_len(const b2rl_replay *h);
int64_t b2rl_replay_napp(const b2rl_replay *h);
int64_t b2rl_replay_npop(const b2rl_replay *h);
/* Bytes of HBM the handle holds. */
int64_t b2rl_replay_device_bytes(const b2rl_replay *h);

/* Copy `n` parts into the ring.  `src` is host (src_on_device = 0; staged
 * through pinned memory, asynchronous) or device memory, n * part_bytes
 * contiguous bytes.  The ring slots assigned (sequential modulo
 * part_capacity) are written to slots_out_host[n].  Replaces the implicit
 * "keep a reference to the frame ndarray" of the reference. */
int b2rl_replay_put_parts(b2rl_replay *h, const void *src, int src_on_device,
                          int64_t n, int32_t *slots_out_host, void *stream);

/* A batch of assembled experiences (structure of arrays, n entries). */
typedef struct {
    const int32_t *state_parts; /* [n][stack] part slots of exp[0].state      */
    const int32_t *next_parts;  /* [n][stack] part slots of exp[-1].next_state*/
    const void *action;         /* [n][action_bytes]                          */
    const double *rewards;      /* [n][n_step], entries >= len are ignored    */
    const uint8_t *len;         /* [n] transitions in the experience, 1..n_step */
    const uint8_t *terminal;    /* [n] any(is_state_terminal)                 */
    const double *priority;     /* [n] or NULL = current max_priority
                                   (collections/prioritized.py:42-44)         */
} b2rl_experiences;

/* Append n experiences in order, evicting the oldest when full.  Replaces
 * PrioritizedBuffer.append / popleft (collections/prioritized.py:39-54) and
 * RandomAccessQueue.append (random_access_queue.py:80-83).  Arrays are host
 * memory (on_device = 0) or device memory.  n <= capacity. */
int b2rl_replay_append(b2rl_replay *h, const b2rl_experiences *e, int64_t n,
                       int on_device, void *stream);

/* ------------------------------------------------------------------------
 * Prioritized sampling.
 * ---------------------------------------------------------------------- */
typedef enum {
    /* Bit-exact restatement of SumTreeQueue.prioritized_sample(remove=True)
     * (collections/prioritized.py:294-312): n sequential draws without
     * replacement, draw k uses pos = u[k] * root_k. */
    B2RL_SAMPLE_EXACT = 0,
    /* All n descents run concurrently on the frozen tree (sampling WITH
     * replacement, pos = u[k] * root_0).  Same marginal distribution for the
     * first draw; not index-identical to the reference. */
    B2RL_SAMPLE_PARALLEL = 1
} b2rl_sample_mode;

/* Draw n leaves.  u_host[n]: uniforms in [0,1) drawn by the caller in the
 * reference's order (numpy legacy RandomState.random_sample; see
 * np.random.uniform(0.0, root) at collections/prioritized.py:302).
 * Outputs (device, may be NULL): index_dev[n] logical indices (0 = oldest),
 * priority_dev[n] the priorities found (fp64).  The sampled leaves are
 * zeroed in the sum tree (EXACT mode) until b2rl_per_update_*; the handle
 * remembers the sampled slots.  Fails with B2RL_ERR_PROTOCOL if a previous
 * sample has not been answered (collections/prioritized.py:98). */
int b2rl_per_sample(b2rl_replay *h, const double *u_host, int32_t n, int mode,
                    int64_t *index_dev, double *priority_dev, void *stream);

typedef enum {
    B2RL_NORM_NONE = 0,  /* w = (len * prob) ** -beta                         */
    B2RL_NORM_BATCH = 1, /* w = (prob / min(prob in batch)) ** -beta          */
    B2RL_NORM_MEMORY = 2 /* w = (prob / (min_tree_root / total)) ** -beta     */
} b2rl_weight_norm;

/* Importance-sampling weights of the last sample; replaces
 * PriorityWeightError.weights_from_probabilities
 * (replay_buffers/prioritized.py:57-66) and the probability computation of
 * collections/prioritized.py:59-60,79-82.  weight_dev[n] f32 (may be NULL),
 * prob_dev[n] fp64 (may be NULL). */
int b2rl_per_weights(b2rl_replay *h, double beta, int norm, float *weight_dev,
                     double *prob_dev, void *stream);

/* Answer the last sample with new priorities (fp64, > 0; host or device).
 * Replaces PrioritizedBuffer.set_last_priority
 * (collections/prioritized.py:107-116): leaves of both trees are rewritten,
 * max_priority is raised. */
int b2rl_per_update_priorities(b2rl_replay *h, const double *priority,
                               int on_device, int32_t n, void *stream);

/* Same, from TD errors on the device (err_is_f64: 0 = float, 1 = double):
 * priority = (clip(err, error_min, error_max) + eps) ** alpha, replacing
 * priority_from_errors (replay_buffers/prioritized.py:47-55).  Set
 * error_min > error_max to disable clipping.  alpha == 0.5 uses sqrt. */
int b2rl_per_update_errors(b2rl_replay *h, const void *err_dev, int err_is_f64,
                           int32_t n, double alpha, double eps,
                           double error_min, double error_max, void *stream);

/* Copy scalar state to the host (synchronises `stream`): total priority,
 * min-tree root, max_priority, device-side napp / npop. */
typedef struct {
    double total;
    double min;
    double max_priority;
    int64_t napp;
    int64_t npop;
    int32_t scout_hits; /* draws of the last exact sample whose subtree was
                           already staged by the scout warp (diagnostic)   */
    int32_t reserved;
} b2rl_per_info;
int b2rl_per_get_info(b2rl_replay *h, b2rl_per_info *out_host, void *stream);

/* Read leaves [first, first+n) of the sum tree by logical index into
 * out_host (synchronises). Test / checkpoint helper. */
int b2rl_per_read_priorities(b2rl_replay *h, int64_t first, int64_t n,
                             double *out_host, void *stream);

/* Read heap nodes [first_node, first_node+n) of the sum tree (which = 0) or
 * the min tree (which = 1) into out_host, after any pending write-back
 * (synchronises). Node 1 is the root, the leaves of ring slots 0..2P-1 are
 * nodes 2P..4P-1, node 0 is unused. Test helper. */
int b2rl_per_read_tree(b2rl_replay *h, int which, int64_t first_node, int64_t n,
                       double *out_host, void *stream);

/* Restore max_priority when a checkpoint is loaded: the reference pickles the
 * whole PrioritizedBuffer, max_priority included (pfrl/replay_buffers/
 * replay_buffer.py:85-94; pfrl/collections/prioritized.py:32). Synchronises. */
int b2rl_per_set_max_priority(b2rl_replay *h, double max_priority, void *stream);

/* ------------------------------------------------------------------------
 * Minibatch gather; replaces batch_experiences (pfrl/replay_buffer.py:
 * 157-212) + batch_states (pfrl/utils/batch_states.py:18-36) + the H2D copy.
 * ---------------------------------------------------------------------- */
typedef enum {
    B2RL_OBS_RAW = 0,       /* copy part bytes unchanged                      */
    B2RL_OBS_U8_TO_F32 = 1  /* out = float(u8) * obs_scale  (phi = x/255)     */
} b2rl_obs_mode;

typedef struct {
    void *state;      /* [n][stack*part_bytes] bytes, or f32 [n][stack*part_bytes] */
    void *next_state; /* same layout                                          */
    void *action;     /* [n][action_bytes]                                    */
    float *reward;    /* [n] sum_i gamma^i r_i, fp64 compensated sum -> f32   */
    float *terminal;  /* [n] 1.0 if any transition terminal                   */
    float *discount;  /* [n] gamma ** len                                     */
    double *step_rewards; /* [n][n_step] raw per-step rewards (entries >= len are 0) */
    uint8_t *len;     /* [n] transitions per experience                       */
} b2rl_batch_out;

/* index_dev: n logical indices on the device, or NULL to gather the
 * experiences drawn by the last b2rl_per_sample.  gamma_pow_host[n_step+1]
 * holds gamma**i computed by the caller (CPython float pow, so the bits match
 * the reference's `gamma**i`).  Any output pointer may be NULL. */
int b2rl_replay_gather(b2rl_replay *h, const int64_t *index_dev, int32_t n,
                       const double *gamma_pow_host, int obs_mode,
                       float obs_scale, const b2rl_batch_out *out,
                       void *stream);

/* ------------------------------------------------------------------------
 * Sequence gather for recurrent (episodic) updates; replaces
 * batch_recurrent_experiences (pfrl/replay_buffer.py:219-287) + the per-episode
 * batch_states + pack_sequence (pfrl/utils/recurrent.py:249-277) + the H2D copy.
 * Store built with n_step = 1.  Sequence b is the records first[b] ..
 * first[b] + len[b] - 1 (logical indices); its step t is written at the
 * packed row  sum_{t' < t} batch_sizes[t'] + b  (pack_sequence order, time
 * major), batch_sizes[t'] = #{b : len[b] > t'}.
 * ---------------------------------------------------------------------- */
#define B2RL_SEQ_MAX_B 1024
#define B2RL_SEQ_MAX_LEAVES 8

typedef struct {
    void *state;      /* [N][stack*part_bytes] bytes, or f32 (U8_TO_F32), N = sum(len) */
    void *next_state; /* same layout                                          */
    void *action;     /* [N][action_bytes]                                    */
    float *reward;    /* [N] fp32 rounding of the stored fp64 reward          */
    float *terminal;  /* [N] 1.0 / 0.0                                        */
} b2rl_seq_out;

/* Recurrent states of the records, kept by the caller in HBM: row r of
 * `ring` holds the state (r, 0) and the next state (r, 1) of the record whose
 * absolute append index a satisfies a % ring_rows == r, flattened to
 * row_floats floats each; present[r][k] = 0 marks a stored None.  The state
 * of each sequence's FIRST record is written to the leaves: leaf i takes the
 * floats [offset[i], offset[i] + d0[i] * inner[i]) of the row as a
 * [d0, inner] block and writes it as out[i] = f32 [d0][B][inner] (zeros for
 * None), i.e. concatenate_recurrent_states of [d0, inner]-shaped entries. */
typedef struct {
    const float *ring;       /* [ring_rows][2][row_floats] */
    const uint8_t *present;  /* [ring_rows][2] */
    int64_t ring_rows;
    int32_t row_floats;
    int32_t n_leaves;
    int32_t offset[B2RL_SEQ_MAX_LEAVES], d0[B2RL_SEQ_MAX_LEAVES], inner[B2RL_SEQ_MAX_LEAVES];
    float *out_state[B2RL_SEQ_MAX_LEAVES];
    float *out_next_state[B2RL_SEQ_MAX_LEAVES];
} b2rl_seq_states;

/* first_host / len_host / end_host: B host arrays, 1 <= B <= B2RL_SEQ_MAX_B;
 * end[b] is one past the last record of the episode sequence b is cut from.
 * Requires 0 <= first[b], len[b] >= 1, first[b] + len[b] <= end[b] <= live
 * records, len non-increasing (a stable sort by length, longest first), else
 * B2RL_ERR_RANGE.  states may be NULL.  One launch, no synchronisation, no
 * allocation. */
int b2rl_replay_gather_sequences(b2rl_replay *h, const int64_t *first_host,
                                 const int32_t *len_host, const int64_t *end_host,
                                 int32_t B, int obs_mode, float obs_scale,
                                 const b2rl_seq_out *out, const b2rl_seq_states *states,
                                 void *stream);

/* ------------------------------------------------------------------------
 * Sequence gather of a recurrent PPO minibatch (or dataset pass) out of a
 * time-major rollout [T][E][...]; replaces the per-episode batch_states +
 * torch.tensor of per-transition scalars + concatenate_recurrent_states +
 * pack_sequence + H2D of _update_once_recurrent and
 * _add_log_prob_and_value_to_episodes_recurrent (pfrl/agents/ppo.py:56-107,
 * 534-606).
 *
 * table_host: int64 [first[B]][len[B]][row_off[Lmax + 1]], Lmax = len[0].
 * Sequence b is env first[b] % E, steps first[b] / E .. + len[b] - 1, so its
 * step t is the flat slot first[b] + t * E; it is written at the packed row
 * row_off[t] + b, row_off[t] = sum_b' min(len[b'], t) (pack_sequence order).
 * Requires len[b] >= 1, len non-increasing (a stable sort, longest first),
 * first[b] >= 0, first[b] / E + len[b] <= T and the row offsets to be those
 * of the lengths, else B2RL_ERR_RANGE.  B is not capped.  The table goes to
 * table_dev (caller-owned, >= table_dev_capacity int64) in one
 * cudaMemcpyAsync on `stream`: a pinned table_host must stay untouched until
 * that copy has run.
 *
 * cols[c] copies row_bytes bytes of flat slot s of src ([T*E][row_bytes]) to
 * row r of dst ([N][row_bytes], N = row_off[Lmax]).  index_out (optional)
 * receives the flat slot of every packed row.  states (optional) is a
 * b2rl_seq_states whose ring row r is the flat slot r (ring_rows >= T*E): each
 * sequence's first slot is written to out_state (side 0) / out_next_state
 * (side 1) of every leaf that has one.  One launch, no synchronisation, no
 * allocation. */
#define B2RL_ROLLOUT_MAX_COLS 8

typedef struct {
    const void *src; /* [T*E][row_bytes] */
    void *dst;       /* [N][row_bytes]   */
    int64_t row_bytes;
} b2rl_rollout_col;

int b2rl_rollout_gather_sequences(const int64_t *table_host, int64_t *table_dev,
                                  int64_t table_dev_capacity, int32_t B, int64_t T, int64_t E,
                                  const b2rl_rollout_col *cols, int32_t n_cols,
                                  int64_t *index_out, const b2rl_seq_states *states,
                                  void *stream);

/* ------------------------------------------------------------------------
 * Fused replay step: ONE persistent launch per minibatch that
 *   1. writes back the priorities of the PREVIOUS sample if its TD errors were
 *      registered with b2rl_per_defer_errors (set_last_priority,
 *      collections/prioritized.py:107-116),
 *   2. draws n leaves (b2rl_per_sample semantics) and computes their
 *      importance weights (b2rl_per_weights semantics),
 *   3. gathers the minibatch (b2rl_replay_gather semantics); the gather CTAs
 *      consume the draws 32 at a time while the sampler is still drawing.
 * Replaces the reference's update loop body around
 * pfrl/replay_buffer.py:329-356 -> pfrl/replay_buffers/prioritized.py:117-126
 * -> pfrl/replay_buffer.py:157-212.
 * ---------------------------------------------------------------------- */
typedef struct {
    int32_t n;             /* draws                                          */
    int32_t mode;          /* b2rl_sample_mode                               */
    const double *u;       /* n uniforms in [0,1), reference order           */
    int32_t u_on_device;   /* 0: host memory (copied through a pinned ring),
                              1: device memory, alive until the stream has
                              passed the call                                */
    int32_t norm;          /* b2rl_weight_norm                               */
    double beta;           /* IS exponent                                    */
    const double *gamma_pow_host; /* gamma**i, i = 0..n_step (host)          */
    int32_t obs_mode;      /* b2rl_obs_mode                                  */
    float obs_scale;
    int64_t *index_dev;    /* [n] logical indices, or NULL                   */
    double *priority_dev;  /* [n] priorities found, or NULL                  */
    float *weight_dev;     /* [n] importance weights, or NULL                */
    double *prob_dev;      /* [n] probabilities, or NULL                     */
    b2rl_batch_out out;    /* any pointer may be NULL                        */
} b2rl_step_args;

int b2rl_replay_step(b2rl_replay *h, const b2rl_step_args *args, void *stream);

/* Phase durations (ns) of the last b2rl_replay_step launch, from timestamps the
 * kernel leaves behind (synchronises `stream`): out_ns[0] deferred write-back,
 * [1] sampling (until the last draw is published), [2] gather tail (from there to the
 * exit of the last CTA), [3] the whole launch; [4..35] clock-cycle sums of the exact
 * sampler's pipeline segments when the library runs with B2RL_V6_CYCLES=1 (else 0);
 * [31..35] phases of the multi-CTA write-back in ns since CTA 0's entry: entries collected,
 * subtree stored, arrival ticket taken (all CTA 0), subtree roots loaded, completion flag
 * released (last CTA); with B2RL_WB_FINE=1 in the environment also [28..30]: CTA 0's sort /
 * unique done, siblings fetched, level loop done.  out_ns_host has 36 entries.  Measurement aid (bench.py, tools/v6_pipeline.py). */
int b2rl_step_times(b2rl_replay *h, uint64_t *out_ns_host, void *stream);

/* Answer the last sample with TD errors on the device WITHOUT launching: the
 * write-back runs at the head of the next b2rl_replay_step launch, or before
 * the next call that reads or writes the trees (append, sample, get_info, ...),
 * whichever comes first -- so every later operation sees exactly the state
 * b2rl_per_update_errors would have left.  err_dev must stay alive and
 * unchanged until then.  Same arguments as b2rl_per_update_errors. */
int b2rl_per_defer_errors(b2rl_replay *h, const void *err_dev, int err_is_f64,
                          int32_t n, double alpha, double eps,
                          double error_min, double error_max);

/* TD errors as HOST doubles (the reference's update_errors(list of Python floats),
 * pfrl/replay_buffers/prioritized.py:47-55,125-126).  The priorities
 *   (min(hi, max(lo, d)) + eps) ** alpha
 * are computed on the host with libm's pow, the function behind CPython's float **, in the
 * reference's operation order -- bit-identical to its list comprehension -- and must be > 0
 * (collections/prioritized.py:109).  has_min / has_max = 0 stand for error_min / error_max =
 * None.  defer = 0: write back now (one launch); defer = 1: fold the write-back into the
 * next b2rl_replay_step like b2rl_per_defer_errors.  b2rl_host_priority_from_errors is the
 * arithmetic alone (no device needed). */
int b2rl_host_priority_from_errors(const double *err, int32_t n, double alpha, double eps,
                                   int has_min, double error_min, int has_max,
                                   double error_max, double *out);
int b2rl_per_update_host_errors(b2rl_replay *h, const double *err_host, int32_t n,
                                double alpha, double eps, int has_min, double error_min,
                                int has_max, double error_max, int defer, void *stream);
/* Apply a deferred write-back now (no-op if none is registered). */
int b2rl_per_flush(b2rl_replay *h, void *stream);

/* ------------------------------------------------------------------------
 * Fused loss kernels (fp32, device pointers, deterministic reductions).
 * `mean` != 0: divide the batch sum by B ("mean" batch_accumulator).
 * `weights` may be NULL (uniform replay).  `scratch` is B floats.
 * ---------------------------------------------------------------------- */

/* Categorical (C51 / Rainbow) loss: projects the next-state distribution
 * next_p[B,n] through Tz = r + (1-terminal)*discount*z onto the support
 * z[n], then cross-entropy with y[B,n].  Replaces
 * _apply_categorical_projection (pfrl/agents/categorical_dqn.py:7-57) and
 * CategoricalDQN._compute_loss (:178-204).  Outputs: t_out[B,n] projected
 * target, delta_out[B] per-sample loss (the priority error), loss_out[1]. */
int b2rl_c51_loss_fwd(const float *y, const float *next_p, const float *reward,
                      const float *discount, const float *terminal,
                      const float *weights, const float *z, int32_t B,
                      int32_t n_atoms, int mean, float *t_out, float *delta_out,
                      float *scratch, float *loss_out, void *stream);
int b2rl_c51_loss_bwd(const float *y, const float *t, const float *weights,
                      const float *grad_loss, int32_t B, int32_t n_atoms,
                      int mean, float *grad_y, void *stream);

/* Scalar TD loss: y = q[i, action[i]], t = r + discount*(1-terminal)*next_q,
 * Huber(delta=1) if clip_delta else 0.5*(y-t)^2.  Replaces
 * DQN._compute_target_values / _compute_loss and compute_[weighted_]value_loss
 * (pfrl/agents/dqn.py:44-104, 388-470).  delta_out = |y - t|. */
int b2rl_td_loss_fwd(const float *q, const int64_t *action, const float *next_q,
                     const float *reward, const float *discount,
                     const float *terminal, const float *weights, int32_t B,
                     int32_t n_actions, int clip_delta, int mean, float *y_out,
                     float *t_out, float *delta_out, float *scratch,
                     float *loss_out, void *stream);
int b2rl_td_loss_bwd(const float *y, const float *t, const float *weights,
                     const int64_t *action, const float *grad_loss, int32_t B,
                     int32_t n_actions, int clip_delta, int mean, float *grad_q,
                     void *stream);

/* Targets of the advantage-learning and DPP agents (`mode`), fused with the
 * scalar TD loss of b2rl_td_loss_fwd (same y/t/delta/loss outputs; the
 * gradient is b2rl_td_loss_bwd's).  tq, tnq: target net at s and s' [B,nA];
 * nq: online net at s' (DOUBLE_PAL only, else NULL).  T = r +
 * discount*(1-terminal)*nextV; A(x) = x[a] - max x; L the DPP operator.
 *   AL          nextV = max tnq            t = T + alpha*A(tq)
 *   PAL         nextV = max tnq            t = T + alpha*max(A(tq), A(tnq))
 *   DOUBLE_PAL  nextV = tnq[argmax nq]     t as PAL
 *   DPP         L = sum softmax(eta*x)*x   t = tq[a] + T(nextV = L tnq) - L tq
 *   DPPL        L = logsumexp(eta*x)/eta   t as DPP
 *   DPP_GREEDY  L = max x                  t as DPP
 * Replaces _compute_y_and_t of pfrl/agents/al.py, pal.py, double_pal.py and
 * dpp.py.  alpha and eta are rounded to fp32 once (eta > 0 for DPP, DPPL). */
#define B2RL_ADV_AL 0
#define B2RL_ADV_PAL 1
#define B2RL_ADV_DOUBLE_PAL 2
#define B2RL_ADV_DPP 3
#define B2RL_ADV_DPPL 4
#define B2RL_ADV_DPP_GREEDY 5
int b2rl_adv_td_loss_fwd(int mode, const float *q, const int64_t *action,
                         const float *tq, const float *tnq, const float *nq,
                         const float *reward, const float *discount,
                         const float *terminal, const float *weights, int32_t B,
                         int32_t n_actions, double alpha, double eta,
                         int clip_delta, int mean, float *y_out, float *t_out,
                         float *delta_out, float *scratch, float *loss_out,
                         void *stream);

/* NAF head (FCQuadraticStateQFunction): L with L[i][i] = exp(diag_pre[i]) and
 * the n(n-1)/2 entries of non_diag below the diagonal in np.tril_indices(n, -1)
 * order; mat = L L^T [B,n,n].  non_diag may be NULL when n = 1.  The backward
 * takes grad_mat (any, not assumed symmetric) and writes the gradients of
 * diag_pre and non_diag.  Any n. */
int b2rl_naf_head_fwd(const float *diag_pre, const float *non_diag, int32_t B,
                      int32_t n, float *mat, void *stream);
int b2rl_naf_head_bwd(const float *diag_pre, const float *non_diag,
                      const float *grad_mat, int32_t B, int32_t n,
                      float *grad_diag_pre, float *grad_non_diag, void *stream);

/* TD loss of the DQN family with a QuadraticActionValue (NAF):
 * Q(u) = v - 1/2 (u - mu)^T P (u - mu), max = v when neither bound is given,
 * else Q(clamp(mu)).  y = Q(s, a) from (mu, mat, v) of the online net at s;
 * (tmu, tmat, tv) and (tnmu, tnmat, tnv) the target net at s and s'; nmu the
 * online net's mu at s'; lo / hi the target net's bounds and nlo / nhi the
 * online net's ([n] each, any may be NULL).  T = r + discount*(1-terminal)*nextV.
 *   NAF_DQN         nextV = max'(s')              t = T
 *   NAF_DOUBLE_DQN  nextV = Q'(s', clamp(nmu))    t = T
 *   ADV_AL          nextV = max'(s')              t = T + alpha*A'(s, a)
 *   ADV_PAL         nextV = max'(s')              t = T + alpha*max(A'(s,a), A'(s',a))
 *   ADV_DOUBLE_PAL  nextV = Q'(s', clamp(nmu))    t as PAL
 *   ADV_DPP_GREEDY  nextV = max'(s')              t = Q'(s, a) + T - max'(s)
 * with A'(x, a) = Q'(x, a) - max'(x).  tmu/tmat/tv are needed except for the
 * DQN modes, nmu for the double modes.  Outputs as b2rl_td_loss_fwd.  The
 * backward writes d loss / d (mu, mat, v) of the online net at s. */
#define B2RL_NAF_DQN 6
#define B2RL_NAF_DOUBLE_DQN 7
int b2rl_naf_td_loss_fwd(int mode, const float *mu, const float *mat,
                         const float *v, const float *action, const float *tmu,
                         const float *tmat, const float *tv, const float *tnmu,
                         const float *tnmat, const float *tnv, const float *nmu,
                         const float *lo, const float *hi, const float *nlo,
                         const float *nhi, const float *reward,
                         const float *discount, const float *terminal,
                         const float *weights, int32_t B, int32_t n,
                         double alpha, int clip_delta, int mean, float *y_out,
                         float *t_out, float *delta_out, float *scratch,
                         float *loss_out, void *stream);
int b2rl_naf_td_loss_bwd(const float *mu, const float *mat, const float *action,
                         const float *y, const float *t, const float *weights,
                         const float *grad_loss, int32_t B, int32_t n,
                         int clip_delta, int mean, float *grad_mu,
                         float *grad_mat, float *grad_v, void *stream);

/* Quantile Huber loss of IQN: |tau - 1[t<y]| * Huber(y, t) over [B, N, N'],
 * mean over N', sum over N (compute_eltwise_huber_quantile_loss and the value
 * losses of pfrl/agents/iqn.py:176-250); delta_out = mean over (N, N'). */
int b2rl_quantile_huber_fwd(const float *y, const float *t, const float *taus,
                            const float *weights, int32_t B, int32_t N,
                            int32_t Np, int mean, float *delta_out,
                            float *scratch, float *loss_out, void *stream);
int b2rl_quantile_huber_bwd(const float *y, const float *t, const float *taus,
                            const float *weights, const float *grad_loss,
                            int32_t B, int32_t N, int32_t Np, int mean,
                            float *grad_y, void *stream);

/* ------------------------------------------------------------------------
 * PPO: generalised advantage estimation over a time-major rollout [T, E] and
 * the clipped-surrogate loss (forward value and gradients in one launch).
 * ---------------------------------------------------------------------- */

/* GAE, replaces _add_advantage_and_value_target_to_episode(s)
 * (pfrl/agents/ppo.py:36-53) and the std_mean of :476-478.
 * cut[t,e] = 1 marks the last transition of an episode segment (done, reset
 * or flush); valid (may be NULL) masks unused slots.  scratch: 3 doubles per
 * 128 environments.  stats[2] = mean, std (unbiased=False) of adv. */
int b2rl_gae(const float *reward, const float *nonterminal, const float *v,
             const float *v_next, const uint8_t *cut, const uint8_t *valid,
             int32_t T, int32_t E, double gamma, double lambda, float *adv,
             float *v_teacher, double *scratch, float *stats, void *stream);

/* PPO._lossfun (pfrl/agents/ppo.py:634-671) + the advantage standardisation
 * of :495 (adv_stats = {mean, std} or NULL).  The ratio is clamped to
 * float(1 - clip_eps), float(1 + clip_eps), rounded once from double as torch
 * rounds Python-float bounds.  clip_eps_vf < 0 selects the unclipped value
 * loss.  Gradients follow torch's rules for the reference expression: min and
 * max split a tie evenly, clamp passes the gradient on its bounds.  Outputs
 * d loss/d{log_prob, entropy, v_pred} and losses[4] = {total, policy, value,
 * entropy}.  scratch: 3 doubles per 256 samples. */
int b2rl_ppo_loss(const float *log_prob, const float *entropy,
                  const float *v_pred, const float *log_prob_old,
                  const float *v_pred_old, const float *adv,
                  const float *v_teacher, const float *adv_stats, int32_t M,
                  double clip_eps, float clip_eps_vf, float value_coef,
                  float entropy_coef, float *g_log_prob, float *g_entropy,
                  float *g_v_pred, double *scratch, float *losses, void *stream);

/* ------------------------------------------------------------------------
 * TRPO policy update (pfrl/agents/trpo.py:415-699, pfrl/utils/
 * conjugate_gradient.py): fp32 storage, fp64 accumulation, device pointers.
 * kind 0 = Independent(Normal(loc, scale), 1): params loc, scale [N, A] and
 * actions fp32 [N, A]; kind 1 = Categorical(logits): params logits [N, K]
 * (A = K, p1 / old1 / g1 / u1 / m1 unused) and actions int64 [N].
 * ---------------------------------------------------------------------- */

/* gain = mean(exp(logp - log_prob_old) * adv) + entropy_coef * mean(entropy),
 * kl = mean KL(old || new), by torch's formulas (Normal log_prob / entropy /
 * kl, Categorical's normalised logits, p_old == 0 -> 0 and p_new == 0 -> inf).
 * adv_stats = {mean, std} standardises adv as (adv - mean) / (std + 1e-8) in
 * fp32, or NULL.  out[3] = gain, kl, mean entropy.  g0 (and g1) non-NULL also
 * write d gain / d params per row.  scratch: 3 doubles per 256 rows. */
int b2rl_trpo_objective(int32_t kind, int32_t N, int32_t A, const float *p0,
                        const float *p1, const float *old0, const float *old1,
                        const void *actions, const float *log_prob_old,
                        const float *adv, const float *adv_stats,
                        double entropy_coef, float *g0, float *g1,
                        double *scratch, float *out, void *stream);

/* Fisher metric of the distribution parameters at p, applied to the tangent u
 * and divided by N: diag(1/scale^2, 2/scale^2) (Gaussian; m1 may be NULL for a
 * constant scale) or diag(p) - p p^T on the logits (categorical). */
int b2rl_trpo_fisher(int32_t kind, int32_t N, int32_t A, const float *p0,
                     const float *p1, const float *u0, const float *u1,
                     float *m0, float *m1, void *stream);

/* Conjugate gradient on n floats (one CTA per launch).  init: x = 0, r = p =
 * b, state[2] doubles = {r.r, converged}.  iter (once per CG iteration, with
 * Ap = A p): alpha = rr / p.Ap, x += alpha p, r -= alpha Ap, then either
 * ||r|| < tol marks the state converged (later iterations return at once) or
 * p = r + (r.r / rr) p.  step: dId = float(x.Ax), full_step =
 * float(sqrt(2 max_kl / (dId + 1e-8))) * x; dId may be NULL. */
int b2rl_trpo_cg_init(int64_t n, const float *b, float *x, float *r, float *p,
                      double *state, void *stream);
int b2rl_trpo_cg_iter(int64_t n, const float *Ap, float *x, float *r, float *p,
                      double *state, double tol, void *stream);
int b2rl_trpo_cg_step(int64_t n, const float *x, const float *Ax, double max_kl,
                      float *full_step, float *dId, void *stream);

/* Line-search decision over n_cand (<= 64) evaluated candidates theta_old +
 * 2^-i full_step: cand[i][3] and gain0[3] are objective outputs.  The first
 * candidate with a finite gain and KL, double(gain_i) - double(gain0) >= 0 and
 * kl_i <= max_kl wins.  theta = theta_old + 2^-i * full_step (fp32 multiply,
 * then add), or theta_old bit for bit when none wins.  record[3] = winner's
 * kl, its step size (0 if none), 1 if one won. */
int b2rl_trpo_line_search(int32_t n_cand, const float *cand, const float *gain0,
                          double max_kl, int64_t n, const float *theta_old,
                          const float *full_step, float *theta, float *record,
                          void *stream);

/* ------------------------------------------------------------------------
 * ACER's discrete-action loss gradient on one sequence of T steps
 * (pfrl/agents/acer.py:16-115, 207-248, 423-552): fp32 storage, fp64
 * accumulation, device pointers, one CTA.
 * z, q [T, K]: the policy's Categorical._param (normalised logits) and the Q
 * values.  avg_z [T, K]: the average model's logits (NULL without the trust
 * region).  mu_z [T, K]: the behaviour policy's logits, or NULL for the online
 * update (rho = 1).  actions int64 [T], rewards fp64 [T].  bootstrap: the
 * device fp32 value of the state after the last step, or NULL for a terminal
 * (R = 0).  truncate = 0 means truncation_threshold None; the threshold may be
 * 0 or inf.  average_kl (fp64 [1], read and written) takes each step's
 * KL(avg || pi) in reversed step order when use_trust_region is set.
 * Writes g_z = d total / d z and g_q = d total / d q [T, K].  scratch: 10
 * doubles per step. */
int b2rl_acer_loss(int32_t T, int32_t K, const float *z, const float *q,
                   const float *avg_z, const float *mu_z, const int64_t *actions,
                   const double *rewards, const float *bootstrap, double gamma,
                   int32_t truncate, double truncation_threshold,
                   int32_t use_trust_region, double delta, double beta,
                   double pi_loss_coef, double q_loss_coef,
                   int32_t normalize_by_steps, int32_t use_q_opc,
                   double *average_kl, double average_kl_decay, double *scratch,
                   float *g_z, float *g_q, void *stream);

/* ------------------------------------------------------------------------
 * REINFORCE's loss gradient over the N recorded steps of an update
 * (pfrl/agents/reinforce.py:176-195): loss = sum_rows(-R log pi(a) - beta H)
 * / batchsize.  fp32 storage, fp64 arithmetic, device pointers, one warp per
 * row.  A Categorical gives z [N, D] (Categorical._param, normalised logits),
 * int64 actions [N] and g_z [N, D]; loc and action_values are then NULL.  An
 * Independent(Normal, 1) gives loc [N, D], scale [N, D] (NULL = 1), the
 * sampled fp32 action_values [N, D] and g_loc [N, D]; g_scale [N, D] is
 * written unless NULL; z is then NULL.  returns fp32 [N].  row_loss and
 * row_entropy [N] (optional) take each row's loss term and entropy. */
int b2rl_reinforce_loss(int64_t N, int32_t D, const float *z, const float *loc,
                        const float *scale, const int64_t *actions,
                        const float *action_values, const float *returns,
                        int32_t batchsize, double beta, float *g_z, float *g_loc,
                        float *g_scale, float *row_loss, float *row_entropy,
                        void *stream);

/* ------------------------------------------------------------------------
 * A3C's loss gradient over the N recorded steps of one segment
 * (pfrl/agents/a3c.py:177-204): returns R from the fp64 scan R = R * gamma + r
 * backwards from *bootstrap (NULL = terminal, R = 0), rounded to fp32;
 * adv = R - v; loss = pi_factor * sum_rows(-adv log pi(a) - beta H)
 * + v_factor * sum_rows((v - R)^2) / 2.  fp32 storage, fp64 arithmetic, device
 * pointers, one warp per row.  The policy is given as for b2rl_reinforce_loss
 * (z, actions and g_z, or loc, scale, action_values, g_loc and g_scale).
 * v fp32 [N], rewards fp64 [N].  Writes g_v [N]; returns [N] (fp32) unless
 * NULL; row_pi_loss and row_v_loss [N] (both or neither) take each row's
 * term of pi_loss and v_loss. */
int b2rl_a3c_loss(int64_t N, int32_t D, const float *z, const float *loc,
                  const float *scale, const int64_t *actions,
                  const float *action_values, const float *v, const double *rewards,
                  const float *bootstrap, double gamma, double beta, double pi_factor,
                  double v_factor, float *g_z, float *g_loc, float *g_scale, float *g_v,
                  float *returns, float *row_pi_loss, float *row_v_loss, void *stream);

/* ------------------------------------------------------------------------
 * SAC / TD3 / DDPG update tail (fp32, device pointers).
 * ---------------------------------------------------------------------- */

/* Polyak averaging of up to any number of (target, source) fp32 tensor pairs in
 * one launch per 96 pairs: target = target * float(1 - tau) + float(tau) * source,
 * each operation rounded separately -- bit for bit soft_copy_param's
 * `target.mul_(1 - tau); target.add_(tau * source)` (pfrl/utils/copy_param.py:9-22,
 * called from SoftActorCritic.sync_target_network, soft_actor_critic.py:199-212).
 * pairs_host is read before the call returns.  Every pair needs non-NULL pointers
 * (an empty pair included) and numel >= 0, and tau must lie in [0, 1]; all of it is
 * checked before the first launch, so a refused call changes no target.  Pairs
 * are updated concurrently: no target may share memory with another target or a
 * source. */
typedef struct {
    void *dst;       /* target tensor (device, fp32, contiguous) */
    const void *src; /* source tensor (device, fp32, contiguous) */
    int64_t numel;
} b2rl_tensor_pair;
int b2rl_polyak(const b2rl_tensor_pair *pairs_host, int32_t n_pairs, double tau,
                void *stream);

/* Entropy-regularised TD target of SoftActorCritic.update_q_func
 * (pfrl/agents/soft_actor_critic.py:225-240):
 *   out = reward + discount * (1 - terminal) * (min(q1, q2) - temperature * log_prob)
 * with the reference's operation order and one rounding per operation; min is
 * torch.min's: NaN when either Q is NaN.
 * temperature_dev (device scalar) takes precedence over `temperature`. */
int b2rl_sac_target(const float *reward, const float *discount, const float *terminal,
                    const float *q1, const float *q2, const float *log_prob,
                    const float *temperature_dev, float temperature, int32_t n,
                    float *out, void *stream);

/* TD3's default target-policy smoothing (pfrl/agents/td3.py:20-24) for a given noise
 * draw, n elements:
 *   out = clamp(action + clamp(0.2 * noise, -0.5, 0.5), -1, 1)
 * with one rounding per operation, as torch's eager sequence (clamp passes NaN through).
 * The noise is the caller's torch.randn_like(action), so the random stream is the
 * reference's.  0 < n < 2^39. */
int b2rl_td3_smooth(const float *action, const float *noise, int64_t n, float *out,
                    void *stream);

/* The critic update of TD3 (pfrl/agents/td3.py:181-236) and DDPG
 * (pfrl/agents/ddpg.py:150-173) after the forwards, in one launch, for n > 0 rows:
 *   target  = reward + d * (1 - terminal) * next_q
 *             (d = discount[i], the n-step discount of TD3, or gamma when discount is
 *             NULL, as DDPG; next_q = torch.min(next_q1, next_q2), or next_q1 when
 *             next_q2 is NULL), rounded like the reference's expression;
 *   loss_c  = mse_loss(target, pred_c) with reduction "mean" (a deterministic fp32 sum in
 *             an order of this kernel's own, divided by n);
 *   grad_c  = float(2.0 / n) * (pred_c - target), rounded as torch's mse_loss backward,
 *             which multiplies this by the upstream gradient.
 * c = 1, and c = 2 when pred_q2 is not NULL (then grad2 and loss2 are required).
 * A CTA takes B2RL_CRITIC_LOSS_ROWS_PER_CTA rows; when n exceeds that, `partial` must
 * hold 2 * ceil(n / B2RL_CRITIC_LOSS_ROWS_PER_CTA) floats of scratch (else it may be
 * NULL).  The call neither allocates nor synchronises. */
#define B2RL_CRITIC_LOSS_ROWS_PER_CTA 1024
int b2rl_td3_critic_loss(const float *reward, const float *discount, float gamma,
                         const float *terminal, const float *next_q1, const float *next_q2,
                         const float *pred_q1, const float *pred_q2, int32_t n, float *target,
                         float *grad1, float *grad2, float *loss1, float *loss2,
                         float *partial, void *stream);

/* ------------------------------------------------------------------------
 * Dense contraction kept in exact fp32: first Nature-DQN convolution,
 * x[N,4,84,84] * w[32,4,8,8] (stride 4) + bias -> out[N,32,20,20].
 * Replaces the cuDNN call behind nn.Conv2d(4, 32, 8, stride=4)
 * (pfrl/nn/atari_cnn.py:30-36, pfrl/q_functions/dueling_dqn.py:34-40,91-97)
 * in the forward direction; bias may be NULL. */
int b2rl_conv_nature1_fwd(const float *x, const float *w, const float *bias,
                          int32_t n_images, float *out, void *stream);
/* Same layer on uint8 images x[N,4,84,84] (what b2rl_replay_gather / b2rl_replay_step
 * emit with B2RL_OBS_RAW): the kernel expands float(x) * scale in shared memory, i.e.
 * phi = x / 255 (examples/atari/train_dqn_batch_ale.py:229-231) is folded into the
 * convolution and the f32 batch never exists in HBM.  Bit-identical to
 * b2rl_conv_nature1_fwd on the B2RL_OBS_U8_TO_F32 output for the same scale. */
int b2rl_conv_nature1_fwd_u8(const uint8_t *x, float scale, const float *w,
                             const float *bias, int32_t n_images, float *out,
                             void *stream);

/* ------------------------------------------------------------------------
 * Dense layers on the Hopper tensor cores (wgmma) with fp32 results (3 x TF32 split):
 *   C[M,N] = A[M,K] . B[N,K]^T (+ bias[N]) (relu)
 * Replaces the cuBLAS SGEMM behind F.linear and its two backward products
 * (pfrl/q_functions/dueling_dqn.py:67-129, pfrl/nn/noisy_linear.py:53-70,
 * pfrl/nn/atari_cnn.py:17-47).  a_mn_major / b_mn_major = 0: the operand is stored
 * row-major with the contraction index contiguous ([M][K] / [N][K], leading dimension
 * lda / ldb); = 1: stored with the contraction index as the row index ([K][M] / [K][N]),
 * which is how dX = dY . W (B = W) and dW = dY^T . X (A = dY, B = X) read their operands
 * without a transposed copy.  Small products are cut along K; the partial tiles need
 * b2rl_gemm_workspace_bytes(M, N, K) bytes of 16-byte aligned device memory (0 = none)
 * and are summed in a fixed order, so results are run-to-run deterministic.
 * bias may be NULL. */
int64_t b2rl_gemm_workspace_bytes(int32_t M, int32_t N, int32_t K);
int b2rl_gemm_tf32x3(const float *A, int32_t lda, int32_t a_mn_major,
                     const float *B, int32_t ldb, int32_t b_mn_major,
                     const float *bias, int32_t relu, float *C, int32_t ldc,
                     int32_t M, int32_t N, int32_t K,
                     void *workspace, int64_t workspace_bytes, void *stream);

/* The same product with operands that are read in place through index tables: the
 * convolutions of the Nature trunk (pfrl/nn/atari_cnn.py:30-44,
 * pfrl/q_functions/dueling_dqn.py:34-40,91-97 -- cuDNN forward / dgrad / wgrad in the
 * reference) as implicit GEMMs.  A gather operand's element (row, k) lives at
 *   row_off[row] + k_off[k]
 * and -- when the coordinate tables are given -- is zero unless
 *   0 <= y + dy < y_limit and 0 <= x + dx < x_limit,
 * y | x << 16 = row_yx[row] (unsigned 16-bit halves), dy | dx << 16 = k_yx[k] (signed 16-bit
 * halves).  The k tables must be padded to a multiple of 32 entries and 16-byte aligned.
 * uint8 sources are read as float(byte) * scale.  The output is dense (ld) or, with
 * row_tab, scattered: C[m, n] at row_tab[m] + n * col_stride.  pfrl_b200/ops/conv.py builds
 * the tables (forward, input gradient per stride phase, weight gradient). */
enum { B2RL_GEMM_K_MAJOR = 0, B2RL_GEMM_MN_MAJOR = 1, B2RL_GEMM_GATHER = 2 };
typedef struct b2rl_gemm_operand {
    const void *data;        /* fp32, or uint8 when u8 != 0 (gather mode only) */
    int32_t mode;            /* B2RL_GEMM_* */
    int32_t ld;              /* dense modes: elements between rows */
    const int32_t *row_off;  /* gather: element offset per row (device memory) */
    const int32_t *row_yx;   /* gather: coordinates per row, or NULL */
    const int32_t *k_off;    /* gather: element offset per k */
    const int32_t *k_yx;     /* gather: coordinate steps per k, or NULL */
    int32_t y_limit, x_limit;
    int32_t lanes_along_k;   /* coalescing hint: consecutive k are close in memory */
    int32_t u8;
    float scale;
} b2rl_gemm_operand;
typedef struct b2rl_gemm_output {
    float *data;
    int32_t ld;              /* dense: C[m * ld + n] */
    const int32_t *row_tab;  /* scatter when not NULL */
    int32_t col_stride;
    const float *bias;       /* [N] or NULL; 4-byte aligned, may start at any float */
    int32_t relu;
} b2rl_gemm_output;
/* Debug aid: %globaltimer stamps of the phases of every CTA of the following launches are
 * written to device_buffer (8 x uint64 per CTA); NULL switches it off. */
int b2rl_gemm_debug_times(void *device_buffer);
int b2rl_gemm_tf32x3_ex(const b2rl_gemm_operand *A, const b2rl_gemm_operand *B,
                        const b2rl_gemm_output *C, int32_t M, int32_t N, int32_t K,
                        void *workspace, int64_t workspace_bytes, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* B2RL_H */
