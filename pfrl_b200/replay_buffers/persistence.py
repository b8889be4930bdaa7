"""save / load of device replay buffers (AbstractReplayBuffer.save/load,
pfrl/replay_buffer.py:69-85).  The live window is exported through the gather
kernel in chunks (raw observations, per-step rewards, priorities) into one
.npz archive and re-appended on load."""
import numpy as np
import torch


class _FramePool:
    """Frames of frame-stacked (LazyFrames) observations, stored once: consecutive
    observations share all but one frame, so the archive of a 1 M-transition Atari buffer
    is ~7 GB of frames + index rows instead of 56 GB of stacked observations."""

    def __init__(self):
        self.ids = {}
        self.frames = []

    def index(self, stacked, stack):
        """stacked: [m, stack * c, ...] -> int64 [m, stack] of frame ids."""
        m = stacked.shape[0]
        fr = stacked.reshape((m, stack, -1))
        out = np.empty((m, stack), dtype=np.int64)
        for i in range(m):
            for j in range(stack):
                key = fr[i, j].tobytes()
                k = self.ids.get(key)
                if k is None:
                    k = len(self.frames)
                    self.ids[key] = k
                    self.frames.append(fr[i, j].copy())
                out[i, j] = k
        return out


def save_buffer(buf, filename):
    if getattr(buf, "_waiting", False):
        # between sample() and update_errors() the sampled leaves are zero in the sum
        # tree (collections/prioritized.py:98-116); the reference pickles whatever is
        # there and fails on load, we refuse up front
        raise RuntimeError("cannot save a prioritised buffer between sample() and "
                           "update_errors(): the sampled priorities are not restored yet")
    buf._flush()
    n = len(buf)
    lay = buf.layout
    lazy = bool(lay is not None and lay.lazy and not lay.on_device)
    meta = dict(n=n, num_steps=buf.num_steps, prioritized=buf._prioritized, format=2,
                lazy=int(lazy), stack=int(lay.stack) if lay is not None else 1)
    if n == 0:
        np.savez(filename if str(filename).endswith(".npz") else open(filename, "wb"), **meta)
        return
    from pfrl_b200.replay_buffers.device_buffer import DeviceExperiences

    chunks = {k: [] for k in ("state", "next_state", "action", "step_rewards", "len", "term")}
    pool = _FramePool() if lazy else None
    for lo in range(0, n, 4096):
        m = min(4096, n - lo)
        idx = torch.arange(lo, lo + m, dtype=torch.int64, device=buf.device)
        out = buf._gather(DeviceExperiences(buf, m, index=idx), 1.0, None, raw=True,
                          want_steps=True)
        st, ns = out["state"].cpu().numpy(), out["next_state"].cpu().numpy()
        if lazy:  # frame ids instead of stacked observations
            st, ns = pool.index(st, lay.stack), pool.index(ns, lay.stack)
        chunks["state"].append(st)
        chunks["next_state"].append(ns)
        chunks["action"].append(out["action"].cpu().numpy())
        chunks["step_rewards"].append(out["step_rewards"].cpu().numpy())
        chunks["len"].append(out["len"].cpu().numpy())
        chunks["term"].append(out["is_state_terminal"].cpu().numpy())
    arrays = {k: np.concatenate(v) for k, v in chunks.items()}
    if lazy:
        arrays["frames"] = np.stack(pool.frames).reshape((len(pool.frames),) + tuple(lay.part_shape))
    if buf._prioritized:
        arrays["priority"] = buf.store.read_priorities()
        arrays["max_priority"] = np.float64(buf.store.info()["max_priority"])
    with open(filename, "wb") as f:
        np.savez(f, **meta, **arrays)


def _reset(buf):
    if buf.store is not None:
        buf.store.close()
    buf.store = None
    buf._n_total = 0
    buf._pend_parts, buf._pend_exp = [], []
    buf._part_head = 0
    buf._part_cache.clear()
    buf._live_min_seq.clear()
    buf.last_n_transitions.clear()
    if buf._prioritized:
        buf._waiting = False
        buf._last_handle = None


def _restore(buf, records, max_priority):
    """Re-append ``records`` = iterable of (state, next_state, action,
    step_rewards, terminal, priority-or-None), oldest first."""
    _reset(buf)
    for s, ns, action, rewards, term, priority in records:
        if buf.store is None:
            buf._create_store(s, action)
        s_slots, s_min = buf._parts_of(s)
        n_slots, n_min = buf._parts_of(ns)
        act = buf.layout._action_array(action).tobytes()
        if buf._prioritized and priority is None:
            raise ValueError("a prioritised buffer cannot be restored without priorities")
        buf._pend_exp.append((s_slots, n_slots, act, [float(r) for r in rewards], len(rewards),
                              bool(term), None if priority is None else float(priority)))
        buf._note_live(buf._n_total, (min(s_min, n_min),))
        buf._n_total += 1
        if len(buf._pend_exp) >= 4096:
            buf._flush()
    buf._flush()
    if buf._prioritized and buf.store is not None and max_priority is not None:
        buf.store.set_max_priority(max_priority)


def load_buffer(buf, filename):
    from pfrl_b200.replay_buffers import reference_pickle

    if reference_pickle.looks_like_pickle(filename):
        return load_reference_pickle(buf, filename)
    with open(filename, "rb") as f:
        z = np.load(f, allow_pickle=False)
        z = {k: z[k] for k in z.files}
    n = int(z["n"])
    assert int(z["num_steps"]) == buf.num_steps
    pr = z.get("priority")

    lazy = bool(int(z.get("lazy", 0)))
    if lazy:
        # the observations come back as LazyFrames over SHARED frame objects: the store
        # takes every frame once (identity de-duplication) and the layout stays the
        # frame-stacked one, so appending LazyFrames after load() works
        from pfrl_b200.utils.lazy_frames import LazyFrames

        frames = [f for f in z["frames"]]

        def obs(row):
            return LazyFrames([frames[int(i)] for i in row], stack_axis=0)
    else:
        def obs(row):
            return row

    def records():
        for k in range(n):
            L = int(z["len"][k])
            yield (obs(z["state"][k]), obs(z["next_state"][k]), z["action"][k],
                   z["step_rewards"][k][:L], z["term"][k], None if pr is None else pr[k])

    mp = z.get("max_priority")
    _restore(buf, records(), None if mp is None else float(mp))


def load_reference_pickle(buf, filename):
    """Fill a device buffer from the reference's ``replay_buffer.pkl``
    (pfrl/replay_buffers/replay_buffer.py:85-94, agents/dqn.py:794-810).  An
    experience keeps what batch_experiences reads (replay_buffer.py:157-212):
    state / action of its first transition, next_state of its last, the
    per-step rewards and any(is_state_terminal)."""
    from pfrl_b200.replay_buffers import reference_pickle

    ref = reference_pickle.read(filename)
    if buf._prioritized and ref.priorities is None:
        raise TypeError("%s holds a uniform buffer; cannot load it into a prioritised one"
                        % filename)
    exps = ref.experiences
    if any(len(e) > buf.num_steps for e in exps):
        raise ValueError("checkpoint holds %d-step experiences, buffer was built with "
                         "num_steps=%d" % (max(len(e) for e in exps), buf.num_steps))
    pri = ref.priorities if buf._prioritized else None

    def records():
        for k, e in enumerate(exps):
            yield (e[0]["state"], e[-1]["next_state"], e[0]["action"],
                   [t["reward"] for t in e], any(t["is_state_terminal"] for t in e),
                   None if pri is None else pri[k])

    _restore(buf, records(), ref.max_priority if buf._prioritized else None)
