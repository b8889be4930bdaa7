"""Host-memory emulation of pfrl_b200.store.DeviceReplayStore's write side
(put_parts / append / set_max_priority), for `-m "not gpu"` tests of the host
logic that feeds it (n-step windows, frame de-duplication, checkpoint
restore).  TEST INFRASTRUCTURE ONLY -- the product has no host fallback."""
import numpy as np
import torch


class FakeStore:
    instances = []

    def __init__(self, capacity, part_bytes, stack=1, n_step=1, action_bytes=8,
                 prioritized=True, part_capacity=None, device=0, max_batch=4096):
        self.capacity, self.part_bytes, self.stack = capacity, part_bytes, stack
        self.n_step, self.action_bytes, self.prioritized = n_step, action_bytes, prioritized
        self.part_capacity = part_capacity or 2 * capacity + 64
        self.device = torch.device("cpu")
        self.parts = np.zeros((self.part_capacity, part_bytes), dtype=np.uint8)
        self.part_head = 0
        self.records = []          # live window, oldest first
        self.max_priority = 1.0
        self.closed = False
        FakeStore.instances.append(self)

    def close(self):
        self.closed = True

    def __len__(self):
        return len(self.records)

    def put_parts(self, parts):
        a = np.ascontiguousarray(parts).reshape(-1, self.part_bytes)
        # b2rl_replay_put_parts refuses more parts than the ring holds
        assert len(a) <= self.part_capacity, "put_parts: %d parts exceed the ring (%d)" % (
            len(a), self.part_capacity)
        slots = (self.part_head + np.arange(len(a))) % self.part_capacity
        self.parts[slots] = a
        self.part_head += len(a)
        return slots.astype(np.int32)

    def append(self, state_parts, next_parts, action, rewards, length, terminal, priority=None):
        sp = np.asarray(state_parts, dtype=np.int32).reshape(-1, self.stack)
        n = len(sp)
        nx = np.asarray(next_parts, dtype=np.int32).reshape(n, self.stack)
        act = np.asarray(action).view(np.uint8).reshape(n, self.action_bytes)
        rw = np.asarray(rewards, dtype=np.float64).reshape(n, self.n_step)
        for i in range(n):
            pr = self.max_priority if priority is None else float(priority[i])
            self.records.append(dict(sp=sp[i].copy(), nx=nx[i].copy(), action=act[i].copy(),
                                     rewards=rw[i].copy(), len=int(length[i]),
                                     terminal=int(terminal[i]), priority=pr))
        del self.records[:max(0, len(self.records) - self.capacity)]

    def set_max_priority(self, value):
        self.max_priority = float(value)

    # -- read-back helpers for assertions --------------------------------------
    def obs(self, slots, dtype, part_nbytes, part_shape):
        frames = [self.parts[s, :part_nbytes].view(dtype).reshape(part_shape) for s in slots]
        return np.concatenate(frames, axis=0) if len(frames) > 1 else frames[0]


def _neumaier(values):
    """CPython's float sum() (compensated since 3.12), which is what the
    reference's `sum(gamma ** i * r_i)` evaluates to (pfrl/replay_buffer.py:185-188)."""
    return sum(values)


class OracleBackedStore(FakeStore):
    """FakeStore + the read side, with the priority trees served by the CPU
    oracle (oracle/per_oracle.c).  Lets the golden traces of the reference run
    through the REAL host logic of the device buffers on a machine without a
    GPU; index arithmetic comes from the oracle, so this checks the host code,
    not the kernels."""

    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        from oracle.replay import OraclePrioritizedBuffer

        self.tree = OraclePrioritizedBuffer(self.capacity) if self.prioritized else None
        self.napp = 0
        self._last_idx = None
        self._last = None

    def append(self, state_parts, next_parts, action, rewards, length, terminal, priority=None):
        n = np.asarray(state_parts).reshape(-1, self.stack).shape[0]
        if self.tree is not None:
            # a restored max_priority (set_max_priority) lives here; the oracle tree only
            # learns its max through set_last_priority
            self.max_priority = max(self.max_priority, self.tree.max_priority)
        super().append(state_parts, next_parts, action, rewards, length, terminal, priority)
        self.napp += n
        if self.tree is not None:
            for i in range(n):
                self.tree.append(None, self.max_priority if priority is None
                                 else float(priority[i]))

    def sample(self, u, mode=0, want_index=True, want_priority=True):
        assert mode == 0, "the oracle restates the exact (sequential) sampler only"
        idx, pri, total, mn = self.tree.sample_indices(len(u), u)
        self._last_idx, self._last = idx, (pri, total, mn)
        return torch.from_numpy(idx.copy()), torch.from_numpy(pri.copy())

    def weights(self, n, beta, norm, want_prob=False):
        pri, total, mn = self._last
        probs = [p / total for p in pri.tolist()]
        if norm == 0:       # NORM_NONE: (N * prob) ** -beta
            w = [(len(self.records) * p) ** -beta for p in probs]
        else:
            min_p = min(probs) if norm == 1 else mn / total
            w = [(p / min_p) ** -beta for p in probs]
        w = torch.tensor(w, dtype=torch.float32)
        return (w, torch.tensor(probs, dtype=torch.float64)) if want_prob else w

    def update_priorities(self, priority):
        priority = np.asarray(priority, dtype=np.float64)
        for i, p in zip(self._last_idx.tolist(), priority.tolist()):
            self.records[i]["priority"] = p
        self.tree.set_last_priority(priority)
        self.max_priority = self.tree.max_priority
        self._last_idx = None

    def update_host_errors(self, errors, alpha, eps, error_min, error_max, defer):
        """The product path of update_errors(host list): the priorities come from the LIBRARY's
        host arithmetic (b2rl_host_priority_from_errors, libm pow) -- so the CPU replays of the
        reference's golden traces also pin that arithmetic, not only the Python formula."""
        import ctypes

        from pfrl_b200 import _lib

        e = np.ascontiguousarray(errors, dtype=np.float64)
        out = np.empty_like(e)
        _lib.check(_lib.load().b2rl_host_priority_from_errors(
            e.ctypes.data_as(ctypes.c_void_p), e.shape[0], float(alpha), float(eps),
            int(error_min is not None), 0.0 if error_min is None else float(error_min),
            int(error_max is not None), 0.0 if error_max is None else float(error_max),
            out.ctypes.data_as(ctypes.c_void_p)))
        assert (out > 0.0).all()  # collections/prioritized.py:109
        self.update_priorities(out)

    def read_priorities(self, first=0, n=None):
        n = len(self.records) - first if n is None else n
        return np.array([r["priority"] for r in self.records[first:first + n]], dtype=np.float64)

    def info(self):
        return dict(total=self.tree.total(), min=self.tree.min(),
                    max_priority=max(self.tree.max_priority, self.max_priority), napp=self.napp,
                    npop=self.napp - len(self.records), scout_hits=0)

    def gather(self, n, gamma_pow, index=None, obs_mode=0, obs_scale=1.0, obs_dtype=None,
               obs_shape=None, action_dtype=torch.int64, action_shape=(), want_obs=True,
               want_steps=False):
        idx = self._last_idx if index is None else index.numpy()
        assert len(idx) == n
        recs = [self.records[int(i)] for i in idx]
        out = {}
        if want_obs:
            for key, slot_key in (("state", "sp"), ("next_state", "nx")):
                raw = np.stack([self.parts[r[slot_key]].reshape(-1) for r in recs])
                if obs_mode == 1:   # OBS_U8_TO_F32
                    t = torch.from_numpy(raw.astype(np.float32) * np.float32(obs_scale))
                else:
                    t = torch.from_numpy(raw)
                    if obs_dtype is not None and obs_dtype != torch.uint8:
                        t = t.view(obs_dtype)
                if obs_shape is not None:
                    t = t.view((n,) + tuple(obs_shape))
                out[key] = t
        abytes = np.stack([r["action"] for r in recs])
        out["action"] = torch.from_numpy(abytes).view(action_dtype).view((n,) + tuple(action_shape))
        out["reward"] = torch.tensor(
            [_neumaier([gamma_pow[i] * r["rewards"][i] for i in range(r["len"])]) for r in recs],
            dtype=torch.float64).float()
        out["discount"] = torch.tensor([gamma_pow[r["len"]] for r in recs],
                                       dtype=torch.float64).float()
        out["is_state_terminal"] = torch.tensor([float(r["terminal"]) for r in recs])
        if want_steps:
            out["step_rewards"] = torch.from_numpy(np.stack([r["rewards"] for r in recs]))
            out["len"] = torch.tensor([r["len"] for r in recs], dtype=torch.uint8)
        return out
