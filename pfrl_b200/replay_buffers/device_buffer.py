"""HBM-resident n-step replay buffers behind the reference's buffer API.

Host side of the drop-in classes ``ReplayBuffer`` / ``PrioritizedReplayBuffer``
(reference: pfrl/replay_buffers/replay_buffer.py:11-94,
pfrl/replay_buffers/prioritized.py:69-126).  The n-step window bookkeeping is
plain Python (a few integers per transition); observations, records and the
priority trees live in a ``DeviceReplayStore`` (libb2rl.so) and are only
touched by CUDA kernels.

Differences from the reference that a user can observe
  * ``sample(n)`` returns a ``DeviceExperiences`` sequence.  Passed to
    ``batch_experiences`` / ``agent.update`` it is gathered on the device;
    indexed or iterated it materialises the reference's list-of-dict form
    (intermediate n-step states are not stored, they come back as ``None``).
  * observations must be array-like (ndarray, scalar, CUDA tensor) or
    LazyFrames-like objects exposing ``_frames``; frames / arrays are
    de-duplicated by object identity, like LazyFrames shares frame arrays.
  * priorities are fp64 on the device (see DESIGN.md, "dtype contract").
"""
import collections

import numpy as np
import torch

from pfrl_b200 import _lib
from pfrl_b200.store import DeviceReplayStore
from pfrl_b200.utils.random import sample_n_k

_UNBOUNDED_DEFAULT = 1 << 20


def _round16(n):
    return (n + 15) // 16 * 16


class _Layout:
    """How observations / actions map onto parts and bytes."""

    def __init__(self, state, action):
        frames = getattr(state, "_frames", None)
        if frames is not None:
            if getattr(state, "stack_axis", 0) != 0:
                # parts are laid out back to back in the gathered observation, which is a
                # concatenation along the FIRST axis (chw frames); hwc stacks interleave
                raise TypeError(
                    "device replay buffers need LazyFrames stacked along axis 0 (channel-first "
                    "frames, e.g. VectorFrameStack(stack_axis=0) / FrameStack(channel_order="
                    "'chw')); got stack_axis=%r" % (state.stack_axis,))
            first = frames[0]
            self.lazy = True
            self.stack = len(frames)
            self.on_device = isinstance(first, torch.Tensor)
            if self.on_device:
                self.part_dtype = first.dtype
                self.part_shape = tuple(first.shape)
                nbytes = first.numel() * first.element_size()
            else:
                first = np.asarray(first)
                self.part_dtype = first.dtype
                self.part_shape = first.shape
                nbytes = first.nbytes
            if len(self.part_shape) == 0:
                self.obs_shape = (self.stack,)
            else:
                self.obs_shape = (self.stack * self.part_shape[0],) + tuple(self.part_shape[1:])
        else:
            self.lazy = False
            self.stack = 1
            self.on_device = isinstance(state, torch.Tensor)
            if self.on_device:
                self.part_dtype = state.dtype
                self.part_shape = tuple(state.shape)
                nbytes = state.numel() * state.element_size()
            else:
                arr = np.asarray(state)
                if arr.dtype == object:
                    raise TypeError(
                        "device replay buffers need array-like observations, got %r" % type(state))
                self.part_dtype = arr.dtype
                self.part_shape = arr.shape
                nbytes = arr.nbytes
            self.obs_shape = self.part_shape
        self.part_nbytes = nbytes
        self.part_bytes = _round16(max(nbytes, 1))
        a = self._action_array(action, first=True)
        self.action_dtype = a.dtype
        self.action_shape = a.shape
        self.action_bytes = max(a.nbytes, 1)

    def _action_array(self, action, first=False):
        if isinstance(action, torch.Tensor):
            action = action.detach().cpu().numpy()
        if first:
            a = np.asarray(action)
            if a.dtype == np.float64 and not isinstance(action, np.ndarray):
                a = a.astype(np.float32)  # torch.as_tensor(list of py floats) is float32
            if a.dtype.kind in "iub" and a.dtype != np.int64:
                a = a.astype(np.int64)
            return a
        return np.asarray(action, dtype=self.action_dtype).reshape(self.action_shape)

    def torch_obs_dtype(self):
        if isinstance(self.part_dtype, torch.dtype):
            return self.part_dtype
        return torch.from_numpy(np.empty(0, dtype=self.part_dtype)).dtype

    def torch_action_dtype(self):
        return torch.from_numpy(np.empty(0, dtype=self.action_dtype)).dtype


class DeviceExperiences(collections.abc.Sequence):
    """The result of ``sample(n)``: n experiences that still live in HBM."""

    def __init__(self, buffer, n, index=None, weights=None, pending=False):
        self.buffer = buffer
        self.n = n
        self.index = index  # CUDA int64 logical indices (None only for pending PER)
        self.weights = weights  # CUDA f32 or None
        self.pending = pending  # gather through the handle's last sampled slots
        self._lists = None
        # fused step: the raw gather outputs that came out of the same launch as
        # the draws, and the (gamma, obs_mode, obs_scale) they were made for
        self._prefetched = None
        self._prefetch_key = None

    def __len__(self):
        return self.n

    def batch(self, gamma, phi, device=None):
        """Device-side batch_experiences (pfrl/replay_buffer.py:157-212)."""
        return self.buffer._gather(self, gamma, phi)

    def _materialise(self):
        if self._lists is None:
            self._lists = self.buffer._materialise(self)
        return self._lists

    def __getitem__(self, i):
        return self._materialise()[i]

    def __iter__(self):
        return iter(self._materialise())


class DeviceNStepBuffer:
    """Common machinery of the two device-backed buffers."""

    _prioritized = False

    def __init__(self, capacity=None, num_steps=1, device=None, part_capacity=None,
                 max_batch=4096, unbounded_capacity=_UNBOUNDED_DEFAULT):
        assert num_steps > 0
        self._capacity = capacity
        self.num_steps = num_steps
        self._alloc_capacity = capacity if capacity is not None else unbounded_capacity
        self._device_arg = device
        self._part_capacity_arg = part_capacity
        self._max_batch = max_batch
        self.store = None
        self.layout = None
        self.last_n_transitions = collections.defaultdict(
            lambda: collections.deque([], maxlen=num_steps))
        # host mirrors / pending work
        self._n_total = 0          # experiences ever emitted
        self._pend_parts = []      # arrays / tensors waiting for upload
        self._pend_exp = []        # (state_slots, next_slots, action, rewards, len, term, prio)
        self._part_head = 0        # sequence number of the next part
        self._part_cache = collections.OrderedDict()  # id(obj) -> (seq, obj)
        # (experience number, oldest part seq it references): sliding-window minimum
        # over the live experiences in append order (_note_live)
        self._live_min_seq = collections.deque()

    # -- reference API ------------------------------------------------------
    @property
    def capacity(self):
        return self._capacity

    def __len__(self):
        return min(self._n_total, self._alloc_capacity)

    def append(self, state, action, reward, next_state=None, next_action=None,
               is_state_terminal=False, env_id=0, **kwargs):
        # n-step window: pfrl/replay_buffers/replay_buffer.py:33-62
        if self.store is None:
            self._create_store(state, action)
        s_slots, s_min = self._parts_of(state)
        if next_state is None:
            n_slots, n_min = s_slots, s_min
        else:
            n_slots, n_min = self._parts_of(next_state)
        rec = (s_slots, self.layout._action_array(action).tobytes(), float(reward), n_slots,
               bool(is_state_terminal), min(s_min, n_min))
        window = self.last_n_transitions[env_id]
        window.append(rec)
        if is_state_terminal:
            while window:
                self._emit(window)
                window.popleft()
        elif len(window) == self.num_steps:
            self._emit(window)

    def stop_current_episode(self, env_id=0):
        # pfrl/replay_buffers/replay_buffer.py:64-76
        window = self.last_n_transitions[env_id]
        if 0 < len(window) < self.num_steps:
            self._emit(window)
        if 0 < len(window) <= self.num_steps:
            window.popleft()
        while window:
            self._emit(window)
            window.popleft()

    def save(self, filename):
        from pfrl_b200.replay_buffers import persistence

        persistence.save_buffer(self, filename)

    def load(self, filename):
        from pfrl_b200.replay_buffers import persistence

        persistence.load_buffer(self, filename)

    def append_trajectory(self, frames, actions, rewards, terminals=None, env_id=0):
        """Bulk-append one environment's pre-recorded trajectory.

        ``frames``: uint8 array / CUDA tensor ``[T + stack, *frame_shape]``;
        the observation at step t is ``frames[t : t + stack]`` (frame
        stacking with shared frames, like VectorFrameStack + LazyFrames).
        ``actions[T]``, ``rewards[T]``, ``terminals[T]`` describe the T
        transitions.  Produces exactly the experiences the per-transition
        ``append`` would (n-step windows, shorter tails at terminals; an
        unfinished tail at the end is NOT emitted), in the same order, but
        assembles them with vectorised numpy and uploads the frames in one
        copy.  ``stack`` is taken from the buffer layout if it exists, else
        must be given by a previous ``append``/``configure``.
        """
        if self._pend_exp or self._pend_parts:
            self._flush()
        T = len(actions)
        stack = self._traj_stack
        assert frames.shape[0] == T + stack
        if terminals is None:
            terminals = np.zeros(T, dtype=bool)
        terminals = np.asarray(terminals, dtype=bool)
        if self.store is None:
            # infer the layout from a LazyFrames-like view of the first observation
            # (frames get a leading stack axis: (84, 84) -> (1, 84, 84))
            def _as_part(f):
                if isinstance(f, torch.Tensor):
                    return f[None] if f.dim() == 2 else f
                f = np.asarray(f)
                return f[None] if f.ndim == 2 else f

            first_obs = type("_FirstObs", (), {})()
            first_obs._frames = [_as_part(frames[i]) for i in range(stack)]
            self._create_store(first_obs, actions[0])
        lay = self.layout
        n_frames = frames.shape[0]
        assert n_frames <= self._part_capacity
        # upload the frames: sequential ring slots
        if isinstance(frames, torch.Tensor):
            fb = frames.contiguous().view(n_frames, -1)
            assert fb.shape[1] == lay.part_bytes, "frame bytes must be a multiple of 16"
            slots = self.store.put_parts(fb)
        else:
            fb = np.ascontiguousarray(frames).reshape(n_frames, -1).view(np.uint8)
            assert fb.shape[1] == lay.part_bytes, "frame bytes must be a multiple of 16"
            slots = self.store.put_parts(fb)
        seq0 = self._part_head
        self._part_head += n_frames
        slots = slots.astype(np.int64)
        # n-step windows: experience starting at s covers [s, e], e = min(s+n-1, episode end)
        n = self.num_steps
        nxt_term = np.full(T + 1, T + n, dtype=np.int64)  # next terminal step at or after t
        for t in range(T - 1, -1, -1):
            nxt_term[t] = t if terminals[t] else nxt_term[t + 1]
        starts = np.arange(T, dtype=np.int64)
        ends = np.minimum(starts + n - 1, nxt_term[:T])
        keep = ends <= T - 1
        starts, ends = starts[keep], ends[keep]
        m = len(starts)
        lens = (ends - starts + 1).astype(np.uint8)
        offs = np.arange(stack, dtype=np.int64)
        sp = slots[starts[:, None] + offs[None, :]].astype(np.int32)
        nx = slots[ends[:, None] + 1 + offs[None, :]].astype(np.int32)
        rw = np.zeros((m, n), dtype=np.float64)
        rewards = np.asarray(rewards, dtype=np.float64)
        for i in range(n):
            ok = starts + i <= ends
            rw[ok, i] = rewards[starts[ok] + i]
        term = terminals[ends].astype(np.uint8)
        act = np.stack([lay._action_array(a) for a in np.asarray(actions)[starts]]) \
            if lay.action_shape != () else np.asarray(actions, dtype=lay.action_dtype)[starts]
        cap = self._alloc_capacity
        for lo in range(0, m, cap):
            hi = min(m, lo + cap)
            self.store.append(sp[lo:hi], nx[lo:hi], np.ascontiguousarray(act[lo:hi]),
                              rw[lo:hi], lens[lo:hi], term[lo:hi])
        self._note_live(self._n_total, (seq0 + starts).tolist())
        self._n_total += m
        self._check_live_parts()
        return m

    _traj_stack = 4

    # -- internals ----------------------------------------------------------
    def _create_store(self, state, action):
        self.layout = lay = _Layout(state, action)
        dev = self._device_arg
        if dev is None:
            dev = torch.cuda.current_device()
        elif isinstance(dev, torch.device):
            dev = dev.index if dev.index is not None else torch.cuda.current_device()
        cap = self._alloc_capacity
        pc = self._part_capacity_arg
        if pc is None:
            pc = 2 * cap + 4096
        self.store = DeviceReplayStore(
            cap, lay.part_bytes, stack=lay.stack, n_step=self.num_steps,
            action_bytes=lay.action_bytes, prioritized=self._prioritized,
            part_capacity=pc, device=int(dev), max_batch=self._max_batch)
        self._part_capacity = pc
        self.device = self.store.device

    def _part_seq(self, obj):
        """Sequence number of the ring part holding ``obj`` (uploading it if it
        is new).  Identity-based sharing = LazyFrames' frame sharing."""
        key = id(obj)
        hit = self._part_cache.get(key)
        if hit is not None and hit[1] is obj and hit[0] > self._part_head - self._part_capacity:
            return hit[0]
        seq = self._part_head
        self._part_head += 1
        self._pend_parts.append(obj)
        self._part_cache[key] = (seq, obj)
        if len(self._part_cache) > 8192:
            self._part_cache.popitem(last=False)
        # one upload never holds more parts than the ring (put_parts refuses that)
        if len(self._pend_parts) >= min(1024, self._part_capacity):
            self._flush_parts()
        return seq

    def _parts_of(self, obs):
        frames = getattr(obs, "_frames", None)
        if frames is None:
            frames = (obs,)
        seqs = [self._part_seq(f) for f in frames]
        pc = self._part_capacity
        return tuple(s % pc for s in seqs), min(seqs)

    def _emit(self, window):
        first, last = window[0], window[-1]
        rewards = [r[2] for r in window]
        term = any(r[4] for r in window)
        min_seq = min(r[5] for r in window)
        self._pend_exp.append((first[0], last[3], first[1], rewards, len(window), term,
                               self._new_priority()))
        self._note_live(self._n_total, (min_seq,))
        self._n_total += 1
        if self._capacity is None and self._n_total > self._alloc_capacity:
            raise MemoryError(
                "unbounded (capacity=None) device buffer outgrew its %d-experience allocation; "
                "pass unbounded_capacity=... to reserve more" % self._alloc_capacity)
        if len(self._pend_exp) >= 4096:
            self._flush()

    def _note_live(self, first, seqs):
        """Experiences number first, first + 1, ... became live; seqs[j] (non-decreasing)
        is the sequence number of the oldest part that experience first + j references.
        A later experience can reference an older part than the ones before it (a part
        reused through the identity cache, e.g. an env that hands out the same reset
        observation again), so the overrun check needs the minimum over all live
        experiences, not the oldest experience's: the deque keeps the candidates, seqs
        non-decreasing front to back."""
        if not seqs:
            return
        q = self._live_min_seq
        keep = self._alloc_capacity
        if len(seqs) > keep:  # only the last `capacity` of them stay live
            first += len(seqs) - keep
            seqs = seqs[-keep:]
        while q and q[-1][1] >= seqs[0]:
            q.pop()
        q.extend(zip(range(first, first + len(seqs)), seqs))
        while q[0][0] < first + len(seqs) - keep:
            q.popleft()  # evicted from the record ring

    def _check_live_parts(self):
        """MemoryError if a live experience references a part that the ring has already
        overwritten (sample() would silently return another observation)."""
        q = self._live_min_seq
        if q and self._part_head - q[0][1] > self._part_capacity:
            raise MemoryError(
                "part ring overrun: live experiences reference parts that were overwritten; "
                "construct the buffer with a larger part_capacity (now %d)" % self._part_capacity)

    def _new_priority(self):
        return None

    def _flush_parts(self):
        parts = self._pend_parts
        if not parts:
            return
        self._pend_parts = []
        lay = self.layout
        on_dev = [isinstance(p, torch.Tensor) and p.is_cuda for p in parts]
        if all(on_dev):
            flat = torch.stack([p.reshape(-1) for p in parts]).view(torch.uint8)
            if lay.part_nbytes != lay.part_bytes:
                buf = torch.zeros((len(parts), lay.part_bytes), dtype=torch.uint8,
                                  device=self.device)
                buf[:, :lay.part_nbytes] = flat
                flat = buf
            slots = self.store.put_parts(flat.contiguous())
        else:
            buf = np.zeros((len(parts), lay.part_bytes), dtype=np.uint8)
            np_dtype = lay.part_dtype if not isinstance(lay.part_dtype, torch.dtype) else \
                torch.empty(0, dtype=lay.part_dtype).numpy().dtype
            for i, p in enumerate(parts):
                if isinstance(p, torch.Tensor):
                    p = p.detach().cpu().numpy()
                a = np.ascontiguousarray(np.asarray(p, dtype=np_dtype))
                buf[i, :lay.part_nbytes] = a.reshape(-1).view(np.uint8)
            slots = self.store.put_parts(buf)
        expect = (self._part_head - len(parts)) % self._part_capacity
        assert int(slots[0]) == expect, "part ring bookkeeping out of sync"

    def _flush(self):
        self._flush_parts()
        # also with nothing pending: parts uploaded since the last flush may have
        # overwritten what live experiences reference
        self._check_live_parts()
        pend = self._pend_exp
        if not pend:
            return
        self._pend_exp = []
        cap = self._alloc_capacity
        lay = self.layout
        for lo in range(0, len(pend), cap):
            chunk = pend[lo:lo + cap]
            n = len(chunk)
            sp = np.array([c[0] for c in chunk], dtype=np.int32).reshape(n, lay.stack)
            nx = np.array([c[1] for c in chunk], dtype=np.int32).reshape(n, lay.stack)
            act = np.frombuffer(b"".join(c[2] for c in chunk), dtype=np.uint8)
            rw = np.zeros((n, self.num_steps), dtype=np.float64)
            for i, c in enumerate(chunk):
                rw[i, :c[4]] = c[3]
            ln = np.array([c[4] for c in chunk], dtype=np.uint8)
            tm = np.array([c[5] for c in chunk], dtype=np.uint8)
            prio = None
            if self._prioritized and chunk[0][6] is not None:
                prio = np.array([c[6] for c in chunk], dtype=np.float64)
            self.store.append(sp, nx, act, rw, ln, tm, priority=prio)

    def _gamma_pow(self, gamma):
        # CPython float pow, like `gamma ** i` / `gamma ** len(elem)` in the
        # reference (pfrl/replay_buffer.py:186,203)
        return [gamma ** i for i in range(self.num_steps + 1)]

    def _gather(self, exps, gamma, phi, raw=False, want_steps=False):
        lay = self.layout
        mode = None if raw else getattr(phi, "b2rl_obs_mode", None)
        index = None if exps.pending else exps.index
        common = dict(index=index, action_dtype=lay.torch_action_dtype(),
                      action_shape=lay.action_shape, want_steps=want_steps)
        gp = self._gamma_pow(gamma)
        key = self._plan_key(gamma, phi, raw)
        pre = None
        if not want_steps and exps._prefetched is not None and exps._prefetch_key == key:
            pre = dict(exps._prefetched)  # outputs of the fused step launch
        elif self._prioritized and exps.pending and not want_steps and not raw:
            # remember what the agent asks for: the next sample() gathers in the
            # same launch as it draws (b2rl_replay_step)
            self._plan = (key, gamma, phi, raw)
        if mode == _lib.OBS_U8_TO_F32:
            assert lay.torch_obs_dtype() == torch.uint8
            padded = lay.part_nbytes != lay.part_bytes
            if pre is not None:
                out = pre
                if not padded:
                    for k in ("state", "next_state"):
                        out[k] = out[k].view((exps.n,) + tuple(lay.obs_shape))
            else:
                out = self.store.gather(exps.n, gp, obs_mode=mode, obs_scale=phi.b2rl_obs_scale,
                                        obs_shape=None if padded else lay.obs_shape, **common)
            if padded:  # parts are padded to 16 B in the ring: drop the pad columns
                for k in ("state", "next_state"):
                    t = out[k].view(exps.n, lay.stack, lay.part_bytes)[:, :, :lay.part_nbytes]
                    out[k] = t.contiguous().view((exps.n,) + tuple(lay.obs_shape))
        else:
            out = pre if pre is not None else self.store.gather(
                exps.n, gp, obs_mode=_lib.OBS_RAW, **common)
            for k in ("state", "next_state"):
                t = out[k]  # [n, stack * part_bytes] uint8
                if lay.part_nbytes != lay.part_bytes:
                    t = t.view(exps.n, lay.stack, lay.part_bytes)[:, :, :lay.part_nbytes].contiguous()
                out[k] = t.view(exps.n, -1).view(lay.torch_obs_dtype()).view(
                    (exps.n,) + tuple(lay.obs_shape))
            if mode is None and not raw:
                # arbitrary host phi: reference behaviour (phi per observation on
                # the host, collate, copy back) -- slow but exact
                from pfrl_b200.utils.batch_states import batch_states

                for k in ("state", "next_state"):
                    host = out[k].cpu().numpy()
                    out[k] = batch_states(list(host), self.device, phi)
        if exps.weights is not None:
            out["weights"] = exps.weights
        return out

    @staticmethod
    def _plan_key(gamma, phi, raw):
        mode = None if raw else getattr(phi, "b2rl_obs_mode", None)
        if mode == _lib.OBS_U8_TO_F32:
            return (float(gamma), int(mode), float(phi.b2rl_obs_scale))
        return (float(gamma), int(_lib.OBS_RAW), 1.0)

    def _materialise(self, exps):
        out = self._gather(exps, 1.0, None, raw=True, want_steps=True)
        if self.device.type == "cuda":
            torch.cuda.current_stream().synchronize()
        st = out["state"].cpu().numpy()
        ns = out["next_state"].cpu().numpy()
        ac = out["action"].cpu().numpy()
        sr = out["step_rewards"].cpu().numpy()
        ln = out["len"].cpu().numpy()
        tm = out["is_state_terminal"].cpu().numpy()
        w = exps.weights.cpu().numpy() if exps.weights is not None else None
        lists = []
        for k in range(exps.n):
            L = int(ln[k])
            steps = []
            for j in range(L):
                steps.append(dict(
                    state=st[k] if j == 0 else None,
                    action=(ac[k].item() if ac[k].shape == () else ac[k]) if j == 0 else None,
                    reward=float(sr[k, j]),
                    next_state=ns[k] if j == L - 1 else None,
                    next_action=None,
                    is_state_terminal=bool(tm[k]) and j == L - 1,
                ))
            if w is not None:
                steps[0]["weight"] = float(w[k])
            lists.append(steps)
        return lists


class ReplayBuffer(DeviceNStepBuffer):
    """Uniform experience replay (pfrl/replay_buffers/replay_buffer.py:11-94)
    with the store in HBM.  ``sample`` draws its distinct indices on the host
    with the reference's ``sample_n_k`` stream and gathers on the device."""

    _prioritized = False

    def sample(self, num_experiences):
        assert len(self) >= num_experiences
        self._flush()
        idx = sample_n_k(len(self), num_experiences)
        index = torch.as_tensor(np.asarray(idx, dtype=np.int64)).to(self.device, non_blocking=True)
        return DeviceExperiences(self, num_experiences, index=index)


class PriorityWeightError(object):
    """Proportional prioritisation parameters and host-side arithmetic
    (pfrl/replay_buffers/prioritized.py:10-66)."""

    def __init__(self, alpha, beta0, betasteps, eps, normalize_by_max, error_min, error_max):
        assert 0.0 <= alpha
        assert 0.0 <= beta0 <= 1.0
        self.alpha = alpha
        self.beta = beta0
        self.beta_add = 0 if betasteps is None else (1.0 - beta0) / betasteps
        self.eps = eps
        if normalize_by_max is True:
            normalize_by_max = "batch"
        assert normalize_by_max in [False, "batch", "memory"]
        self.normalize_by_max = normalize_by_max
        self.error_min = error_min
        self.error_max = error_max

    def priority_from_errors(self, errors):
        lo, hi, eps, alpha = self.error_min, self.error_max, self.eps, self.alpha
        out = []
        for d in errors:
            if lo is not None:
                d = max(lo, d)
            if hi is not None:
                d = min(hi, d)
            out.append((d + eps) ** alpha)
        return out

    def weights_from_probabilities(self, probabilities, min_probability):
        """Host form of the importance weights (replay_buffers/prioritized.py:57-66),
        for code that calls it directly; ``sample()`` computes the same numbers on the
        device (k_weights).  Advances the beta schedule like the reference."""
        if self.normalize_by_max == "batch":
            min_probability = np.min(probabilities)
        if self.normalize_by_max:
            weights = [(p / min_probability) ** -self.beta for p in probabilities]
        else:
            weights = [(len(self) * p) ** -self.beta for p in probabilities]
        self.beta = min(1.0, self.beta + self.beta_add)
        return weights


class PrioritizedReplayBuffer(DeviceNStepBuffer, PriorityWeightError):
    """Proportional prioritised replay (pfrl/replay_buffers/prioritized.py:
    69-126) on GPU segment trees.

    ``sample_mode="exact"`` (default) reproduces the reference's sampled
    indices bit for bit under the same numpy seed; ``"parallel"`` draws all
    indices concurrently on the frozen tree (with replacement).
    """

    _prioritized = True

    def __init__(self, capacity=None, alpha=0.6, beta0=0.4, betasteps=2e5, eps=0.01,
                 normalize_by_max=True, error_min=0, error_max=1, num_steps=1, *,
                 device=None, part_capacity=None, max_batch=4096, sample_mode="exact",
                 unbounded_capacity=_UNBOUNDED_DEFAULT, fused=True):
        DeviceNStepBuffer.__init__(self, capacity, num_steps, device=device,
                                   part_capacity=part_capacity, max_batch=max_batch,
                                   unbounded_capacity=unbounded_capacity)
        PriorityWeightError.__init__(self, alpha, beta0, betasteps, eps, normalize_by_max,
                                     error_min=error_min, error_max=error_max)
        assert sample_mode in ("exact", "parallel")
        self.sample_mode = sample_mode
        self._waiting = False
        # fused=True: once batch_experiences has been seen with a device-side phi,
        # sample() draws, weighs and gathers in ONE launch (b2rl_replay_step) and a
        # CUDA-tensor update_errors() is folded into the head of the next one.  The
        # results are those of the separate calls (tests/test_fused_step_gpu.py).
        self.fused = fused
        self._plan = None

    def sample(self, n):
        assert len(self) >= n
        # sample / update_errors must alternate (collections/prioritized.py:98)
        assert not self._waiting
        self._flush()
        # one legacy-MT double per draw, in order: np.random.uniform(0.0, root)
        # consumes exactly random_sample() (collections/prioritized.py:302)
        u = np.random.random_sample(n)
        mode = _lib.SAMPLE_EXACT if self.sample_mode == "exact" else _lib.SAMPLE_PARALLEL
        norm = {False: _lib.NORM_NONE, "batch": _lib.NORM_BATCH, "memory": _lib.NORM_MEMORY}[
            self.normalize_by_max]
        pre = key = None
        if self.fused and self._plan is not None and hasattr(self.store, "step"):
            key, gamma, phi, raw = self._plan
            lay = self.layout
            pre = self.store.step(
                u, self._gamma_pow(gamma), self.beta, norm, mode=mode, obs_mode=key[1],
                obs_scale=key[2], action_dtype=lay.torch_action_dtype(),
                action_shape=lay.action_shape)
            index, weights = pre.pop("index"), pre.pop("weights")
        else:
            index, _ = self.store.sample(u, mode=mode, want_priority=False)
            weights = self.store.weights(n, self.beta, norm)
        self.beta = min(1.0, self.beta + self.beta_add)  # prioritized.py:65
        self._waiting = True
        self._last_n = n
        self._last_handle = DeviceExperiences(self, n, index=index, weights=weights, pending=True)
        self._last_handle._prefetched = pre
        self._last_handle._prefetch_key = key
        return self._last_handle

    def update_errors(self, errors):
        """TD errors of the last sample -> new priorities.

        A CUDA tensor stays on the device (fused clip / +eps / pow / tree
        write-back); any host sequence goes through the reference's exact
        Python-float formula so that seeded runs stay bit-identical."""
        assert self._waiting  # collections/prioritized.py:108
        assert len(errors) == self._last_n  # :110
        if isinstance(errors, torch.Tensor) and errors.is_cuda:
            e = errors.detach()
            if e.dtype not in (torch.float32, torch.float64):
                e = e.float()
            if self.fused and self._plan is not None and hasattr(self.store, "defer_errors"):
                # no launch: folded into the head of the next fused step (or applied
                # before the next append / tree access, whichever comes first)
                self.store.defer_errors(e.contiguous().view(-1), self.alpha, self.eps,
                                        self.error_min, self.error_max)
            else:
                self.store.update_errors(e.contiguous().view(-1), self.alpha, self.eps,
                                         self.error_min, self.error_max)
        elif hasattr(self.store, "update_host_errors"):
            # host floats: the reference's list comprehension (max / min / + eps / ** alpha in
            # Python floats) evaluated inside the library with the same libm pow, one call;
            # with the fused step planned, the write-back rides on the next launch
            if isinstance(errors, torch.Tensor):
                errors = errors.detach().cpu().numpy()
            try:
                self.store.update_host_errors(
                    errors, self.alpha, self.eps, self.error_min, self.error_max,
                    defer=self.fused and self._plan is not None)
            except _lib.B2rlError as exc:
                if "must be > 0" in str(exc):
                    raise AssertionError(str(exc))  # collections/prioritized.py:109
                raise
        else:
            if isinstance(errors, torch.Tensor):
                errors = errors.tolist()
            pr = self.priority_from_errors(errors)
            assert all(p > 0.0 for p in pr)  # collections/prioritized.py:109
            self.store.update_priorities(np.asarray(pr, dtype=np.float64))
        self._waiting = False
        # the handle's "slots of the pending sample" are gone; it can still be
        # gathered / materialised through its logical indices
        self._last_handle.pending = False
        self._last_handle = None
