"""HBM-resident episodic replay buffer for recurrent agents (DRQN).

Same constructor and methods as pfrl/replay_buffers/episodic.py:9-98.  The
observations and records live in the part ring and record store of
``DeviceNStepBuffer`` (with ``num_steps=1``); what this class adds:

  * an episode table on the host: (first absolute record index, length) of
    every live episode, in commit order.  An episode's records are appended
    to the store together when it is committed, so an episode is always a run
    of consecutive ring slots;
  * eviction in whole episodes: the oldest episodes are dropped *before* the
    new one's records are appended, so the store (which keeps the last
    ``capacity`` records) never evicts a record of a live episode;
  * part liveness over episodes: commit order is not upload order (an env's
    long episode can start before another env's short one and be committed
    after it), so the part-ring overrun check uses the oldest part referenced
    by any live episode or any uncommitted current episode;
  * a recurrent-state ring in HBM: ``recurrent_state`` / ``next_recurrent_state``
    of every transition (device tensors, numpy arrays or None; any nesting of
    tuples) flattened to one row of fp32 words each, at row ``absolute index % capacity``.
    A leaf keeps the dtype it was appended in: 4- and 8-byte types are stored as their
    bits, fp16 widened to fp32, and both come back unchanged;
  * a behaviour-policy ring in HBM for ACER: the ``mu`` distribution appended with a
    transition, as one row at the same row index, in the distribution's dtype (a
    ``Categorical``'s normalised logits [K], or an ``Independent(Normal, 1)``'s loc and
    scale [2A]).  The first ``mu`` fixes the layout.  The host episode table also
    records which episodes ended on a terminal, so a sampled subsequence's last
    transition is known to be terminal or not without reading the device.

``sample_episodes`` returns ``DeviceEpisodes``; ``batch_recurrent_experiences``
turns it into the packed minibatch with one kernel launch
(b2rl_replay_gather_sequences).  Indexed or iterated it materialises the
reference's list-of-lists-of-dicts form.
"""
import collections
import hashlib
import pickle

import numpy as np
import torch
from torch.nn.utils.rnn import PackedSequence

from pfrl_b200 import _lib
from pfrl_b200.collections.random_access_queue import RandomAccessQueue
from pfrl_b200.replay_buffers.device_buffer import _UNBOUNDED_DEFAULT, DeviceNStepBuffer
from pfrl_b200.utils.random import sample_n_k


def _leaves(state):
    if isinstance(state, tuple):
        out = []
        for s in state:
            out.extend(_leaves(s))
        return out
    return [state]


def _structure(state):
    """Nesting of a state: a leaf is its shape, a tuple is a tuple of structures."""
    if isinstance(state, tuple):
        return tuple(_structure(s) for s in state)
    return tuple(state.shape)


def _rebuild(structure, leaves):
    it = iter(leaves)

    def build(s):
        if isinstance(s, tuple) and (not s or isinstance(s[0], tuple)):
            return tuple(build(x) for x in s)
        return next(it)

    return build(structure)


class DeviceEpisodes(collections.abc.Sequence):
    """The result of ``EpisodicReplayBuffer.sample_episodes``: n (sub)episodes
    that still live in HBM, described by absolute record ranges."""

    def __init__(self, buffer, first, length, end, last_terminal=None):
        self.buffer = buffer
        self.first = np.asarray(first, dtype=np.int64)    # absolute record index
        self.length = np.asarray(length, dtype=np.int32)
        self.end = np.asarray(end, dtype=np.int64)        # one past the episode's last record
        # whether each (sub)episode's last transition is terminal (host)
        self.last_terminal = (np.zeros(len(self.length), dtype=bool) if last_terminal is None
                              else np.asarray(last_terminal, dtype=bool))
        self._lists = None

    def __len__(self):
        return len(self.length)

    def sorted_by_length(self):
        """Stable sort, longest first: what ``sorted(episodes, key=len,
        reverse=True)`` does to the materialised lists."""
        order = np.argsort(-self.length, kind="stable")
        return DeviceEpisodes(self.buffer, self.first[order], self.length[order],
                              self.end[order], self.last_terminal[order])

    def batch(self, gamma, phi, device=None):
        """Device-side batch_recurrent_experiences (pfrl/replay_buffer.py:219-287)."""
        return self.buffer._gather_sequences(self, gamma, phi)

    def _materialise(self):
        if self._lists is None:
            self._lists = self.buffer._materialise_episodes(self)
        return self._lists

    def __getitem__(self, i):
        return self._materialise()[i]

    def __iter__(self):
        return iter(self._materialise())


class EpisodicReplayBuffer(DeviceNStepBuffer):
    """Episodic experience replay (pfrl/replay_buffers/episodic.py:9-98) with the
    store in HBM."""

    _prioritized = False

    def __init__(self, capacity=None, *, device=None, part_capacity=None, max_batch=4096,
                 unbounded_capacity=_UNBOUNDED_DEFAULT):
        DeviceNStepBuffer.__init__(self, capacity, 1, device=device, part_capacity=part_capacity,
                                   max_batch=max_batch, unbounded_capacity=unbounded_capacity)
        self.current_episode = collections.defaultdict(list)  # env_id -> [(rec, rs, next_rs)]
        self._episodes = RandomAccessQueue()   # (abs first, length, oldest part seq), commit order
        self._n_live = 0                       # transitions of the live episodes
        self._ep_count = 0                     # episodes ever committed
        self._min_seq = collections.deque()    # (episode number, seq): sliding-window minimum
        self._rs_struct = None                 # structure of the first non-None state
        self._rs_dtypes = None                 # appended dtype of every leaf
        self._rs_leaves = None                 # [(offset, d0, inner)] per leaf, in fp32 words
        self._rs_ring = None                   # [alloc, 2, D] fp32 words (HBM)
        self._rs_present = None                # [alloc, 2] uint8 (HBM)
        self._rs_present_host = None           # host mirror of _rs_present
        self._pend_rs = []                     # (ring row * 2 + side, flat row or None)
        self._current_mu = collections.defaultdict(list)  # env_id -> [mu row or None]
        self._terminal_ends = set()            # abs end of the live episodes ending terminal
        self._mu_layout = None                 # (distribution class, width, dtype) of the first mu
        self._mu_ring = None                   # [alloc, width] in that dtype (HBM)
        self._mu_present_host = None           # [alloc] bool
        self._pend_mu = []                     # (ring row, mu row or None)

    # -- reference API ------------------------------------------------------
    def __len__(self):
        return self._n_live

    @property
    def n_episodes(self):
        return len(self._episodes)

    def append(self, state, action, reward, next_state=None, next_action=None,
               is_state_terminal=False, env_id=0, **kwargs):
        if self.store is None:
            self._create_store(state, action)
        s_slots, s_min = self._parts_of(state)
        if next_state is None:
            n_slots, n_min = s_slots, s_min
        else:
            n_slots, n_min = self._parts_of(next_state)
        rec = (s_slots, self.layout._action_array(action).tobytes(), float(reward), n_slots,
               bool(is_state_terminal), min(s_min, n_min))
        # everything that can refuse the transition runs before any of it is kept
        rs = self._flat_state(kwargs.get("recurrent_state"))
        nrs = self._flat_state(kwargs.get("next_recurrent_state"))
        mu = self._flat_mu(kwargs.get("mu"))
        self.current_episode[env_id].append((rec, rs, nrs))
        self._current_mu[env_id].append(mu)
        if is_state_terminal:
            self.stop_current_episode(env_id=env_id)

    def stop_current_episode(self, env_id=0):
        episode = self.current_episode.pop(env_id, None)
        mus = self._current_mu.pop(env_id, None)
        if not episode:
            return
        L = len(episode)
        cap = self._capacity
        if cap is not None:
            # drop whole oldest episodes first: afterwards the live records are the
            # last <= capacity records of the store, which keeps exactly those
            while len(self._episodes) and self._n_live + L > cap:
                f, L_old, _ = self._episodes.popleft()
                self._n_live -= L_old
                self._terminal_ends.discard(f + L_old)
            if L > cap:
                return  # longer than the whole buffer: the reference drops it too
        elif self._n_total + L > self._alloc_capacity:
            raise MemoryError(
                "unbounded (capacity=None) device buffer outgrew its %d-experience allocation; "
                "pass unbounded_capacity=... to reserve more" % self._alloc_capacity)
        first = self._n_total
        for j, (rec, rs, nrs) in enumerate(episode):
            self._pend_exp.append((rec[0], rec[3], rec[1], [rec[2]], 1, rec[4], None))
            row = (first + j) % self._alloc_capacity
            if rs is not None or nrs is not None or self._rs_struct is not None:
                self._pend_rs.append((row * 2, rs))
                self._pend_rs.append((row * 2 + 1, nrs))
            if self._mu_layout is not None:
                self._pend_mu.append((row, mus[j]))
        self._n_total += L
        self._n_live += L
        seq = min(rec[5] for rec, _, _ in episode)
        self._episodes.append((first, L, seq))
        if episode[-1][0][4]:
            self._terminal_ends.add(first + L)
        while self._min_seq and self._min_seq[-1][1] >= seq:
            self._min_seq.pop()
        self._min_seq.append((self._ep_count, seq))
        self._ep_count += 1
        if len(self._pend_exp) >= 4096:
            self._flush()

    def sample(self, n):
        """n transitions, uniformly (sample_n_k) over the live episodes' records."""
        from pfrl_b200.replay_buffers.device_buffer import DeviceExperiences

        assert self._n_live >= n
        self._flush()
        lo = min(self._n_total, self._alloc_capacity) - self._n_live
        idx = np.asarray(sample_n_k(self._n_live, n), dtype=np.int64) + lo
        index = torch.as_tensor(idx).to(self.device, non_blocking=True)
        return DeviceExperiences(self, n, index=index)

    def sample_episodes(self, n_episodes, max_len=None):
        """n distinct episodes (sample_n_k), each cut to a random window of
        max_len transitions (one np.random.randint per longer episode, in sample
        order, like random_subseq)."""
        assert len(self._episodes) >= n_episodes
        picked = [self._episodes[i] for i in sample_n_k(len(self._episodes), n_episodes)]
        first, length, end, term = [], [], [], []
        for f, L, _ in picked:
            start, n = f, L
            if max_len is not None and L > max_len:
                start = f + np.random.randint(0, L - max_len + 1)
                n = max_len
            first.append(start)
            length.append(n)
            end.append(f + L)
            term.append(start + n == f + L and f + L in self._terminal_ends)
        return DeviceEpisodes(self, first, length, end, term)

    def save(self, filename):
        """Own format: the pickled live episodes in the reference's transition dicts, with
        every transition's states as numpy.  Frame-stacked observations are saved as
        ``LazyFrames`` whose equal frames are one shared array, so a loaded buffer keeps
        the layout and stores every frame once, as the saved one did."""
        episodes = self._all_episodes()
        lay = self.layout
        if lay is not None and lay.lazy:
            from pfrl_b200.utils.lazy_frames import LazyFrames

            shared = {}

            def frames_of(obs):
                parts = []
                for x in np.split(np.asarray(obs), lay.stack, axis=0):
                    x = np.ascontiguousarray(x).reshape(lay.part_shape)
                    key = hashlib.blake2b(x, digest_size=16).digest()  # 128-bit content key
                    parts.append(shared.setdefault(key, x))
                return LazyFrames(parts, stack_axis=0)

            for ep in episodes:
                for t in ep:
                    t["state"] = frames_of(t["state"])
                    t["next_state"] = frames_of(t["next_state"])
        with open(filename, "wb") as f:
            pickle.dump(episodes, f)

    def load(self, filename):
        with open(filename, "rb") as f:
            episodes = pickle.load(f)
        self.__init__(self._capacity, device=self._device_arg,
                      part_capacity=self._part_capacity_arg, max_batch=self._max_batch,
                      unbounded_capacity=self._alloc_capacity if self._capacity is None
                      else _UNBOUNDED_DEFAULT)
        for ep in episodes:
            for t in ep:
                self.append(**t)
            self.stop_current_episode()

    def append_trajectory(self, *args, **kwargs):
        raise NotImplementedError(
            "EpisodicReplayBuffer keeps an episode table: append transitions with append()")

    # -- recurrent states -----------------------------------------------------
    def _flat_state(self, state):
        if state is None:
            return None
        leaves = [x.detach() if isinstance(x, torch.Tensor)
                  else torch.from_numpy(np.ascontiguousarray(x)) for x in _leaves(state)]
        dtypes = tuple(x.dtype for x in leaves)
        if self._rs_struct is None:
            specs, off = [], 0
            for x in leaves:
                shape = tuple(x.shape)
                assert len(shape) >= 1, "recurrent state tensors need at least one axis"
                inner = int(np.prod(shape[1:])) if len(shape) > 1 else 1
                inner *= _state_words(x.dtype)
                specs.append((off, shape[0], inner))
                off += shape[0] * inner
            assert len(specs) <= _lib.SEQ_MAX_LEAVES
            self._rs_struct = _structure(state)
            self._rs_dtypes = dtypes
            self._rs_leaves = specs
            self._rs_width = off
        assert _structure(state) == self._rs_struct, "recurrent state layout changed"
        if dtypes != self._rs_dtypes:
            raise TypeError("recurrent state dtypes changed: %s, the buffer holds %s"
                            % (dtypes, self._rs_dtypes))
        parts = [_state_to_words(x).reshape(-1) for x in leaves]
        return parts[0] if len(parts) == 1 else torch.cat(parts)

    def _flush_states(self):
        pend = self._pend_rs
        if not pend:
            return
        self._pend_rs = []
        if self._rs_struct is None:
            return  # only None states so far: nothing to store
        dev = self.device
        if self._rs_ring is None:
            self._rs_ring = torch.zeros((self._alloc_capacity, 2, self._rs_width),
                                        dtype=torch.float32, device=dev)
            self._rs_present = torch.zeros((self._alloc_capacity, 2), dtype=torch.uint8,
                                           device=dev)
            self._rs_present_host = np.zeros((self._alloc_capacity, 2), dtype=np.uint8)
        # more than `capacity` pending transitions reuse ring rows: only the last
        # write of a row may reach the scatter (duplicate indices have no order)
        pend = list({k: (k, r) for k, r in pend}.values())
        keys = np.array([k for k, _ in pend], dtype=np.int64)
        flags = np.array([r is not None for _, r in pend], dtype=np.uint8)
        self._rs_present_host.reshape(-1)[keys] = flags
        self._rs_present.view(-1)[torch.as_tensor(keys).to(dev)] = \
            torch.as_tensor(flags).to(dev)
        have = [(k, r) for k, r in pend if r is not None]
        if have:
            rows = torch.stack([r if r.device == dev else r.to(dev) for _, r in have])
            idx = torch.as_tensor(np.array([k for k, _ in have], dtype=np.int64)).to(dev)
            self._rs_ring.view(-1, self._rs_width).index_copy_(0, idx, rows)

    # -- behaviour policies (ACER's mu) -------------------------------------------
    def _flat_mu(self, mu):
        """One row of ``mu`` in its dtype (a device or host tensor; no copy to the host)."""
        if mu is None:
            return None
        D = torch.distributions
        if type(mu) is D.Categorical:
            row = mu.logits.detach().reshape(-1)
        elif (type(mu) is D.Independent and type(mu.base_dist) is D.Normal
              and mu.reinterpreted_batch_ndims == 1):
            row = torch.cat([mu.base_dist.loc.detach().reshape(-1),
                             mu.base_dist.scale.detach().reshape(-1)])
        else:
            raise NotImplementedError(
                "EpisodicReplayBuffer stores mu as a Categorical or an Independent(Normal, 1) "
                "distribution, got %s" % type(mu).__name__)
        layout = (type(mu), int(row.numel()), row.dtype)
        if self._mu_layout is None:
            self._mu_layout = layout
        assert layout == self._mu_layout, \
            "mu layout changed: %s of width %d (%s), the buffer holds %s of width %d (%s)" % (
                layout[0].__name__, layout[1], layout[2], self._mu_layout[0].__name__,
                self._mu_layout[1], self._mu_layout[2])
        return row

    def _flush_mu(self):
        pend = self._pend_mu
        if not pend:
            return
        self._pend_mu = []
        dev = self.device
        if self._mu_ring is None:
            self._mu_ring = torch.zeros((self._alloc_capacity, self._mu_layout[1]),
                                        dtype=self._mu_layout[2], device=dev)
            self._mu_present_host = np.zeros(self._alloc_capacity, dtype=bool)
        # only the last write of a ring row may reach the scatter
        pend = list({k: (k, r) for k, r in pend}.values())
        self._mu_present_host[[k for k, _ in pend]] = [r is not None for _, r in pend]
        have = [(k, r) for k, r in pend if r is not None]
        if have:
            rows = torch.stack([r if r.device == dev else r.to(dev) for _, r in have])
            idx = torch.as_tensor(np.array([k for k, _ in have], dtype=np.int64))
            self._mu_ring.index_copy_(0, idx.to(dev, non_blocking=True), rows)

    def _mu_distribution(self, row):
        """``row`` [width] rebuilt as the stored class with a batch axis of 1."""
        cls, width, _ = self._mu_layout
        if cls is torch.distributions.Categorical:
            return cls(logits=row[None])
        A = width // 2
        return torch.distributions.Independent(
            torch.distributions.Normal(loc=row[None, :A], scale=row[None, A:]), 1)

    def mu_rows(self, eps):
        """The [T, width] mu rows of the one subsequence in ``eps``, on the device (a run
        of consecutive ring rows, so a slice or two; no synchronisation)."""
        assert len(eps) == 1 and self._mu_layout is not None
        self._flush()
        cap = self._alloc_capacity
        r0, T = int(eps.first[0]) % cap, int(eps.length[0])
        assert self._mu_present_host[(r0 + np.arange(T)) % cap].all(), \
            "a sampled transition was appended without mu"
        if r0 + T <= cap:
            return self._mu_ring[r0:r0 + T]
        return torch.cat([self._mu_ring[r0:], self._mu_ring[:r0 + T - cap]])

    # -- internals ----------------------------------------------------------
    def _oldest_live_part(self):
        seqs = []
        while self._min_seq and self._min_seq[0][0] < self._ep_count - len(self._episodes):
            self._min_seq.popleft()  # its episode was evicted
        if self._min_seq:
            seqs.append(self._min_seq[0][1])
        for ep in self.current_episode.values():
            if ep:
                seqs.append(min(rec[5] for rec, _, _ in ep))
        return min(seqs) if seqs else None

    def _flush(self):
        self._flush_parts()
        oldest = self._oldest_live_part()
        if oldest is not None and self._part_head - oldest > self._part_capacity:
            raise MemoryError(
                "part ring overrun: live or current episodes reference parts that were "
                "overwritten; construct the buffer with a larger part_capacity (now %d)"
                % self._part_capacity)
        DeviceNStepBuffer._flush(self)  # _live_min_seq stays empty: no second check there
        self._flush_states()
        self._flush_mu()

    def _logical(self, eps):
        npop = self._n_total - min(self._n_total, self._alloc_capacity)
        return eps.first - npop, eps.end - npop

    def _gather_sequences(self, eps, gamma, phi, raw=False):
        self._flush()
        lay = self.layout
        mode = None if raw else getattr(phi, "b2rl_obs_mode", None)
        obs_mode = _lib.OBS_U8_TO_F32 if mode == _lib.OBS_U8_TO_F32 else _lib.OBS_RAW
        first, end = self._logical(eps)
        lengths = eps.length
        B = len(lengths)
        states = None
        want_states = False
        if self._rs_ring is not None and B > 0:
            rows = (eps.first % self._alloc_capacity)
            pres = self._rs_present_host[rows]
            want_states = bool(pres.any())
            if want_states:
                states = (self._rs_ring, self._rs_present, self._rs_leaves)
        out = self.store.gather_sequences(
            first, lengths, end, obs_mode=obs_mode,
            obs_scale=phi.b2rl_obs_scale if obs_mode == _lib.OBS_U8_TO_F32 else 1.0,
            action_dtype=lay.torch_action_dtype(), states=states)
        N = int(lengths.sum())
        padded = lay.part_nbytes != lay.part_bytes
        for k in ("state", "next_state"):
            t = out[k]
            if padded:  # parts are padded to 16 B in the ring: drop the pad columns
                t = t.view(N, lay.stack, -1)[:, :, :lay.part_nbytes].contiguous()
            if obs_mode == _lib.OBS_RAW:
                t = t.view(N, -1).view(lay.torch_obs_dtype())
            t = t.view((N,) + tuple(lay.obs_shape))
            if mode is None and not raw and phi is not None:
                # arbitrary host phi: the reference's per-observation phi on the host
                from pfrl_b200.utils.batch_states import batch_states

                t = batch_states(list(t.cpu().numpy()), self.device, phi)
            out[k] = t
        batch_sizes = torch.as_tensor(
            np.array([(lengths > t).sum() for t in range(int(lengths[0]))], dtype=np.int64)
            if B else np.zeros(0, dtype=np.int64))
        batch = {
            "state": PackedSequence(out["state"], batch_sizes),
            "next_state": PackedSequence(out["next_state"], batch_sizes),
            "action": out["action"].view((N,) + tuple(lay.action_shape)),
            "reward": out["reward"],
            "is_state_terminal": out["is_state_terminal"],
            "discount": torch.full((N,), gamma, dtype=torch.float32, device=self.device),
            "recurrent_state": None,
            "next_recurrent_state": None,
        }
        if want_states:
            for key, leaves in (("recurrent_state", out["state_leaves"]),
                                ("next_recurrent_state", out["next_state_leaves"])):
                shaped = []
                for x, dt, shape in zip(leaves, self._rs_dtypes,
                                        _leaves_of_structure(self._rs_struct)):
                    x = _state_from_words(x, dt)  # [d0, B, inner words] -> appended dtype
                    shaped.append(x.view((shape[0], B) + tuple(shape[1:])))
                batch[key] = _rebuild(self._rs_struct, shaped)
            # a sequence whose first state was stored as None gets zeros, as
            # concatenate_recurrent_states does; all None on one side gives None
            rows = eps.first % self._alloc_capacity
            for side, key in ((0, "recurrent_state"), (1, "next_recurrent_state")):
                if not self._rs_present_host[rows, side].any():
                    batch[key] = None
        return batch

    def _materialise_episodes(self, eps):
        """The reference's list-of-lists-of-dicts view (synchronises)."""
        order = np.argsort(-eps.length, kind="stable")
        srt = DeviceEpisodes(self, eps.first[order], eps.length[order], eps.end[order])
        b = self._gather_sequences(srt, 1.0, None, raw=True)
        if self.device.type == "cuda":
            torch.cuda.current_stream().synchronize()
        st = b["state"].data.cpu().numpy()
        ns = b["next_state"].data.cpu().numpy()
        ac = b["action"].cpu().numpy()
        rw = self._rewards_f64(srt)
        tm = b["is_state_terminal"].cpu().numpy()
        # every transition's own states, as the reference stores them
        absolute = np.concatenate([np.arange(f, f + L) for f, L in zip(srt.first, srt.length)])
        states = self._host_states(absolute)
        mus = None
        if self._mu_ring is not None:
            rows = absolute % self._alloc_capacity
            mu_rows = self._mu_ring[torch.as_tensor(rows).to(self.device)]
            present = self._mu_present_host[rows]
            mus = [self._mu_distribution(mu_rows[i]) if present[i] else None
                   for i in range(len(rows))]
        Lmax = int(srt.length[0]) if len(srt) else 0
        row0 = np.concatenate([[0], np.cumsum([(srt.length > t).sum() for t in range(Lmax)])])
        lists = [None] * len(srt)
        k = 0
        for j in range(len(srt)):
            ep = []
            for t in range(int(srt.length[j])):
                rs, nrs = states[k]
                k += 1
                r = int(row0[t]) + j
                a = ac[r]
                tr = dict(state=st[r], action=a.item() if a.shape == () else a,
                          reward=rw[j][t], next_state=ns[r], next_action=None,
                          is_state_terminal=bool(tm[r]),
                          recurrent_state=rs, next_recurrent_state=nrs)
                if mus is not None and mus[k - 1] is not None:
                    tr["mu"] = mus[k - 1]
                ep.append(tr)
            lists[order[j]] = ep
        return lists

    def _rewards_f64(self, eps):
        """The stored fp64 rewards (the packed batch carries them rounded to fp32)."""
        sr = self._rewards_f64_device(eps).cpu().numpy().tolist()
        res, k = [], 0
        for L in eps.length:
            res.append(sr[k:k + int(L)])
            k += int(L)
        return res

    def _rewards_f64_device(self, eps):
        """The stored fp64 rewards of ``eps``'s records, concatenated, on the device (the
        indices go up with a non-blocking copy from page-locked memory)."""
        from pfrl_b200.replay_buffers.device_buffer import DeviceExperiences

        self._flush()
        first, _ = self._logical(eps)
        idx = np.concatenate([np.arange(f, f + L) for f, L in zip(first, eps.length)])
        index = torch.from_numpy(idx)
        if self.device.type == "cuda":
            index = index.pin_memory()
        ex = DeviceExperiences(self, len(idx), index=index.to(self.device, non_blocking=True))
        out = self._gather(ex, 1.0, None, raw=True, want_steps=True)
        return out["step_rewards"][:, 0]

    def _host_states(self, absolute):
        """(recurrent_state, next_recurrent_state) of the records with the given absolute
        indices, as numpy in the stored structure (None where None was stored); one
        device-to-host copy."""
        if self._rs_ring is None:
            return [(None, None)] * len(absolute)
        rows = np.asarray(absolute, dtype=np.int64) % self._alloc_capacity
        flat = self._rs_ring[torch.as_tensor(rows).to(self.device)].cpu()
        # every leaf of every row, back in its appended dtype: [rows, 2, elements]
        cols = [_state_from_words(flat[:, :, off:off + d0 * inner], dt).numpy()
                for (off, d0, inner), dt in zip(self._rs_leaves, self._rs_dtypes)]
        present = self._rs_present_host[rows]
        shapes = _leaves_of_structure(self._rs_struct)
        out = []
        for i in range(len(rows)):
            pair = []
            for side in (0, 1):
                if not present[i, side]:
                    pair.append(None)
                    continue
                leaves = [c[i, side].reshape(shape) for c, shape in zip(cols, shapes)]
                pair.append(_rebuild(self._rs_struct, leaves))
            out.append(tuple(pair))
        return out

    def _all_episodes(self):
        self._flush()
        if not len(self._episodes):
            return []
        eps = DeviceEpisodes(self, [f for f, _, _ in self._episodes],
                             [L for _, L, _ in self._episodes],
                             [f + L for f, L, _ in self._episodes])
        out = []
        for lo in range(0, len(eps), _lib.SEQ_MAX_B):
            sl = slice(lo, lo + _lib.SEQ_MAX_B)
            out.extend(self._materialise_episodes(
                DeviceEpisodes(self, eps.first[sl], eps.length[sl], eps.end[sl])))
        return out


def _state_words(dtype):
    """fp32 words per element of a recurrent-state leaf of ``dtype`` in the ring: 4- and
    8-byte types are stored as their bits, fp16 widened to fp32 (exact both ways)."""
    if dtype == torch.float16:
        return 1
    size = torch.empty(0, dtype=dtype).element_size()
    if size not in (4, 8) or dtype.is_complex:
        raise TypeError("EpisodicReplayBuffer stores recurrent states of 4- or 8-byte dtypes "
                        "or float16, got %s" % dtype)
    return size // 4


def _state_to_words(x):
    if x.dtype == torch.float32:
        return x
    if x.dtype == torch.float16:
        return x.float()
    return x.contiguous().view(torch.float32)  # the bits, word by word


def _state_from_words(x, dtype):
    """``x`` [..., words] fp32 back to ``dtype`` [..., elements]."""
    if dtype == torch.float32:
        return x
    if dtype == torch.float16:
        return x.to(dtype)
    return x.contiguous().view(dtype)


def _leaves_of_structure(structure):
    if isinstance(structure, tuple) and (not structure or isinstance(structure[0], tuple)):
        out = []
        for s in structure:
            out.extend(_leaves_of_structure(s))
        return out
    return [structure]
