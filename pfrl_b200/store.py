"""Thin Python owner of a ``b2rl_replay`` handle (include/b2rl.h).

torch is used only for device memory (output tensors) and the current CUDA
stream; every operation is a C-ABI call into libb2rl.so.
"""
import ctypes

import numpy as np
import torch

from . import _lib
from ._lib import (  # noqa: F401
    NORM_BATCH, NORM_MEMORY, NORM_NONE, OBS_RAW, OBS_U8_TO_F32, SAMPLE_EXACT,
    SAMPLE_PARALLEL,
)


def _np_ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _stream(device=None):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


_ITEMSIZE = {}


def _itemsize(dtype):
    sz = _ITEMSIZE.get(dtype)
    if sz is None:
        sz = _ITEMSIZE[dtype] = torch.empty((), dtype=dtype).element_size()
    return sz


class DeviceReplayStore:
    """HBM part ring + experience records (+ fp64 sum/min trees)."""

    def __init__(self, capacity, part_bytes, stack=1, n_step=1, action_bytes=8,
                 prioritized=True, part_capacity=None, device=0, max_batch=4096):
        self.L = _lib.load()
        if part_capacity is None:
            part_capacity = 2 * capacity + 64
        self.cfg = _lib.ReplayConfig(
            capacity=capacity, part_capacity=part_capacity, part_bytes=part_bytes,
            stack=stack, n_step=n_step, action_bytes=action_bytes,
            prioritized=int(bool(prioritized)), device=device, max_batch=max_batch,
        )
        self.device = torch.device("cuda", device)
        h = ctypes.c_void_p()
        _lib.check(self.L.b2rl_replay_create(ctypes.byref(self.cfg), ctypes.byref(h)))
        self.h = h
        self.capacity = capacity
        self.part_bytes = part_bytes
        self.stack = stack
        self.n_step = n_step
        self.action_bytes = action_bytes
        self.prioritized = bool(prioritized)
        self.part_capacity = part_capacity
        self.max_batch = max_batch

    def close(self):
        if getattr(self, "h", None):
            self.L.b2rl_replay_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __len__(self):
        return int(self.L.b2rl_replay_len(self.h))

    @property
    def napp(self):
        return int(self.L.b2rl_replay_napp(self.h))

    @property
    def npop(self):
        return int(self.L.b2rl_replay_npop(self.h))

    @property
    def device_bytes(self):
        return int(self.L.b2rl_replay_device_bytes(self.h))

    # -- parts -------------------------------------------------------------
    def put_parts(self, parts):
        """Copy parts (numpy [n, part_bytes] uint8-viewable, or a CUDA tensor)
        into the ring; returns their slots as int32 numpy."""
        if isinstance(parts, torch.Tensor):
            assert parts.is_cuda and parts.is_contiguous()
            n = parts.numel() * parts.element_size() // self.part_bytes
            slots = np.empty(n, dtype=np.int32)
            _lib.check(self.L.b2rl_replay_put_parts(
                self.h, ctypes.c_void_p(parts.data_ptr()), 1, n, _np_ptr(slots), _stream(self.device)))
            return slots
        a = np.ascontiguousarray(parts)
        n = a.nbytes // self.part_bytes
        assert n * self.part_bytes == a.nbytes
        slots = np.empty(n, dtype=np.int32)
        _lib.check(self.L.b2rl_replay_put_parts(self.h, _np_ptr(a), 0, n, _np_ptr(slots), _stream(self.device)))
        return slots

    # -- append ------------------------------------------------------------
    def append(self, state_parts, next_parts, action, rewards, length, terminal,
               priority=None):
        sp = np.ascontiguousarray(state_parts, dtype=np.int32).reshape(-1, self.stack)
        n = sp.shape[0]
        nx = np.ascontiguousarray(next_parts, dtype=np.int32).reshape(n, self.stack)
        act = np.ascontiguousarray(action)
        assert act.nbytes == n * self.action_bytes, (act.nbytes, n, self.action_bytes)
        rw = np.ascontiguousarray(rewards, dtype=np.float64).reshape(n, self.n_step)
        ln = np.ascontiguousarray(length, dtype=np.uint8).reshape(n)
        tm = np.ascontiguousarray(terminal, dtype=np.uint8).reshape(n)
        pr = None
        if priority is not None:
            pr = np.ascontiguousarray(priority, dtype=np.float64).reshape(n)
        e = _lib.Experiences(
            state_parts=sp.ctypes.data, next_parts=nx.ctypes.data, action=act.ctypes.data,
            rewards=rw.ctypes.data, len=ln.ctypes.data, terminal=tm.ctypes.data,
            priority=None if pr is None else pr.ctypes.data,
        )
        _lib.check(self.L.b2rl_replay_append(self.h, ctypes.byref(e), n, 0, _stream(self.device)))

    # -- prioritized sampling ------------------------------------------------
    def sample(self, u, mode=SAMPLE_EXACT, want_index=True, want_priority=True):
        u = np.ascontiguousarray(u, dtype=np.float64)
        n = u.shape[0]
        idx = torch.empty(n, dtype=torch.int64, device=self.device) if want_index else None
        pri = torch.empty(n, dtype=torch.float64, device=self.device) if want_priority else None
        _lib.check(self.L.b2rl_per_sample(
            self.h, _np_ptr(u), n, mode,
            ctypes.c_void_p(idx.data_ptr()) if want_index else None,
            ctypes.c_void_p(pri.data_ptr()) if want_priority else None, _stream(self.device)))
        return idx, pri

    def weights(self, n, beta, norm, want_prob=False):
        w = torch.empty(n, dtype=torch.float32, device=self.device)
        p = torch.empty(n, dtype=torch.float64, device=self.device) if want_prob else None
        _lib.check(self.L.b2rl_per_weights(
            self.h, float(beta), int(norm), ctypes.c_void_p(w.data_ptr()),
            ctypes.c_void_p(p.data_ptr()) if want_prob else None, _stream(self.device)))
        return (w, p) if want_prob else w

    def update_priorities(self, priority):
        if isinstance(priority, torch.Tensor):
            assert priority.is_cuda and priority.dtype == torch.float64 and priority.is_contiguous()
            _lib.check(self.L.b2rl_per_update_priorities(
                self.h, ctypes.c_void_p(priority.data_ptr()), 1, priority.numel(), _stream(self.device)))
        else:
            p = np.ascontiguousarray(priority, dtype=np.float64)
            _lib.check(self.L.b2rl_per_update_priorities(self.h, _np_ptr(p), 0, p.shape[0], _stream(self.device)))

    def update_errors(self, errors, alpha, eps, error_min, error_max):
        assert isinstance(errors, torch.Tensor) and errors.is_cuda and errors.is_contiguous()
        assert errors.dtype in (torch.float32, torch.float64)
        if error_min is None and error_max is None:
            error_min, error_max = 1.0, 0.0  # min > max disables clipping
        elif error_min is None:
            error_min = -float("inf")
        elif error_max is None:
            error_max = float("inf")
        _lib.check(self.L.b2rl_per_update_errors(
            self.h, ctypes.c_void_p(errors.data_ptr()), int(errors.dtype == torch.float64),
            errors.numel(), float(alpha), float(eps), float(error_min), float(error_max),
            _stream(self.device)))

    def defer_errors(self, errors, alpha, eps, error_min, error_max):
        """Answer the last sample without a launch: the write-back runs at the
        head of the next fused step (or before the next tree access).  The
        tensor is kept alive until then."""
        assert isinstance(errors, torch.Tensor) and errors.is_cuda and errors.is_contiguous()
        assert errors.dtype in (torch.float32, torch.float64)
        if error_min is None and error_max is None:
            error_min, error_max = 1.0, 0.0  # min > max disables clipping
        elif error_min is None:
            error_min = -float("inf")
        elif error_max is None:
            error_max = float("inf")
        _lib.check(self.L.b2rl_per_defer_errors(
            self.h, ctypes.c_void_p(errors.data_ptr()), int(errors.dtype == torch.float64),
            errors.numel(), float(alpha), float(eps), float(error_min), float(error_max)))
        self._deferred_errors = errors

    def update_host_errors(self, errors, alpha, eps, error_min, error_max, defer):
        """TD errors as host floats -> priorities with the reference's Python-float arithmetic
        (libm pow, computed inside the library) -> write-back now, or folded into the next
        fused step (defer)."""
        e = np.ascontiguousarray(errors, dtype=np.float64)
        _lib.check(self.L.b2rl_per_update_host_errors(
            self.h, _np_ptr(e), e.shape[0], float(alpha), float(eps),
            int(error_min is not None), 0.0 if error_min is None else float(error_min),
            int(error_max is not None), 0.0 if error_max is None else float(error_max),
            int(bool(defer)), _stream(self.device)))
        if defer:
            self._deferred_errors = None

    def flush(self):
        _lib.check(self.L.b2rl_per_flush(self.h, _stream(self.device)))
        self._deferred_errors = None

    def step(self, u, gamma_pow, beta, norm, mode=SAMPLE_EXACT, obs_mode=OBS_RAW,
             obs_scale=1.0, obs_dtype=None, obs_shape=None, action_dtype=torch.int64,
             action_shape=(), want_obs=True, want_index=True, want_priority=False,
             want_prob=False, out=None):
        """Fused replay step (b2rl_replay_step): [deferred write-back] -> sample ->
        importance weights -> gather, one launch.  u: numpy float64 [n] (host) or a
        CUDA float64 tensor.  Returns (batch dict, index, weights[, priority, prob]).
        `out`: dict of preallocated output tensors from an earlier call (reused)."""
        n = int(u.shape[0])
        dev = self.device
        gp = np.ascontiguousarray(gamma_pow, dtype=np.float64)
        assert gp.shape[0] == self.n_step + 1
        obs_bytes = self.stack * self.part_bytes
        if out is None:
            out = {}
            if want_obs:
                if obs_mode == OBS_U8_TO_F32:
                    odt, oshape = torch.float32, (n, obs_bytes)
                else:
                    odt = obs_dtype or torch.uint8
                    oshape = (n, obs_bytes // _itemsize(odt))
                out["state"] = torch.empty(oshape, dtype=odt, device=dev)
                out["next_state"] = torch.empty(oshape, dtype=odt, device=dev)
            # the call sits on the host's critical path between two launches and every torch op
            # costs 3-5 us there: the four f32 vectors come out of one [4, n] allocation with
            # one unbind (slice + view chains measured slower than separate torch.empty calls)
            (out["reward"], out["is_state_terminal"], out["discount"],
             out["weights"]) = torch.empty((4, n), dtype=torch.float32, device=dev).unbind(0)
            asz = _itemsize(action_dtype)
            out["action"] = torch.empty((n, self.action_bytes // asz), dtype=action_dtype, device=dev)
            if want_index:
                out["index"] = torch.empty(n, dtype=torch.int64, device=dev)
            if want_priority:
                out["priority"] = torch.empty(n, dtype=torch.float64, device=dev)
            if want_prob:
                out["prob"] = torch.empty(n, dtype=torch.float64, device=dev)
        ptr = lambda k: out[k].data_ptr() if k in out else None  # noqa: E731
        if isinstance(u, torch.Tensor):
            assert u.is_cuda and u.dtype == torch.float64 and u.is_contiguous()
            u_ptr, u_dev, keep = u.data_ptr(), 1, u
        else:
            keep = np.ascontiguousarray(u, dtype=np.float64)
            u_ptr, u_dev = keep.ctypes.data, 0
        a = _lib.StepArgs(
            n=n, mode=int(mode), u=u_ptr, u_on_device=u_dev, norm=int(norm), beta=float(beta),
            gamma_pow_host=gp.ctypes.data, obs_mode=int(obs_mode), obs_scale=float(obs_scale),
            index_dev=ptr("index"), priority_dev=ptr("priority"), weight_dev=ptr("weights"),
            prob_dev=ptr("prob"),
            out=_lib.BatchOut(
                state=ptr("state"), next_state=ptr("next_state"), action=ptr("action"),
                reward=ptr("reward"), terminal=ptr("is_state_terminal"),
                discount=ptr("discount"), step_rewards=None, len=None))
        _lib.check(self.L.b2rl_replay_step(self.h, ctypes.byref(a), _stream(self.device)))
        self._deferred_errors = None  # consumed by the launch (stream-ordered)
        res = dict(out)
        if want_obs and obs_shape is not None:
            res["state"] = res["state"].view((n,) + tuple(obs_shape))
            res["next_state"] = res["next_state"].view((n,) + tuple(obs_shape))
        res["action"] = res["action"].view((n,) + tuple(action_shape))
        return res

    def gather_sequences(self, first, length, end, obs_mode=OBS_RAW, obs_scale=1.0,
                         action_dtype=torch.int64, states=None):
        """Packed minibatch of B sequences (b2rl_replay_gather_sequences).
        first / length / end: host int arrays, lengths sorted longest first.
        states: None or (ring, present, leaves) with leaves a list of
        (offset, d0, inner) -- the state outputs are then [d0, B, inner] f32.
        Returns a dict of flat packed tensors (rows in pack_sequence order),
        plus "state_leaves" / "next_state_leaves" lists when states are given."""
        first = np.ascontiguousarray(first, dtype=np.int64)
        length = np.ascontiguousarray(length, dtype=np.int32)
        end = np.ascontiguousarray(end, dtype=np.int64)
        B = int(first.shape[0])
        N = int(length.sum())
        dev = self.device
        obs_bytes = self.stack * self.part_bytes
        odt = torch.float32 if obs_mode == OBS_U8_TO_F32 else torch.uint8
        out = {
            "state": torch.empty((N, obs_bytes), dtype=odt, device=dev),
            "next_state": torch.empty((N, obs_bytes), dtype=odt, device=dev),
            "action": torch.empty((N, self.action_bytes // _itemsize(action_dtype)),
                                  dtype=action_dtype, device=dev),
        }
        out["reward"], out["is_state_terminal"] = torch.empty(
            (2, N), dtype=torch.float32, device=dev).unbind(0)
        so = _lib.SeqOut(state=out["state"].data_ptr(), next_state=out["next_state"].data_ptr(),
                         action=out["action"].data_ptr(), reward=out["reward"].data_ptr(),
                         terminal=out["is_state_terminal"].data_ptr())
        ss = None
        if states is not None:
            ring, present, leaves = states
            assert len(leaves) <= _lib.SEQ_MAX_LEAVES, "at most %d state tensors" % (
                _lib.SEQ_MAX_LEAVES)
            ss = _lib.SeqStates(ring=ring.data_ptr(), present=present.data_ptr(),
                                ring_rows=ring.shape[0], row_floats=ring.shape[2],
                                n_leaves=len(leaves))
            out["state_leaves"], out["next_state_leaves"] = [], []
            for i, (off, d0, inner) in enumerate(leaves):
                s = torch.empty((d0, B, inner), dtype=torch.float32, device=dev)
                n = torch.empty((d0, B, inner), dtype=torch.float32, device=dev)
                ss.offset[i], ss.d0[i], ss.inner[i] = off, d0, inner
                ss.out_state[i], ss.out_next_state[i] = s.data_ptr(), n.data_ptr()
                out["state_leaves"].append(s)
                out["next_state_leaves"].append(n)
        _lib.check(self.L.b2rl_replay_gather_sequences(
            self.h, _np_ptr(first), _np_ptr(length), _np_ptr(end), B, int(obs_mode),
            float(obs_scale), ctypes.byref(so), ctypes.byref(ss) if ss is not None else None,
            _stream(self.device)))
        return out

    def info(self):
        out = _lib.PerInfo()
        _lib.check(self.L.b2rl_per_get_info(self.h, ctypes.byref(out), _stream(self.device)))
        return dict(total=out.total, min=out.min, max_priority=out.max_priority,
                    napp=out.napp, npop=out.npop, scout_hits=out.scout_hits)

    def set_max_priority(self, value):
        _lib.check(self.L.b2rl_per_set_max_priority(self.h, float(value), _stream(self.device)))

    def read_priorities(self, first=0, n=None):
        if n is None:
            n = len(self) - first
        out = np.empty(n, dtype=np.float64)
        _lib.check(self.L.b2rl_per_read_priorities(self.h, first, n, _np_ptr(out), _stream(self.device)))
        return out

    # -- gather --------------------------------------------------------------
    def gather(self, n, gamma_pow, index=None, obs_mode=OBS_RAW, obs_scale=1.0,
               obs_dtype=None, obs_shape=None, action_dtype=torch.int64,
               action_shape=(), want_obs=True, want_steps=False):
        """Assemble a minibatch.  index: CUDA int64 tensor of logical indices,
        or None for the experiences of the pending prioritized sample."""
        gp = np.ascontiguousarray(gamma_pow, dtype=np.float64)
        assert gp.shape[0] == self.n_step + 1
        obs_bytes = self.stack * self.part_bytes
        dev = self.device
        if obs_mode == OBS_U8_TO_F32:
            odt, oshape = torch.float32, (n, obs_bytes)
        else:
            odt = obs_dtype or torch.uint8
            oshape = (n, obs_bytes // _itemsize(odt))
        out = {}
        if want_obs:
            out["state"] = torch.empty(oshape, dtype=odt, device=dev)
            out["next_state"] = torch.empty(oshape, dtype=odt, device=dev)
        asz = torch.empty((), dtype=action_dtype).element_size()
        out["action"] = torch.empty((n, self.action_bytes // asz), dtype=action_dtype, device=dev)
        out["reward"] = torch.empty(n, dtype=torch.float32, device=dev)
        out["is_state_terminal"] = torch.empty(n, dtype=torch.float32, device=dev)
        out["discount"] = torch.empty(n, dtype=torch.float32, device=dev)
        if want_steps:
            out["step_rewards"] = torch.empty((n, self.n_step), dtype=torch.float64, device=dev)
            out["len"] = torch.empty(n, dtype=torch.uint8, device=dev)
        bo = _lib.BatchOut(
            state=out["state"].data_ptr() if want_obs else None,
            next_state=out["next_state"].data_ptr() if want_obs else None,
            action=out["action"].data_ptr(), reward=out["reward"].data_ptr(),
            terminal=out["is_state_terminal"].data_ptr(), discount=out["discount"].data_ptr(),
            step_rewards=out["step_rewards"].data_ptr() if want_steps else None,
            len=out["len"].data_ptr() if want_steps else None,
        )
        _lib.check(self.L.b2rl_replay_gather(
            self.h, ctypes.c_void_p(index.data_ptr()) if index is not None else None, n,
            _np_ptr(gp), int(obs_mode), float(obs_scale), ctypes.byref(bo), _stream(self.device)))
        if want_obs and obs_shape is not None:
            out["state"] = out["state"].view((n,) + tuple(obs_shape))
            out["next_state"] = out["next_state"].view((n,) + tuple(obs_shape))
        out["action"] = out["action"].view((n,) + tuple(action_shape))
        return out
