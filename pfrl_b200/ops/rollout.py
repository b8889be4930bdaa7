"""Packed-sequence gather out of a time-major rollout (csrc/rollout.cu).

A rollout holds its per-step data as ``[T * E, ...]`` tensors, flat slot
``t * E + e``.  A sequence is env ``e`` from step ``t0`` on for ``length`` steps;
it starts at the flat slot ``first = t0 * E + e`` and its step ``t`` is the
slot ``first + t * E``.  For sequences sorted longest first, ``gather_sequences``
returns every column's rows in ``pack_sequence`` order (time-major, row
``row_off[t] + b`` for step t of sequence b), optionally the flat slot of every
packed row, and optionally each sequence's first recurrent states laid out as
``concatenate_recurrent_states`` gives them.

``gather_sequences_torch`` is the same gather as an index tensor and
``index_select``: the formulation on CPU and with ``use_fused=False``.  The
kernel only copies, so both give the same bits.
"""
import ctypes

import numpy as np
import torch

from pfrl_b200 import _lib


def packed_layout(lens):
    """``(batch_sizes, row_off)`` of sequences of lengths ``lens`` (longest first):
    batch_sizes[t] = #{b : lens[b] > t}, row_off = [0, cumsum(batch_sizes)]."""
    lens = np.asarray(lens, dtype=np.int64)
    Lmax = int(lens[0])
    ascending = lens[::-1]
    batch_sizes = (lens.shape[0] - np.searchsorted(ascending, np.arange(Lmax), side="right"))
    batch_sizes = batch_sizes.astype(np.int64)
    row_off = np.zeros(Lmax + 1, dtype=np.int64)
    np.cumsum(batch_sizes, out=row_off[1:])
    return batch_sizes, row_off


def packed_flat_index(first, lens, E):
    """Flat slot of every packed row (numpy int64 [N])."""
    first = np.asarray(first, dtype=np.int64)
    batch_sizes, _ = packed_layout(lens)
    return np.concatenate([first[:n] + t * E for t, n in enumerate(batch_sizes.tolist())])


class StateSpec:
    """Where the leaves of a batched recurrent state sit in a flattened ring row:
    leaf i is floats ``[offset[i], offset[i] + d0[i] * inner[i])`` of the row, a
    ``[d0, inner]`` block of the ``[d0, B, inner]`` leaf."""

    def __init__(self, shapes):
        self.shapes = [(int(d0), int(inner)) for d0, inner in shapes]
        self.offsets = []
        off = 0
        for d0, inner in self.shapes:
            self.offsets.append(off)
            off += d0 * inner
        self.row_floats = off
        if not 1 <= len(self.shapes) <= _lib.SEQ_MAX_LEAVES:
            raise ValueError("a recurrent state of %d leaves (1 to %d supported)"
                             % (len(self.shapes), _lib.SEQ_MAX_LEAVES))

    def flatten(self, leaves):
        """``[d0, E, inner]`` leaves -> ``[E, row_floats]`` rows."""
        return torch.cat([leaf.detach().permute(1, 0, 2).reshape(leaf.shape[1], -1).float()
                          for leaf in leaves], dim=1)


def gather_sequences_torch(first, lens, E, columns, index=False, states=None):
    """Reference formulation.  ``columns``: ``[T * E, ...]`` tensors; ``states``:
    ``(ring [T * E, 2, D] f32, present [T * E, 2] u8, StateSpec, sides)`` with
    ``sides`` a subset of (0, 1).  Returns ``(outs, flat_index or None,
    {side: [leaf]})``."""
    dev = columns[0].device if columns else states[0].device
    idx = torch.as_tensor(packed_flat_index(first, lens, E), device=dev)
    outs = [c.index_select(0, idx) for c in columns]
    leaves = {}
    if states is not None:
        ring, present, spec, sides = states
        f = torch.as_tensor(np.asarray(first, dtype=np.int64), device=ring.device)
        rows = ring.index_select(0, f)                 # [B, 2, D]
        pres = present.index_select(0, f).bool()       # [B, 2]
        B = rows.shape[0]
        for side in sides:
            r = torch.where(pres[:, side, None], rows[:, side], torch.zeros_like(rows[:, side]))
            leaves[side] = [
                r[:, off:off + d0 * inner].reshape(B, d0, inner).permute(1, 0, 2).contiguous()
                for off, (d0, inner) in zip(spec.offsets, spec.shapes)]
    return outs, (idx if index else None), leaves


class SequenceGather:
    """``b2rl_rollout_gather_sequences`` behind torch, for one CUDA device.  The
    sequence table is built in one of two pinned host buffers and copied to a
    device buffer by the call itself; a buffer is refilled only after the event
    recorded behind its last copy has passed."""

    def __init__(self, device):
        self.device = torch.device(device)
        self._pinned = [None, None]
        self._events = [None, None]
        self._k = 0
        self._table_dev = None

    def _table(self, n):
        if self._table_dev is None or self._table_dev.numel() < n:
            cap = max(n, 1024)
            self._table_dev = torch.empty(cap, dtype=torch.int64, device=self.device)
        k = self._k
        self._k ^= 1
        if self._events[k] is not None:
            self._events[k].synchronize()
        if self._pinned[k] is None or self._pinned[k].numel() < n:
            self._pinned[k] = torch.empty(max(n, 1024), dtype=torch.int64, pin_memory=True)
        return k

    def __call__(self, first, lens, E, columns, index=False, states=None):
        """Same arguments and results as ``gather_sequences_torch``; ``columns``
        and the state ring must be contiguous CUDA tensors on this device."""
        L = _lib.load()
        first = np.asarray(first, dtype=np.int64)
        lens = np.asarray(lens, dtype=np.int64)
        B = int(first.shape[0])
        _, row_off = packed_layout(lens)
        N = int(row_off[-1])
        n = 2 * B + row_off.shape[0]
        k = self._table(n)
        host = self._pinned[k].numpy()
        host[:B] = first
        host[B:2 * B] = lens
        host[2 * B:n] = row_off
        if columns:
            T_E = columns[0].shape[0]
        else:
            T_E = states[0].shape[0]
        T = T_E // E
        cols = (_lib.RolloutCol * max(1, len(columns)))()
        outs = []
        for i, c in enumerate(columns):
            assert c.is_contiguous() and c.device == self.device and c.shape[0] == T_E
            o = torch.empty((N,) + tuple(c.shape[1:]), dtype=c.dtype, device=self.device)
            cols[i].src, cols[i].dst = c.data_ptr(), o.data_ptr()
            cols[i].row_bytes = c[0].numel() * c.element_size()
            outs.append(o)
        idx = torch.empty(N, dtype=torch.int64, device=self.device) if index else None
        rs, leaves = None, {}
        if states is not None:
            ring, present, spec, sides = states
            assert ring.is_contiguous() and present.is_contiguous() and ring.dtype == torch.float32
            rs = _lib.SeqStates()
            rs.ring, rs.present = ring.data_ptr(), present.data_ptr()
            rs.ring_rows, rs.row_floats, rs.n_leaves = ring.shape[0], spec.row_floats, len(spec.shapes)
            for side in sides:
                leaves[side] = [torch.empty((d0, B, inner), dtype=torch.float32, device=self.device)
                                for d0, inner in spec.shapes]
            for i, (off, (d0, inner)) in enumerate(zip(spec.offsets, spec.shapes)):
                rs.offset[i], rs.d0[i], rs.inner[i] = off, d0, inner
                if 0 in leaves:
                    rs.out_state[i] = leaves[0][i].data_ptr()
                if 1 in leaves:
                    rs.out_next_state[i] = leaves[1][i].data_ptr()
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream(self.device)
            _lib.check(L.b2rl_rollout_gather_sequences(
                ctypes.c_void_p(self._pinned[k].data_ptr()),
                ctypes.c_void_p(self._table_dev.data_ptr()), self._table_dev.numel(), B, T, E,
                cols, len(columns), None if idx is None else ctypes.c_void_p(idx.data_ptr()),
                None if rs is None else ctypes.byref(rs), ctypes.c_void_p(stream.cuda_stream)))
            ev = self._events[k] or torch.cuda.Event()
            ev.record(stream)
            self._events[k] = ev
        return outs, idx, leaves
