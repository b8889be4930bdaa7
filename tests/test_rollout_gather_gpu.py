"""k_rollout_seq_gather (b2rl_rollout_gather_sequences) against its torch formulation.

The kernel packs sequences (env, t0, length) out of a time-major rollout [T * E, ...]
into pack_sequence order, together with the flat slot of every packed row and the
first slots' recurrent states.  It only copies, so every output must be bit-equal to
ops.rollout.gather_sequences_torch (index tensor + index_select) on the same device.
"""
import ctypes

import numpy as np
import pytest
import torch

from pfrl_b200 import _lib
from pfrl_b200.ops import rollout

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _bits(t):
    return t.detach().contiguous().reshape(-1).view(torch.uint8)


def _spans(rng, T, E, kind):
    """Sequences sorted stably, longest first: (first slots, lengths)."""
    if kind == "ones":        # every step its own sequence: B = T * E
        seqs = [(e, t, 1) for t in range(T) for e in range(E)]
    elif kind == "whole":     # one sequence of length T per env (equal lengths)
        seqs = [(e, 0, T) for e in range(E)]
    else:                     # random episode boundaries, random subset, shuffled
        seqs = []
        for e in range(E):
            t = 0
            while t < T:
                n = int(rng.randint(1, T - t + 1)) if rng.rand() < 0.5 else int(
                    min(T - t, rng.choice([1, 2, 3])))
                seqs.append((e, t, n))
                t += n
        rng.shuffle(seqs)
        keep = max(1, int(len(seqs) * rng.uniform(0.3, 1.0)))
        seqs = seqs[:keep]
    seqs = sorted(seqs, key=lambda s: s[2], reverse=True)
    first = np.array([t * E + e for e, t, _ in seqs], dtype=np.int64)
    lens = np.array([n for _, _, n in seqs], dtype=np.int64)
    return first, lens


def _states(rng, T, E, shapes, mode):
    spec = rollout.StateSpec(shapes)
    ring = torch.randn(T * E, 2, spec.row_floats, device=DEV)
    if mode == "present":
        present = torch.ones(T * E, 2, dtype=torch.uint8, device=DEV)
    else:  # mixed: some first states are None (zeros)
        present = torch.as_tensor(rng.randint(0, 2, (T * E, 2)).astype(np.uint8), device=DEV)
    return ring, present, spec


def _compare(first, lens, E, columns, index, states):
    g = rollout.SequenceGather(DEV)
    k_outs, k_idx, k_leaves = g(first, lens, E, columns, index, states)
    t_outs, t_idx, t_leaves = rollout.gather_sequences_torch(first, lens, E, columns, index,
                                                            states)
    torch.cuda.synchronize()
    assert len(k_outs) == len(t_outs)
    for k, t in zip(k_outs, t_outs):
        assert k.dtype == t.dtype and k.shape == t.shape
        assert torch.equal(_bits(k), _bits(t))
    if index:
        assert torch.equal(k_idx, t_idx)
        assert int(k_idx.numel()) == int(lens.sum())
    else:
        assert k_idx is None
    assert sorted(k_leaves) == sorted(t_leaves)
    for side in t_leaves:
        for k, t in zip(k_leaves[side], t_leaves[side]):
            assert k.shape == t.shape
            assert torch.equal(_bits(k), _bits(t))


@pytest.mark.parametrize("T", [1, 7, 128, 129])
@pytest.mark.parametrize("E", [1, 3, 8, 256])
@pytest.mark.parametrize("kind", ["random", "ones", "whole"])
def test_shapes_and_sequence_tables(T, E, kind):
    rng = np.random.RandomState(T * 1000 + E)
    first, lens = _spans(rng, T, E, kind)
    N = T * E
    obs = torch.randn(N, 5, device=DEV)                      # 20 B rows
    act = torch.randint(0, 7, (N,), device=DEV)              # int64 scalar
    adv = torch.randn(N, device=DEV)                         # 4 B rows
    ring, present, spec = _states(rng, T, E, [(1, 3), (1, 3)], "mixed")
    _compare(first, lens, E, [obs, act, adv], True, (ring, present, spec, (0, 1)))


@pytest.mark.parametrize("row", ["f32x1", "f32x3", "f32x376", "u8_84x84x4", "u8_13",
                                 "f32x17_action", "i64"])
@pytest.mark.parametrize("T,E", [(7, 3), (128, 8)])
def test_row_sizes_and_dtypes(row, T, E):
    rng = np.random.RandomState(7)
    N = T * E
    col = {
        "f32x1": lambda: torch.randn(N, device=DEV),                           # 4 B
        "f32x3": lambda: torch.randn(N, 3, device=DEV),                        # 12 B
        "f32x376": lambda: torch.randn(N, 376, device=DEV),                    # 1 504 B
        "u8_84x84x4": lambda: torch.randint(0, 256, (N, 4, 84, 84), dtype=torch.uint8,
                                            device=DEV),                       # 28 224 B
        "u8_13": lambda: torch.randint(0, 256, (N, 13), dtype=torch.uint8, device=DEV),
        "f32x17_action": lambda: torch.randn(N, 17, device=DEV),               # 68 B
        "i64": lambda: torch.randint(-5, 5, (N,), device=DEV),
    }[row]()
    for kind in ("random", "ones", "whole"):
        first, lens = _spans(rng, T, E, kind)
        _compare(first, lens, E, [col], False, None)


def test_unaligned_column_views():
    """Rows that are 16-byte multiples but start off a 16-byte boundary take the
    narrower copy path and still land where they belong."""
    T, E = 9, 4
    rng = np.random.RandomState(3)
    base = torch.randint(0, 256, (T * E * 32 + 3,), dtype=torch.uint8, device=DEV)
    col = base[3:].view(T * E, 32)  # 32 B rows at an odd address
    first, lens = _spans(rng, T, E, "random")
    _compare(first, lens, E, [col.contiguous(), col], False, None)


@pytest.mark.parametrize("shapes", [[(1, 8)], [(1, 4), (1, 4)], [(2, 16)],
                                    [(1, 5), (1, 5), (2, 3), (2, 3)]],
                         ids=["1leaf", "2leaves", "2layer", "4leaves"])
@pytest.mark.parametrize("mode", ["present", "mixed"])
@pytest.mark.parametrize("sides", [(0,), (1,), (0, 1)])
def test_recurrent_states(shapes, mode, sides):
    T, E = 33, 5
    rng = np.random.RandomState(11)
    ring, present, spec = _states(rng, T, E, shapes, mode)
    for kind in ("random", "ones", "whole"):
        first, lens = _spans(rng, T, E, kind)
        _compare(first, lens, E, [], True, (ring, present, spec, sides))
        _compare(first, lens, E, [torch.randn(T * E, 2, device=DEV)], False,
                 (ring, present, spec, sides))


def test_state_rows_wider_than_the_leaves_and_absent_states():
    """Floats of the ring row outside every leaf are never read into an output;
    an absent side is all zeros."""
    T, E = 4, 2
    ring = torch.randn(T * E, 2, 10, device=DEV)
    present = torch.zeros(T * E, 2, dtype=torch.uint8, device=DEV)
    present[:, 1] = 1
    spec = rollout.StateSpec([(1, 4)])
    spec.row_floats = 10
    first, lens = _spans(np.random.RandomState(0), T, E, "random")
    g = rollout.SequenceGather(DEV)
    _, _, leaves = g(first, lens, E, [], False, (ring, present, spec, (0, 1)))
    assert torch.count_nonzero(leaves[0][0]) == 0
    f = torch.as_tensor(first, device=DEV)
    assert torch.equal(leaves[1][0][0], ring[f, 1, :4])


def test_repeated_calls_reuse_the_pinned_tables():
    """Alternating pinned tables: many back-to-back calls without a synchronisation
    each pack their own sequences."""
    T, E = 16, 4
    col = torch.randn(T * E, 6, device=DEV)
    g = rollout.SequenceGather(DEV)
    rng = np.random.RandomState(5)
    got, want = [], []
    for _ in range(20):
        first, lens = _spans(rng, T, E, "random")
        got.append(g(first, lens, E, [col], True)[0][0])
        want.append(col[torch.as_tensor(rollout.packed_flat_index(first, lens, E), device=DEV)])
    torch.cuda.synchronize()
    for a, b in zip(got, want):
        assert torch.equal(_bits(a), _bits(b))


def _raw_call(table, B, T, E, capacity=None, col=None, dst=None):
    L = _lib.load()
    table = np.ascontiguousarray(table, dtype=np.int64)
    dev_tab = torch.empty(max(capacity or table.size, 1), dtype=torch.int64, device=DEV)
    cols = (_lib.RolloutCol * 1)()
    n_cols = 0
    if col is not None:
        cols[0].src, cols[0].dst, cols[0].row_bytes = col.data_ptr(), dst.data_ptr(), 4
        n_cols = 1
    status = L.b2rl_rollout_gather_sequences(
        table.ctypes.data_as(ctypes.c_void_p), ctypes.c_void_p(dev_tab.data_ptr()),
        dev_tab.numel() if capacity is None else capacity, B, T, E, cols, n_cols,
        None, None, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return status


def _table(first, lens):
    _, row_off = rollout.packed_layout(lens)
    return np.concatenate([first, lens, row_off])


def test_invalid_tables_raise():
    T, E = 5, 3
    col = torch.randn(T * E, device=DEV)
    dst = torch.empty(T * E, device=DEV)
    ok = _table(np.array([0, 1], np.int64), np.array([3, 2], np.int64))
    assert _raw_call(ok, 2, T, E, col=col, dst=dst) == 0
    bad = {
        "length 0": (np.array([0, 1]), np.array([2, 0])),
        "lengths increasing": (np.array([0, 1]), np.array([2, 3])),
        "past the last step": (np.array([2 * E, 1]), np.array([4, 2])),
        "negative first": (np.array([-1, 1]), np.array([2, 2])),
        "env past E at the last step": (np.array([T * E, 0]), np.array([1, 1])),
    }
    for name, (first, lens) in bad.items():
        lens = np.asarray(lens, np.int64)
        row_off = np.zeros(max(int(lens.max()), 1) + 1, np.int64)
        tab = np.concatenate([np.asarray(first, np.int64), lens, row_off])
        with pytest.raises(_lib.B2rlError):
            _lib.check(_raw_call(tab, 2, T, E, col=col, dst=dst))
    wrong_off = ok.copy()
    wrong_off[-1] += 1
    with pytest.raises(_lib.B2rlError):
        _lib.check(_raw_call(wrong_off, 2, T, E, col=col, dst=dst))
    nonzero_start = ok.copy()
    nonzero_start[4] = 1
    with pytest.raises(_lib.B2rlError):
        _lib.check(_raw_call(nonzero_start, 2, T, E, col=col, dst=dst))
    with pytest.raises(_lib.B2rlError):
        _lib.check(_raw_call(ok, 2, T, E, capacity=ok.size - 1, col=col, dst=dst))
    with pytest.raises(_lib.B2rlError):
        _lib.check(_raw_call(ok, 0, T, E, col=col, dst=dst))
    with pytest.raises(_lib.B2rlError):
        _lib.check(_raw_call(ok, 2, T, 0, col=col, dst=dst))
    # the sequence gather raises the same way
    g = rollout.SequenceGather(DEV)
    with pytest.raises(_lib.B2rlError):
        g(np.array([0, 1]), np.array([2, 3]), E, [col])
