"""Helpers for recurrent models and their states (pfrl/utils/recurrent.py).

A batched recurrent state is ``None``, a tensor whose axis 1 is the batch
(``[layers, B, H]`` as ``nn.RNN`` / ``nn.GRU`` use it), or a tuple of such
states (``(h, c)`` of ``nn.LSTM``, one entry per child of a
``RecurrentSequential``).  Sequences are handed to recurrent modules as
``PackedSequence``s sorted by length, longest first; their ``data`` rows are
time-major, the order ``flatten_sequences_time_first`` produces.
"""
import itertools

import numpy as np
import torch
from torch import nn
from torch.nn.utils.rnn import PackedSequence


def is_recurrent(layer):
    """True for the recurrent layers the containers and agents understand."""
    from pfrl_b200.nn.recurrent import Recurrent  # the nn package imports this module

    return isinstance(layer, (nn.LSTM, nn.RNN, nn.GRU, Recurrent))


def _map_state(fn, recurrent_state):
    if recurrent_state is None:
        return None
    if isinstance(recurrent_state, torch.Tensor):
        return fn(recurrent_state)
    if isinstance(recurrent_state, tuple):
        return tuple(_map_state(fn, s) for s in recurrent_state)
    raise ValueError("Invalid recurrent state: {}".format(recurrent_state))


def mask_recurrent_state_at(recurrent_state, indices):
    """A copy of the state with the batch entries ``indices`` set to zero."""

    def mask(s):
        m = torch.ones_like(s)
        m[:, indices] = 0
        return s * m

    return _map_state(mask, recurrent_state)


def get_recurrent_state_at(recurrent_state, indices, detach):
    """The batch entries ``indices`` of a state (axis 1), optionally detached."""

    def pick(s):
        return (s.detach() if detach else s)[:, indices]

    return _map_state(pick, recurrent_state)


def concatenate_recurrent_states(split_recurrent_states):
    """Stack per-sample states (as ``get_recurrent_state_at(..., i)`` returns
    them) into one batched state along a new axis 1.  ``None`` entries become
    zeros shaped like the first non-``None`` one; all ``None`` gives ``None``."""
    like = next((s for s in split_recurrent_states if s is not None), None)
    if like is None:
        return None
    if isinstance(like, torch.Tensor):
        return torch.stack([torch.zeros_like(like) if s is None else s
                            for s in split_recurrent_states], dim=1)
    if isinstance(like, np.ndarray):
        return np.stack([np.zeros_like(like) if s is None else s
                         for s in split_recurrent_states], axis=1)
    if isinstance(like, tuple):
        return tuple(
            concatenate_recurrent_states([None if s is None else s[i]
                                          for s in split_recurrent_states])
            for i in range(len(like)))
    raise ValueError("Invalid recurrent state: {}".format(like))


def _pack_one_step(xs):
    """A [B, ...] batch as B sequences of length 1: the packed data is the batch
    itself, so no copy is made."""
    if isinstance(xs, tuple):
        return tuple(_pack_one_step(x) for x in xs)
    assert isinstance(xs, torch.Tensor)
    return PackedSequence(xs, torch.tensor([xs.shape[0]], dtype=torch.int64))


def one_step_forward(rnn, batch_input, recurrent_state):
    """Advance ``rnn`` by one step on a [B, ...] batch (or tuple of batches).
    Returns the [B, ...] output and the new batched state."""
    y, recurrent_state = rnn(_pack_one_step(batch_input), recurrent_state)
    return unwrap_packed_sequences_recursive(y), recurrent_state


def pack_and_forward(rnn, sequences, recurrent_state):
    """Multi-step forward over sequences.  ``sequences`` is a list of
    per-sequence tensors (or tuples of them) sorted by length, longest first,
    or sequences that are already packed (a ``PackedSequence`` or a tuple of
    them, as the device episodic replay buffer gathers them).  Returns the
    output rows in time-major packed order and the new batched state."""
    y, recurrent_state = rnn(pack_sequences_recursive(sequences), recurrent_state)
    return unwrap_packed_sequences_recursive(y), recurrent_state


def flatten_sequences_time_first(sequences):
    """Concatenate the items of the sequences time step by time step: the row
    order of ``pack_sequence`` for sequences sorted longest first."""
    out = []
    for step in itertools.zip_longest(*sequences):
        out.extend(x for x in step if x is not None)
    return out


def wrap_packed_sequences_recursive(unwrapped, batch_sizes, sorted_indices):
    """Packed data tensor(s) -> ``PackedSequence``(s) with the given layout."""
    if isinstance(unwrapped, torch.Tensor):
        return PackedSequence(unwrapped, batch_sizes=batch_sizes, sorted_indices=sorted_indices)
    if isinstance(unwrapped, tuple):
        return tuple(wrap_packed_sequences_recursive(x, batch_sizes, sorted_indices)
                     for x in unwrapped)
    return unwrapped


def unwrap_packed_sequences_recursive(packed):
    """``PackedSequence``(s) -> their data tensor(s), without padding."""
    if isinstance(packed, PackedSequence):
        return packed.data
    if isinstance(packed, tuple):
        return tuple(unwrap_packed_sequences_recursive(x) for x in packed)
    return packed


def pack_sequences_recursive(sequences):
    """``pack_sequence`` that descends into tuples: a list of N-tuples of
    tensors gives an N-tuple of ``PackedSequence``.  Already packed input is
    returned as it is."""
    if isinstance(sequences, PackedSequence):
        return sequences
    if isinstance(sequences, tuple) and sequences and all(
            isinstance(s, PackedSequence) for s in sequences):
        return sequences
    assert sequences
    first = sequences[0]
    if isinstance(first, torch.Tensor):
        return nn.utils.rnn.pack_sequence(sequences)
    if isinstance(first, tuple):
        return tuple(pack_sequences_recursive([seq[i] for seq in sequences])
                     for i in range(len(first)))
    return sequences


def get_packed_sequence_info(packed):
    """``(batch_sizes, sorted_indices)`` of the first ``PackedSequence`` found
    in ``packed``, or ``None``."""
    if isinstance(packed, PackedSequence):
        return packed.batch_sizes, packed.sorted_indices
    if isinstance(packed, tuple):
        for x in packed:
            info = get_packed_sequence_info(x)
            if info is not None:
                return info
    return None


def recurrent_state_as_numpy(recurrent_state):
    """Tensors of a state -> numpy arrays (a device-to-host copy)."""
    return _map_state(lambda s: s.detach().cpu().numpy(), recurrent_state)


def recurrent_state_from_numpy(recurrent_state, device):
    """Numpy arrays of a state -> tensors on ``device``."""
    if recurrent_state is None:
        return None
    if isinstance(recurrent_state, np.ndarray):
        return torch.from_numpy(recurrent_state).to(device)
    if isinstance(recurrent_state, tuple):
        return tuple(recurrent_state_from_numpy(s, device) for s in recurrent_state)
    raise ValueError("Invalid recurrent state: {}".format(recurrent_state))


def detach_recurrent_state(recurrent_state):
    """The state with every tensor detached from the graph."""
    return _map_state(lambda s: s.detach(), recurrent_state)
