"""Recurrent module interface and its two containers (pfrl/nn/recurrent.py,
recurrent_sequential.py, recurrent_branched.py).

A recurrent module is called as ``module(packed_input, recurrent_state)`` and
returns ``(packed_output, new_recurrent_state)``, like ``torch.nn.LSTM`` with
the sequences packed in a ``torch.nn.utils.rnn.PackedSequence``.  A state of
``None`` means "start from zeros".
"""
from torch import nn

from pfrl_b200.utils.recurrent import (
    get_packed_sequence_info,
    is_recurrent,
    unwrap_packed_sequences_recursive,
    wrap_packed_sequences_recursive,
)


class Recurrent(object):
    """Marker base class: ``forward(packed_input, recurrent_state)`` returns the
    packed output sequences and the new batched state."""

    def forward(self, packed_input, recurrent_state):
        raise NotImplementedError


class RecurrentSequential(Recurrent, nn.Sequential):
    """``nn.Sequential`` that threads one state per recurrent child.

    The recurrent state is a tuple with one entry per recurrent child, in
    order.  Stateless layers see the packed data tensor (time-major rows of
    all sequences), so they run as one batched call; recurrent layers see the
    ``PackedSequence``.
    """

    def forward(self, sequences, recurrent_state):
        children = self.recurrent_children
        if recurrent_state is None:
            states = [None] * len(children)
        else:
            assert len(recurrent_state) == len(children)
            states = list(recurrent_state)
        batch_sizes, sorted_indices = get_packed_sequence_info(sequences)
        new_states = []
        h = sequences
        packed = True
        for layer in self:
            if is_recurrent(layer):
                if not packed:
                    h = wrap_packed_sequences_recursive(h, batch_sizes, sorted_indices)
                    packed = True
                h, rs = layer(h, states[len(new_states)])
                new_states.append(rs)
            else:
                if packed:
                    h = unwrap_packed_sequences_recursive(h)
                    packed = False
                h = layer(h)
        if not packed:
            h = wrap_packed_sequences_recursive(h, batch_sizes, sorted_indices)
        assert len(new_states) == len(children)
        return h, tuple(new_states)

    @property
    def recurrent_children(self):
        """The children that carry a recurrent state, in order."""
        return tuple(child for child in self if is_recurrent(child))


class RecurrentBranched(Recurrent, nn.ModuleList):
    """Runs every (recurrent) child on the same input; the output and the state
    are tuples with one entry per child (recurrent analog of ``Branched``)."""

    def __init__(self, *modules):
        super().__init__(modules)

    def forward(self, sequences, recurrent_state):
        if recurrent_state is None:
            recurrent_state = [None] * len(self)
        outs, states = [], []
        for child, rs in zip(self, recurrent_state):
            y, new_rs = child(sequences, rs)
            outs.append(y)
            states.append(new_rs)
        return tuple(outs), tuple(states)
