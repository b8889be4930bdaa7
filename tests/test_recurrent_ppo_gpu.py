"""Recurrent PPO on cuda:0 through k_rollout_seq_gather.

Every pack the agent launches (dataset pass and minibatches) is checked against the
torch formulation on the same tensors: the pack is a copy, so it must be bit-equal.
The kernel run and a use_fused=False run from the same seeds act alike, and their
parameters stay close (the fused loss and GAE kernels round differently from torch).
"""
import random

import numpy as np
import pytest
import torch

from pfrl_b200.agents.ppo import PPO
from pfrl_b200.ops import rollout
from test_recurrent_ppo_cpu import drive, make_agent

pytestmark = pytest.mark.gpu


def _bits(t):
    return t.detach().contiguous().reshape(-1).view(torch.uint8)


@pytest.mark.parametrize("kind,kw", [
    ("lstm", dict()),
    ("gru", dict(max_recurrent_sequence_len=3, lambd=0.5, minibatch_size=7)),
])
def test_every_pack_is_bit_equal_to_the_torch_formulation(kind, kw):
    agent = make_agent(kind, gpu=0, **kw)
    checked = []
    real = rollout.SequenceGather.__call__

    def checking(self, first, lens, E, columns, index=False, states=None):
        outs, idx, leaves = real(self, first, lens, E, columns, index, states)
        t_outs, t_idx, t_leaves = rollout.gather_sequences_torch(first, lens, E, columns, index,
                                                                states)
        for a, b in zip(outs, t_outs):
            assert a.dtype == b.dtype and torch.equal(_bits(a), _bits(b))
        if index:
            assert torch.equal(idx, t_idx)
        for side in t_leaves:
            for a, b in zip(leaves[side], t_leaves[side]):
                assert torch.equal(_bits(a), _bits(b))
        checked.append(len(first))
        return outs, idx, leaves

    rollout.SequenceGather.__call__ = checking
    try:
        drive(agent, 20, discrete=kind == "lstm")
    finally:
        rollout.SequenceGather.__call__ = real
    assert agent.n_updates > 0 and len(checked) > agent.n_updates


def test_kernel_path_tracks_the_torch_path():
    runs = []
    for fused in (True, False):
        agent = make_agent("lstm", gpu=0)
        agent.use_fused = fused
        random.seed(1)  # the epochs' shuffles
        torch.manual_seed(1)
        torch.cuda.manual_seed(1)
        actions = drive(agent, 12)
        runs.append((agent, actions))
    (a, acts_a), (b, acts_b) = runs
    assert a.n_updates == b.n_updates > 0
    # the first update's rollout is acted with the same parameters
    first = 6
    assert all(np.array_equal(x, y) for x, y in zip(acts_a[:first], acts_b[:first]))
    for p, q in zip(a.model.parameters(), b.model.parameters()):
        torch.testing.assert_close(p, q, rtol=1e-3, atol=1e-4)


def test_many_short_sequences():
    """Mostly one-step episodes: the dataset pass packs close to T * E sequences, more
    than a kernel-parameter table could hold at larger shapes (B is not capped)."""
    agent = make_agent("lstm", gpu=0, update_interval=40 * 8, minibatch_size=32)
    agent.phi = lambda x: x.astype(np.float32) / 255.0
    rng = np.random.RandomState(0)
    obs = [rng.randint(0, 256, 5).astype(np.uint8) for _ in range(8)]
    for _ in range(40):
        agent.batch_act(obs)
        obs = [rng.randint(0, 256, 5).astype(np.uint8) for _ in range(8)]
        done = rng.rand(8) < 0.7
        agent.batch_observe(obs, rng.randn(8), done, np.zeros(8, bool))
    assert agent.n_updates > 0
    assert np.isfinite(dict(agent.get_statistics())["average_value_loss"])


def test_recurrent_ppo_rejects_graph_capture_on_cuda():
    with pytest.raises(ValueError):
        make_agent("lstm", gpu=0, cuda_graph=True)
    assert isinstance(make_agent("lstm", gpu=0), PPO)
