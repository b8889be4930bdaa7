"""Recurrent DQN / DoubleDQN replay the seeded runs of the REAL reference step by step on
CPU (tests/golden/agent_trace_drqn_*.npz, written by oracle/gen_golden_drqn.py): the
actions of every step, the episodes and window starts every update samples, the statistics
after every vector step and the final parameters.  Once with HostEpisodicReplayBuffer and
once with the device EpisodicReplayBuffer over tests/fake_episodic_store.py (its real host
logic: episode table, eviction, state ring, packing)."""
import os
from unittest import mock

import numpy as np
import pytest
import torch

import pfrl_b200
from fake_episodic_store import EpisodicOracleStore
from oracle.gen_golden_drqn import (
    CAPACITY, DRQN_KINDS, make_drqn_agent, record_episode_samples, run_drqn_trace,
)

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def record_device_samples(rbuf, log):
    """sample_episodes of the device buffer -> (episode commit numbers, window starts)."""
    raw = rbuf.sample_episodes

    def sample_episodes(n_episodes, max_len=None):
        eps = raw(n_episodes, max_len)
        table = [(f, L) for f, L, _ in rbuf._episodes]
        popped = rbuf._ep_count - len(table)
        ids, starts = [], []
        for first in eps.first.tolist():
            i = next(i for i, (f, L) in enumerate(table) if f <= first < f + L)
            ids.append(popped + i)
            starts.append(first - table[i][0])
        log.append((ids, starts))
        return eps

    rbuf.sample_episodes = sample_episodes


def replay(kind, buffer, gpu=None, check_actions=None):
    """Run this package's agent on the reference's trace; returns (golden, agent, actions,
    stats, sample log)."""
    g = np.load(os.path.join(GOLD, "agent_trace_drqn_%s.npz" % kind))
    log = []
    if buffer == "host":
        rbuf = pfrl_b200.replay_buffers.HostEpisodicReplayBuffer(CAPACITY)
        record_episode_samples(rbuf, log)
        phi = None
    else:
        rbuf = pfrl_b200.replay_buffers.EpisodicReplayBuffer(
            CAPACITY, device=None if gpu is None else gpu)
        record_device_samples(rbuf, log)
        phi = pfrl_b200.utils.phi.Identity()  # float32 observations: raw copy
    torch.manual_seed(3)
    q, agent = make_drqn_agent(pfrl_b200, kind, rbuf, gpu=gpu, phi=phi)
    q.load_state_dict({k: torch.tensor(g["init_" + k]) for k in q.state_dict()})
    agent.target_model.load_state_dict(q.state_dict())
    np.random.seed(9)
    torch.manual_seed(9)

    def check(t, a):
        assert a == g["actions"][t].tolist(), "actions diverge at step %d" % t

    actions, stats = run_drqn_trace(agent, steps=g["actions"].shape[0], check=check)
    return g, q, stats, log


def check_samples(g, log):
    assert len(log) == g["sample_ids"].shape[0]
    assert np.array_equal(np.asarray([i for i, _ in log]), g["sample_ids"])
    assert np.array_equal(np.asarray([s for _, s in log]), g["sample_starts"])


@pytest.mark.parametrize("buffer", ["host", "device"])
@pytest.mark.parametrize("kind", list(DRQN_KINDS))
def test_drqn_reproduces_the_reference_run_on_cpu(kind, buffer):
    ctx = mock.patch("pfrl_b200.replay_buffers.device_buffer.DeviceReplayStore",
                     EpisodicOracleStore) if buffer == "device" else mock.patch.dict({})
    with ctx, mock.patch("torch.cuda.current_device", return_value=0):
        g, q, stats, log = replay(kind, buffer)
    check_samples(g, log)
    assert np.array_equal(stats[:, 2:], g["stats"][:, 2:])          # n_updates, rlen
    live = ~np.isnan(g["stats"][:, 0])
    np.testing.assert_allclose(stats[live, :2], g["stats"][live, :2], rtol=1e-5, atol=1e-6)
    for k, v in q.state_dict().items():
        np.testing.assert_allclose(v.numpy(), g["final_" + k], rtol=1e-5, atol=1e-6, err_msg=k)
