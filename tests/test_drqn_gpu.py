"""Recurrent DQN / DoubleDQN on cuda:0: the device episodic buffer (one-launch packed
gather, states kept on the device) against the host buffer, and no device-to-host copy
when transitions with recurrent states are stored."""
import numpy as np
import pytest
import torch

import pfrl_b200
from pfrl_b200 import replay_buffers
from pfrl_b200.utils.phi import Identity

import test_drqn_cpu as cpu

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("cls_name", ["DQN", "DoubleDQN"])
@pytest.mark.parametrize("rnn,ep_len", [("rnn", None), ("lstm", 3)])
def test_device_buffer_equals_host_buffer_on_cuda(cls_name, rnn, ep_len):
    cls = getattr(pfrl_b200.agents, cls_name)
    a = cpu._agent(cls, replay_buffers.HostEpisodicReplayBuffer(60), rnn, gpu=0,
                   episodic_update_len=ep_len)
    b = cpu._agent(cls, replay_buffers.EpisodicReplayBuffer(60), rnn, gpu=0,
                   episodic_update_len=ep_len, phi=Identity())
    acts_a = cpu._run(a, 80, seed=5)
    acts_b = cpu._run(b, 80, seed=5)
    assert a.optim_t > 10 and a.optim_t == b.optim_t
    assert acts_a == acts_b
    for p, q in zip(a.model.parameters(), b.model.parameters()):
        torch.testing.assert_close(p, q, rtol=1e-5, atol=1e-6)


def test_drqn_lstm512_synthetic_atari_and_no_d2h_in_observe():
    from pfrl_b200.envs.synthetic import SyntheticAtariVectorEnv
    from pfrl_b200.nn import RecurrentSequential
    from pfrl_b200.q_functions import DiscreteActionValueHead
    from torch import nn

    torch.manual_seed(0)
    q = RecurrentSequential(
        nn.Conv2d(4, 32, 8, stride=4), nn.ReLU(), nn.Conv2d(32, 64, 4, stride=2), nn.ReLU(),
        nn.Conv2d(64, 64, 3, stride=1), nn.Flatten(), nn.ReLU(), nn.Linear(3136, 512),
        nn.ReLU(), nn.LSTM(512, 512), nn.Linear(512, 18), DiscreteActionValueHead())
    agent = pfrl_b200.agents.DoubleDQN(
        q, torch.optim.Adam(q.parameters(), 1e-4), replay_buffers.EpisodicReplayBuffer(10 ** 4),
        0.99, pfrl_b200.explorers.ConstantEpsilonGreedy(0.1, lambda: np.random.randint(18)),
        gpu=0, replay_start_size=200, minibatch_size=8, update_interval=4,
        target_update_interval=100, recurrent=True, episodic_update_len=10,
        phi=pfrl_b200.utils.phi.ScaleU8())
    env = SyntheticAtariVectorEnv(2, device="cuda", seed=0, mean_episode_len=40)
    obs = env.reset()
    for t in range(400):
        acts = agent.batch_act(obs)
        obs, rew, done, info = env.step(acts)
        rew, done = (x.cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)
                     for x in (rew, done))
        reset = [bool(d) for d in done]
        if t == 399:
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                agent.batch_observe(obs, rew, done, reset)
                torch.cuda.synchronize()
            names = [e.name for e in prof.events()]
            assert not any("DtoH" in n or "Device -> Pageable" in n for n in names), names
        else:
            agent.batch_observe(obs, rew, done, reset)
        if any(reset):
            obs = env.reset(np.logical_not(reset))  # mask: True = keep running
    assert agent.optim_t > 10
    assert np.isfinite(agent.get_statistics()[1][1])
