"""GPU: AL, PAL, DoublePAL, DPP, DPPL and DPPGreedy through the fused target-and-loss kernel
(k_adv_td_fwd) on the device replay path:

* the reference's fixed-batch losses (tests/golden/advantage_losses.npz) through the fused
  path, and the same agent's torch formulation on CUDA;
* training on a device PrioritizedReplayBuffer with the fused replay step and with separate
  launches: same sampled indices, trees and parameters, bit for bit;
* cuda_graph=True against eager;
* a small AL run on the synthetic Atari environment (84x84x4 uint8, 18 actions).
"""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))
from test_advantage_agents_cpu import check_fixed_batch_losses  # noqa: E402

from oracle.gen_golden_advantage import ADV_AGENTS, LOSS_NA  # noqa: E402

pytestmark = pytest.mark.gpu

CLASSES = {"al": "AL", "pal": "PAL", "double_pal": "DoublePAL", "dpp": "DPP", "dppl": "DPPL",
           "dpp_greedy": "DPPGreedy"}


@pytest.mark.parametrize("nA", LOSS_NA)
@pytest.mark.parametrize("kind", list(ADV_AGENTS))
def test_fused_fixed_batch_losses_match_reference_and_torch_path(kind, nA):
    torch.backends.cuda.matmul.allow_tf32 = False
    agent, fused = check_fixed_batch_losses(kind, nA, "cuda", gradnorm_rtol=1e-4)
    assert agent.use_fused_loss
    _, torch_path = check_fixed_batch_losses(kind, nA, "cuda", gradnorm_rtol=1e-4,
                                             use_fused_loss=False)
    for use_w in (1, 0):
        np.testing.assert_allclose(fused[use_w][0], torch_path[use_w][0], rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(fused[use_w][1], torch_path[use_w][1], rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(fused[use_w][2], torch_path[use_w][2], rtol=1e-5)


def _agent_class(kind):
    from pfrl_b200.agents import dpp

    import pfrl_b200.agents as agents

    return getattr(agents, CLASSES[kind], None) or getattr(dpp, CLASSES[kind])


def _train(kind, fused_step=True, graph=False, steps=80):
    """A seeded run on 4 device environments with 3-step prioritised replay; returns the
    sampled indices of every update, the parameters, the statistics and the buffer."""
    from pfrl_b200 import explorers, q_functions
    from pfrl_b200.envs import SyntheticContinuousVectorEnv
    from pfrl_b200.replay_buffers import PrioritizedReplayBuffer
    from pfrl_b200.utils import set_random_seed
    from pfrl_b200.utils.phi import Identity

    set_random_seed(3)
    q = q_functions.FCStateQFunctionWithDiscreteAction(12, 4, 64, 2)
    rbuf = PrioritizedReplayBuffer(4096, alpha=0.6, beta0=0.4, betasteps=200, num_steps=3,
                                   fused=fused_step)
    kw = dict(ADV_AGENTS[kind][2])
    agent = _agent_class(kind)(
        # capturable Adam in every run (see tests/test_agents_gpu.py)
        q.cuda(), torch.optim.Adam(q.parameters(), lr=1e-3, capturable=True), rbuf, 0.99,
        explorers.ConstantEpsilonGreedy(0.3, lambda: np.random.randint(4)), gpu=0,
        replay_start_size=64, minibatch_size=32, target_update_interval=40, phi=Identity(),
        cuda_graph=graph, **kw)
    indices = []
    sample = rbuf.sample

    def recording_sample(n):
        exps = sample(n)
        indices.append(exps.index.clone())
        return exps

    rbuf.sample = recording_sample
    env = SyntheticContinuousVectorEnv(4, 12, 1, device="cuda", seed=5, mean_episode_len=20)
    obs = env.reset()
    for _ in range(steps):
        a = agent.batch_act(obs)
        obs, r, d, info = env.step(a)
        agent.batch_observe(obs, r, d, np.zeros(4, dtype=bool))
        obs = env.reset(np.logical_not(d))
    assert agent.optim_t > 200
    assert (agent._graph is not None and agent._graph.graph is not None) == graph
    params = [p.detach().clone() for p in agent.model.parameters()]
    return indices, params, dict(agent.get_statistics()), rbuf


@pytest.mark.parametrize("kind", ["pal", "dpp"])
def test_fused_replay_step_matches_separate_launches(kind):
    runs = [_train(kind, fused_step=f) for f in (True, False)]
    (ia, pa, sa, ba), (ib, pb, sb, bb) = runs
    assert len(ia) == len(ib) and all(torch.equal(x, y) for x, y in zip(ia, ib))
    assert all(torch.equal(x, y) for x, y in zip(pa, pb))
    ba._flush()
    bb._flush()
    fa, fb = ba.store.info(), bb.store.info()
    for k in ("total", "min", "max_priority", "napp", "npop"):
        assert fa[k] == fb[k], k
    assert np.array_equal(ba.store.read_priorities(), bb.store.read_priorities())
    assert sa["average_loss"] == sb["average_loss"] and np.isfinite(sa["average_loss"])


@pytest.mark.parametrize("kind", list(CLASSES))
def test_update_as_cuda_graph_matches_eager(kind):
    """cuda_graph=True replays the forwards, k_adv_td_fwd, backward and Adam as one graph."""
    _, eager, se, _ = _train(kind, graph=False)
    _, graphed, sg, _ = _train(kind, graph=True)
    for a, b in zip(eager, graphed):
        torch.testing.assert_close(a, b, rtol=1e-3, atol=1e-5)
    assert abs(se["average_loss"] - sg["average_loss"]) < 1e-3


def test_al_trains_on_synthetic_atari(tmp_path):
    from pfrl_b200 import agents, experiments, explorers, q_functions
    from pfrl_b200.envs import SyntheticAtariVectorEnv
    from pfrl_b200.replay_buffers import PrioritizedReplayBuffer
    from pfrl_b200.utils import set_random_seed
    from pfrl_b200.utils.phi import ScaleU8

    set_random_seed(0)
    q = q_functions.DuelingDQN(18)
    rbuf = PrioritizedReplayBuffer(4096, alpha=0.5, beta0=0.4, betasteps=1000, num_steps=3)
    agent = agents.AL(q, torch.optim.Adam(q.parameters(), 6.25e-5, eps=1.5e-4), rbuf, 0.99,
                      explorers.ConstantEpsilonGreedy(0.1, lambda: np.random.randint(18)),
                      gpu=0, minibatch_size=32, replay_start_size=200,
                      target_update_interval=400, update_interval=4, phi=ScaleU8())
    env = SyntheticAtariVectorEnv(4, device="cuda", seed=0, n_actions=18, mean_episode_len=50)
    experiments.train_agent_batch(agent, env, 600, str(tmp_path), max_episode_len=80)
    stats = dict(agent.get_statistics())
    assert stats["n_updates"] > 90
    assert np.isfinite(stats["average_loss"]) and np.isfinite(stats["average_q"])


def test_user_dpp_operator_runs_its_own_target_on_cuda():
    """An AbstractDPP subclass with its own L operator has no kernel mode: with the default
    use_fused_loss it computes its own torch target on CUDA, the same as with the flag off."""
    from pfrl_b200 import explorers, q_functions
    from pfrl_b200.agents.dpp import AbstractDPP
    from pfrl_b200.replay_buffers import HostReplayBuffer

    class MeanDPP(AbstractDPP):
        def _l_operator(self, qout):
            return qout.q_values.mean(dim=1)

    torch.manual_seed(0)
    B, obs, nA = 40, 10, 5
    dev = torch.device("cuda")
    batch = {"state": torch.randn(B, obs, device=dev), "next_state": torch.randn(B, obs, device=dev),
             "action": torch.randint(0, nA, (B,), device=dev), "reward": torch.randn(B, device=dev),
             "discount": torch.full((B,), 0.99, device=dev),
             "is_state_terminal": (torch.rand(B, device=dev) < 0.2).float(),
             "weights": torch.rand(B, device=dev) + 0.1}
    qf = q_functions.FCStateQFunctionWithDiscreteAction(obs, nA, 32, 2)
    agent = MeanDPP(qf, torch.optim.SGD(qf.parameters(), lr=0.0), HostReplayBuffer(100), 0.99,
                    explorers.Greedy(), gpu=0, replay_start_size=10, minibatch_size=8)
    res = {}
    for flag in (True, False):
        agent.use_fused_loss = flag
        loss, delta = agent._compute_loss(dict(batch), want_errors=True)
        res[flag] = (loss.item(), delta.cpu())
    y, t = agent._compute_y_and_t(dict(batch))
    assert res[True][0] == res[False][0]
    assert torch.equal(res[True][1], res[False][1])
    assert torch.equal(res[True][1], (y.detach() - t).abs().sum(dim=1).cpu())
