"""GPU: agents on the device replay path (HBM buffers + fused kernels)."""
import numpy as np
import pytest
import torch
from torch import nn

pytestmark = pytest.mark.gpu


def _rainbow(num_steps=3, capacity=4096, batch=32, n_actions=6):
    from pfrl_b200 import agents, explorers, nn as pnn, q_functions
    from pfrl_b200.replay_buffers import PrioritizedReplayBuffer
    from pfrl_b200.utils.phi import ScaleU8

    q = q_functions.DistributionalDuelingDQN(n_actions, 51, -10, 10)
    pnn.to_factorized_noisy(q, sigma_scale=0.5)
    opt = torch.optim.Adam(q.parameters(), 6.25e-5, eps=1.5e-4)
    rbuf = PrioritizedReplayBuffer(capacity, alpha=0.5, beta0=0.4, betasteps=1000,
                                   num_steps=num_steps, normalize_by_max="memory")
    return agents.CategoricalDoubleDQN(
        q, opt, rbuf, gpu=0, gamma=0.99, explorer=explorers.Greedy(), minibatch_size=batch,
        replay_start_size=200, target_update_interval=400, update_interval=4,
        batch_accumulator="mean", phi=ScaleU8())


@pytest.mark.parametrize("env_device", ["cuda", "cpu"])
def test_rainbow_trains_on_synthetic_atari(env_device, tmp_path):
    from pfrl_b200 import experiments
    from pfrl_b200.envs import SyntheticAtariVectorEnv
    from pfrl_b200.utils import set_random_seed

    set_random_seed(0)
    agent = _rainbow()
    env = SyntheticAtariVectorEnv(4, device=env_device, seed=0, n_actions=6, mean_episode_len=50)
    experiments.train_agent_batch(agent, env, 600, str(tmp_path), max_episode_len=80)
    stats = dict(agent.get_statistics())
    assert stats["n_updates"] == (600 - 200) // 4 + 1 or stats["n_updates"] > 90
    assert np.isfinite(stats["average_loss"]) and np.isfinite(stats["average_q"])
    assert stats["rlen"] == len(agent.replay_buffer) > 500
    # frames are shared: ~1 new part per env step (+ resets), not 8
    assert agent.replay_buffer._part_head < 600 * 1.2 + 64


def test_fused_losses_match_torch_formulation():
    """Same batch, same weights: fused TD / C51 kernels vs the reference
    formulas in torch, loss and gradients (fp32, 1e-5)."""
    from pfrl_b200 import agents, explorers, q_functions
    from pfrl_b200.replay_buffers import PrioritizedReplayBuffer

    torch.manual_seed(0)
    B, obs = 64, 12
    dev = torch.device("cuda")
    batch = {
        "state": torch.randn(B, obs, device=dev), "next_state": torch.randn(B, obs, device=dev),
        "action": torch.randint(0, 5, (B,), device=dev),
        "reward": torch.randn(B, device=dev), "discount": torch.full((B,), 0.97, device=dev),
        "is_state_terminal": (torch.rand(B, device=dev) < 0.2).float(),
        "weights": torch.rand(B, device=dev) + 0.1,
    }
    for cls, qf in (
        (agents.DoubleDQN, q_functions.FCStateQFunctionWithDiscreteAction(obs, 5, 64, 2)),
        (agents.DQN, q_functions.FCStateQFunctionWithDiscreteAction(obs, 5, 64, 2)),
        (agents.CategoricalDoubleDQN,
         q_functions.DistributionalFCStateQFunctionWithDiscreteAction(obs, 5, 51, -10, 10, 64, 2)),
    ):
        agent = cls(qf, torch.optim.SGD(qf.parameters(), lr=0.0), PrioritizedReplayBuffer(100),
                    0.99, explorers.Greedy(), gpu=0, replay_start_size=10, minibatch_size=8)
        res = {}
        for fused in (True, False):
            agent.use_fused_loss = fused
            agent.model.zero_grad()
            loss, delta = agent._compute_loss(dict(batch), want_errors=True)
            loss.backward()
            res[fused] = (loss.item(), delta.clone(),
                          [p.grad.clone() for p in agent.model.parameters()])
        np.testing.assert_allclose(res[True][0], res[False][0], rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(res[True][1], res[False][1], rtol=1e-5, atol=1e-6)
        for a, b in zip(res[True][2], res[False][2]):
            torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-6)


def test_ppo_on_device_env():
    from pfrl_b200 import agents, nn as pnn, policies
    from pfrl_b200.envs import SyntheticContinuousVectorEnv
    from pfrl_b200.utils import set_random_seed

    set_random_seed(0)
    obs_dim, act_dim = 24, 5
    model = nn.Sequential(
        nn.Linear(obs_dim, 64), nn.Tanh(),
        pnn.Branched(
            nn.Sequential(nn.Linear(64, act_dim),
                          policies.GaussianHeadWithStateIndependentCovariance(
                              action_size=act_dim, var_type="diagonal",
                              var_func=lambda x: torch.exp(2 * x), var_param_init=0)),
            nn.Linear(64, 1)))
    normalizer = pnn.EmpiricalNormalization(obs_dim, clip_threshold=5)
    opt = torch.optim.Adam(model.parameters(), lr=3e-4, eps=1e-5)
    res = {}
    for fused in (True, False, "graph"):
        set_random_seed(1)
        import copy

        m, nrm = copy.deepcopy(model), copy.deepcopy(normalizer)
        agent = agents.PPO(m, torch.optim.Adam(m.parameters(), lr=3e-4, eps=1e-5),
                           obs_normalizer=nrm, gpu=0, gamma=0.995, lambd=0.95,
                           update_interval=16 * 32, minibatch_size=64, epochs=2, clip_eps=0.2,
                           clip_eps_vf=None, entropy_coef=0.0, cuda_graph=fused == "graph")
        agent.use_fused = bool(fused)
        env = SyntheticContinuousVectorEnv(16, obs_dim, act_dim, device="cuda", seed=3,
                                           mean_episode_len=20)
        obs = env.reset()
        for _ in range(70):
            a = agent.batch_act(obs)
            obs, r, d, info = env.step(a)
            agent.batch_observe(obs, r, d, np.zeros(16, dtype=bool))
            obs = env.reset(np.logical_not(d))
        assert agent.n_updates == 2 * (2 * 16 * 32 // 64)
        res[fused] = [p.detach().clone() for p in agent.model.parameters()]
        stats = dict(agent.get_statistics())
        assert np.isfinite(stats["average_value_loss"]) and np.isfinite(stats["explained_variance"])
    # the fused GAE + loss kernels and the torch formulation give the same training run,
    # and so does replaying the minibatch step as a CUDA graph
    for a, b, c in zip(res[True], res[False], res["graph"]):
        torch.testing.assert_close(a, b, rtol=2e-3, atol=2e-5)
        torch.testing.assert_close(a, c, rtol=2e-3, atol=2e-5)


@pytest.mark.parametrize("use_graph", [False, True])
def test_sac_on_device_env(use_graph):
    from torch import distributions

    from pfrl_b200 import agents, nn as pnn
    from pfrl_b200.envs import SyntheticContinuousVectorEnv
    from pfrl_b200.replay_buffers import ReplayBuffer
    from pfrl_b200.utils import set_random_seed
    from pfrl_b200.utils.phi import Identity

    set_random_seed(0)
    obs_dim, act_dim = 17, 6

    def squashed(x):
        mean, log_scale = torch.chunk(x, 2, dim=1)
        base = distributions.Independent(
            distributions.Normal(mean, torch.exp(torch.clamp(log_scale, -20, 2))), 1)
        return distributions.transformed_distribution.TransformedDistribution(
            base, [distributions.transforms.TanhTransform(cache_size=1)])

    policy = nn.Sequential(nn.Linear(obs_dim, 64), nn.ReLU(), nn.Linear(64, 2 * act_dim),
                           pnn.Lambda(squashed))

    def qf():
        return nn.Sequential(pnn.ConcatObsAndAction(), nn.Linear(obs_dim + act_dim, 64), nn.ReLU(),
                             nn.Linear(64, 1))

    q1, q2 = qf(), qf()
    agent = agents.SoftActorCritic(
        policy, q1, q2, torch.optim.Adam(policy.parameters(), lr=3e-4),
        torch.optim.Adam(q1.parameters(), lr=3e-4), torch.optim.Adam(q2.parameters(), lr=3e-4),
        ReplayBuffer(10 ** 4), gamma=0.99, gpu=0, replay_start_size=128, minibatch_size=64,
        entropy_target=-act_dim, temperature_optimizer_lr=3e-4, phi=Identity(),
        cuda_graph=use_graph)
    env = SyntheticContinuousVectorEnv(8, obs_dim, act_dim, device="cuda", seed=1,
                                       mean_episode_len=30)
    obs = env.reset()
    for _ in range(60):
        a = agent.batch_act(obs)
        obs, r, d, info = env.step(a)
        agent.batch_observe(obs, r, d, np.zeros(8, dtype=bool))
        obs = env.reset(np.logical_not(d))
    stats = dict(agent.get_statistics())
    assert stats["n_updates"] > 300 and np.isfinite(stats["average_q1"])
    assert np.isfinite(stats["average_q_func1_loss"]) and np.isfinite(stats["average_entropy"])
    assert len(agent.replay_buffer) == 8 * 60
    if use_graph:
        assert agent._graph.graph is not None  # the update really ran as a captured graph



def test_iqn_on_device_replay_and_fused_loss():
    """IQN: fused quantile-Huber kernel == torch formulation on the same taus,
    and a short training run on the device PER."""
    from pfrl_b200 import agents, explorers
    from pfrl_b200.agents import iqn
    from pfrl_b200.envs import SyntheticContinuousVectorEnv
    from pfrl_b200.replay_buffers import PrioritizedReplayBuffer
    from pfrl_b200.utils import set_random_seed
    from pfrl_b200.utils.phi import Identity

    set_random_seed(0)
    obs_dim, n_actions, hidden = 12, 4, 32
    q = iqn.ImplicitQuantileQFunction(
        psi=nn.Sequential(nn.Linear(obs_dim, hidden), nn.ReLU()),
        phi=nn.Sequential(iqn.CosineBasisLinear(16, hidden), nn.ReLU()),
        f=nn.Linear(hidden, n_actions))
    agent = agents.IQN(
        q, torch.optim.Adam(q.parameters(), lr=1e-3), PrioritizedReplayBuffer(5000, num_steps=2),
        0.99, explorers.ConstantEpsilonGreedy(0.2, lambda: np.random.randint(n_actions)), gpu=0,
        replay_start_size=64, minibatch_size=32, target_update_interval=50, phi=Identity(),
        quantile_thresholds_N=8, quantile_thresholds_N_prime=8, quantile_thresholds_K=4)
    # loss equivalence with identical taus
    B = 16
    y = torch.randn(B, 8, device="cuda", requires_grad=True)
    t = torch.randn(B, 8, device="cuda")
    taus = torch.rand(B, 8, device="cuda")
    w = torch.rand(B, device="cuda") + 0.1
    from pfrl_b200.ops.losses import quantile_huber_loss

    loss_f, err_f = quantile_huber_loss(y, t, taus, w, mean=True)
    elt = iqn.compute_eltwise_huber_quantile_loss(y, t, taus)
    loss_t = iqn.compute_weighted_value_loss(elt, w, "mean")
    torch.testing.assert_close(loss_f, loss_t, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(err_f, elt.detach().mean((1, 2)), rtol=1e-5, atol=1e-6)
    g_f, = torch.autograd.grad(loss_f, y)
    g_t, = torch.autograd.grad(loss_t, y)
    torch.testing.assert_close(g_f, g_t, rtol=1e-4, atol=1e-7)
    # short run
    env = SyntheticContinuousVectorEnv(4, obs_dim, 1, device="cuda", seed=2, mean_episode_len=25)
    obs = env.reset()
    for _ in range(60):
        a = agent.batch_act(obs)
        obs, r, d, info = env.step(a)
        agent.batch_observe(obs, r, d, np.zeros(4, dtype=bool))
        obs = env.reset(np.logical_not(d))
    stats = dict(agent.get_statistics())
    assert stats["n_updates"] > 100 and np.isfinite(stats["average_loss"])


def test_dqn_update_as_cuda_graph_matches_eager():
    """cuda_graph=True replays forward + fused TD loss + backward + Adam as one
    graph: same parameters as the eager path after the same seeded run."""
    from pfrl_b200 import agents, explorers, q_functions
    from pfrl_b200.envs import SyntheticContinuousVectorEnv
    from pfrl_b200.replay_buffers import PrioritizedReplayBuffer
    from pfrl_b200.utils import set_random_seed
    from pfrl_b200.utils.phi import Identity

    res = {}
    for graph in (False, True):
        set_random_seed(3)
        q = q_functions.FCStateQFunctionWithDiscreteAction(12, 4, 64, 2)
        agent = agents.DoubleDQN(
            # capturable=True in BOTH runs: Adam's capturable path keeps `step` and the
            # bias corrections on the device (fp32), the default path computes them on the
            # host in fp64 -- a 1e-7 difference that prioritized sampling would amplify
            q.cuda(), torch.optim.Adam(q.parameters(), lr=1e-3, capturable=True),
            PrioritizedReplayBuffer(4096, num_steps=3),
            0.99, explorers.ConstantEpsilonGreedy(0.3, lambda: np.random.randint(4)), gpu=0,
            replay_start_size=64, minibatch_size=32, target_update_interval=40, phi=Identity(),
            cuda_graph=graph)
        env = SyntheticContinuousVectorEnv(4, 12, 1, device="cuda", seed=5, mean_episode_len=20)
        obs = env.reset()
        for _ in range(80):
            a = agent.batch_act(obs)
            obs, r, d, info = env.step(a)
            agent.batch_observe(obs, r, d, np.zeros(4, dtype=bool))
            obs = env.reset(np.logical_not(d))
        assert agent.optim_t > 200
        assert (agent._graph is not None and agent._graph.graph is not None) == graph
        res[graph] = ([p.detach().clone() for p in agent.model.parameters()],
                      dict(agent.get_statistics()))
    for a, b in zip(res[False][0], res[True][0]):
        torch.testing.assert_close(a, b, rtol=1e-3, atol=1e-5)
    assert abs(res[False][1]["average_loss"] - res[True][1]["average_loss"]) < 1e-3


def test_td3_on_device_replay():
    from pfrl_b200 import agents, explorers, nn as pnn, policies
    from pfrl_b200.envs import SyntheticContinuousVectorEnv
    from pfrl_b200.replay_buffers import ReplayBuffer
    from pfrl_b200.utils import set_random_seed
    from pfrl_b200.utils.phi import Identity

    set_random_seed(0)
    obs_dim, act_dim = 17, 6
    p = nn.Sequential(nn.Linear(obs_dim, 64), nn.ReLU(), nn.Linear(64, act_dim), nn.Tanh(),
                      policies.DeterministicHead())

    def qf():
        return nn.Sequential(pnn.ConcatObsAndAction(), nn.Linear(obs_dim + act_dim, 64), nn.ReLU(),
                             nn.Linear(64, 1))

    q1, q2 = qf(), qf()
    agent = agents.TD3(
        p, q1, q2, torch.optim.Adam(p.parameters(), lr=3e-4),
        torch.optim.Adam(q1.parameters(), lr=3e-4), torch.optim.Adam(q2.parameters(), lr=3e-4),
        ReplayBuffer(10 ** 4), 0.99, explorers.AdditiveGaussian(0.1, -1, 1), gpu=0,
        replay_start_size=128, minibatch_size=64, phi=Identity())
    env = SyntheticContinuousVectorEnv(8, obs_dim, act_dim, device="cuda", seed=1,
                                       mean_episode_len=30)
    obs = env.reset()
    for _ in range(50):
        a = agent.batch_act(obs)
        obs, r, d, info = env.step(a)
        agent.batch_observe(obs, r, d, np.zeros(8, dtype=bool))
        obs = env.reset(np.logical_not(d))
    stats = dict(agent.get_statistics())
    assert stats["q_func_n_updates"] > 200 and stats["policy_n_updates"] > 100
    assert np.isfinite(stats["average_q1"]) and np.isfinite(stats["average_policy_loss"])


@pytest.mark.gpu
def test_empirical_normalization_on_cuda_matches_reference_golden():
    """SURVEY 8 a13: pfrl/nn/empirical_normalization.py:61-105 on cuda:0 against the fixture the
    real reference produced (the same one the CPU suite checks), tolerance 1e-5."""
    import os

    import numpy as np

    from pfrl_b200.nn import EmpiricalNormalization

    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "empirical_normalization.npz"))
    en = EmpiricalNormalization(7, clip_threshold=5).cuda()
    for i in range(4):
        y = en(torch.tensor(g["x%d" % i], device="cuda"), update=True).cpu().numpy()
        np.testing.assert_allclose(y, g["y%d" % i], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(en.mean.cpu().numpy(), g["mean"], rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(en.std.cpu().numpy(), g["std"], rtol=1e-6)
    assert int(en.count) == int(g["count"])
    out = en(torch.tensor(g["probe"], device="cuda"), update=False).cpu().numpy()
    np.testing.assert_allclose(out, g["probe_out"], rtol=1e-5, atol=1e-6)
