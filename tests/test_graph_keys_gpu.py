"""cuda_graph=True follows what a capture bakes in.  A change to an optimizer's lr, to a loss
coefficient, to a batch layout or, for DQN on data-parallel ranks, the all-reduce between
its two graphs must reach the graphed agent exactly as it reaches an eager agent with the same
(capturable) optimizers.  Each change is made after the first update that replays a graph."""
import os
import random
import sys

import numpy as np
import pytest
import torch
from torch import distributions, nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.gen_golden_losses import _module_attrs, _run_more_trace  # noqa: E402
from oracle.gen_golden_trpo import TRPO_KINDS, make_trpo_agent  # noqa: E402

pytestmark = pytest.mark.gpu
PPO_TOL = dict(rtol=2e-3, atol=2e-5)  # test_ppo_on_device_env's graph-vs-eager bound


def _state(agent):
    return {"%s.%s" % (n, k): v.detach().cpu().clone()
            for n, m in _module_attrs(agent) for k, v in m.state_dict().items()}


def _assert_same(got, want, tol=None):
    assert got.keys() == want.keys()
    for k in want:
        if tol is None:
            assert torch.equal(got[k], want[k]), k
        else:
            torch.testing.assert_close(got[k], want[k], **tol, msg=lambda m: "%s: %s" % (k, m))


def _set_lr(*optimizers, factor=0.01):
    for opt in optimizers:
        for group in opt.param_groups:
            group["lr"] *= factor


def _experiences(rng, n, obs_dim, discrete):
    def transition():
        return dict(state=rng.randn(obs_dim).astype(np.float32),
                    action=int(rng.randint(3)) if discrete else rng.uniform(
                        -1, 1, 1).astype(np.float32),
                    reward=float(rng.randn()), next_state=rng.randn(obs_dim).astype(np.float32),
                    is_state_terminal=bool(rng.rand() < 0.1), next_action=None)

    return [[transition()] for _ in range(n)]


class _DoublingSync:
    """A one-rank stand-in for parallel.GradSync whose collective doubles the bucket: a
    skipped reduce changes the parameters, and ``reduces`` counts the eager calls."""

    def __init__(self):
        self.flat = None
        self.reduces = 0

    def pack(self, model):
        grads = [p.grad.reshape(-1) for p in model.parameters()]
        if self.flat is None:
            self.flat = torch.zeros(sum(g.numel() for g in grads), device=grads[0].device)
        self.flat.copy_(torch.cat(grads))

    def reduce(self, model):
        self.reduces += 1
        self.flat.mul_(2)

    def unpack(self, model):
        off = 0
        for p in model.parameters():
            p.grad.copy_(self.flat[off:off + p.numel()].view_as(p))
            off += p.numel()

    def __call__(self, model):
        self.pack(model)
        self.reduce(model)
        self.unpack(model)


@pytest.mark.parametrize("change", ["lr", "layout", "grad_sync"])
def test_dqn_graph_follows_changes(change):
    from pfrl_b200 import agents, explorers, q_functions
    from pfrl_b200.replay_buffers import ReplayBuffer

    rng = np.random.RandomState(0)
    batches = [_experiences(rng, 24 if change == "layout" and u == 5 else 32, 6, True)
               for u in range(10)]
    runs = []
    for graph in (False, True):
        torch.manual_seed(0)
        q = q_functions.FCStateQFunctionWithDiscreteAction(6, 3, 32, 1).cuda()
        sync = _DoublingSync() if change == "grad_sync" else None
        agent = agents.DoubleDQN(
            q, torch.optim.Adam(q.parameters(), lr=1e-2, capturable=True), ReplayBuffer(100),
            0.9, explorers.Greedy(), gpu=0, replay_start_size=32, minibatch_size=32,
            max_grad_norm=1.0, grad_sync=sync, cuda_graph=graph)
        for u, batch in enumerate(batches):
            if change == "lr" and u == 4:  # update 3 is the first replay
                _set_lr(agent.optimizer)
            agent.update(batch)
        runs.append((agent, _state(agent), sync))
    (_, eager, sync_e), (agent, graphed, sync_g) = runs
    _assert_same(graphed, eager)
    if change == "grad_sync":
        assert sync_e.reduces == sync_g.reduces == len(batches)
    assert agent._graph.graph is not None


def _sac(graph):
    from pfrl_b200 import agents, nn as pnn
    from pfrl_b200.replay_buffers import ReplayBuffer

    def squashed(x):
        mean, log_scale = torch.chunk(x, 2, dim=1)
        base = distributions.Independent(
            distributions.Normal(mean, torch.exp(torch.clamp(log_scale, -5, 2))), 1)
        return distributions.transformed_distribution.TransformedDistribution(
            base, [distributions.transforms.TanhTransform(cache_size=1)])

    def qf():
        return nn.Sequential(pnn.ConcatObsAndAction(), nn.Linear(6, 32), nn.ReLU(),
                             nn.Linear(32, 1))

    policy = nn.Sequential(nn.Linear(5, 32), nn.ReLU(), nn.Linear(32, 2), pnn.Lambda(squashed))
    q1, q2 = qf(), qf()
    opts = [torch.optim.Adam(m.parameters(), lr=1e-2, capturable=True) for m in (policy, q1, q2)]
    agent = agents.SoftActorCritic(
        policy, q1, q2, *opts, ReplayBuffer(100), gamma=0.95, gpu=0, replay_start_size=16,
        minibatch_size=16, entropy_target=-1.0, temperature_optimizer_lr=1e-2, cuda_graph=graph)
    for group in agent.temperature_optimizer.param_groups:
        group["capturable"] = True
    return agent


def test_sac_graph_follows_lr():
    rng = np.random.RandomState(1)
    batches = [_experiences(rng, 16, 5, False) for _ in range(10)]
    runs = []
    for graph in (False, True):
        torch.manual_seed(0)
        agent = _sac(graph)
        for u, batch in enumerate(batches):
            if u == 4:
                _set_lr(agent.policy_optimizer, agent.q_func1_optimizer,
                        agent.q_func2_optimizer, agent.temperature_optimizer)
            agent.update(batch)
        runs.append((agent, _state(agent)))
    _assert_same(runs[1][1], runs[0][1], PPO_TOL)
    assert runs[1][0]._graph.graph is not None


def _ppo(graph):
    import pfrl_b200
    from pfrl_b200 import agents

    model = nn.Sequential(nn.Linear(5, 32), nn.Tanh(), pfrl_b200.nn.Branched(
        nn.Sequential(nn.Linear(32, 2), pfrl_b200.policies.SoftmaxCategoricalHead()),
        nn.Linear(32, 1)))
    return agents.PPO(
        model, torch.optim.Adam(model.parameters(), lr=1e-2, capturable=True),
        obs_normalizer=pfrl_b200.nn.EmpiricalNormalization(5, clip_threshold=5), gpu=0,
        gamma=0.95, lambd=0.9, phi=lambda x: x.astype(np.float32, copy=False),
        update_interval=64, minibatch_size=16, epochs=3, clip_eps=0.2, clip_eps_vf=0.3,
        entropy_coef=0.01, max_grad_norm=0.5, cuda_graph=graph)


def _seeded_trace(make, change, at, kind, steps):
    """Both runs of one case; ``change(agent)`` is applied at step ``at``."""
    runs = []
    for graph in (False, True):
        torch.manual_seed(3)
        agent = make(graph)
        np.random.seed(9)
        torch.manual_seed(9)
        random.seed(9)
        actions, stats = _run_more_trace(
            agent, kind, steps, check=lambda t, a: change(agent) if t == at else None)
        runs.append((agent, actions, stats, _state(agent)))
    return runs


@pytest.mark.parametrize("change", ["lr", "clip_eps"])
def test_ppo_graph_follows_changes(change):
    def apply(agent):
        if change == "lr":
            _set_lr(agent.optimizer)
        else:
            agent.clip_eps *= 0.01

    # 2 envs, 64 steps per update: the first update (12 minibatch rows, the last 9 of them
    # replays) ends at step 31
    (_, _, _, eager), (agent, _, _, graphed) = _seeded_trace(_ppo, apply, 32, "ppo", 200)
    _assert_same(graphed, eager, PPO_TOL)
    assert agent._graph.graph is not None


@pytest.mark.parametrize("change", ["lr", "max_kl"])
def test_trpo_graph_follows_changes(change):
    import pfrl_b200

    kind = TRPO_KINDS[0]

    def make(graph):
        agent = make_trpo_agent(pfrl_b200, kind, gpu=0, cuda_graph=graph)
        for group in agent.vf_optimizer.param_groups:
            group["capturable"] = True
        return agent

    def apply(agent):
        if change == "lr":
            _set_lr(agent.vf_optimizer)
        else:
            agent.max_kl *= 0.01

    # an update every 32 steps; the policy graph is first replayed by the third update
    (_, a0, s0, eager), (agent, a1, s1, graphed) = _seeded_trace(
        make, apply, 96, "sac" if kind == "gauss" else "ppo", 260)
    assert np.array_equal(a0, a1)
    assert np.array_equal(s0, s1, equal_nan=True)
    _assert_same(graphed, eager)
    assert agent._policy_graph.graph is not None and agent._vf_graph.graph is not None
