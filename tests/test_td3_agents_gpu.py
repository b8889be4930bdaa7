"""GPU: TD3 and DDPG with the fused critic update (csrc/sac.cu) and ``cuda_graph=True``.

* The seeded reference runs (tests/golden/agent_trace_td3.npz / agent_trace_ddpg.npz) through
  the driver of tests/test_agent_traces_gpu.py, with ``use_fused`` off and on; the fused runs
  really call the kernels.
* ``cuda_graph=True`` against eager on the same seeded updates: bit for bit where the update
  draws no noise (DDPG, TD3 with an identity smoothing), and the same counters with finite
  statistics for TD3's default smoothing, whose graphed noise is drawn differently.
* A change to a value a capture reads re-captures, and the run then matches eager.
* No host synchronisation in an update on the device replay path.  With a host ``phi`` the
  device buffer's gather itself copies the observations to the host to apply it
  (``DeviceNStepBuffer._gather``), so the check uses a device-side phi (``Identity``)."""
import os
import sys

import numpy as np
import pytest
import torch
from torch import nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from oracle.gen_golden_losses import _module_attrs  # noqa: E402
from test_agent_traces_gpu import test_agent_on_cuda_reproduces_the_reference_run as _trace  # noqa: E402

pytestmark = pytest.mark.gpu
OBS, ACT, B = 5, 2, 16


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("kind", ["td3", "ddpg"])
def test_reference_run_on_cuda(kind, fused, monkeypatch):
    from pfrl_b200 import agents
    from pfrl_b200.ops import sac as sac_ops

    monkeypatch.setattr(getattr(agents, kind.upper()), "use_fused", fused)
    calls = {"td3_smooth": 0, "critic_loss": 0}
    for name in calls:
        def spy(*args, _real=getattr(sac_ops, name), _name=name):
            calls[_name] += 1
            return _real(*args)

        monkeypatch.setattr(sac_ops, name, spy)
    _trace(kind)
    if not fused:
        assert calls == {"td3_smooth": 0, "critic_loss": 0}
    else:
        assert calls["critic_loss"] > 200  # one per update
        assert calls["td3_smooth"] == (calls["critic_loss"] if kind == "td3" else 0)


def _qf():
    from pfrl_b200 import nn as pnn

    return nn.Sequential(pnn.ConcatObsAndAction(), nn.Linear(OBS + ACT, 32), nn.ReLU(),
                         nn.Linear(32, 1))


def _make(kind, graph, rbuf=None, phi=lambda x: x, **kw):
    from pfrl_b200 import agents, explorers, policies
    from pfrl_b200.replay_buffers import ReplayBuffer

    torch.manual_seed(0)
    policy = nn.Sequential(nn.Linear(OBS, 32), nn.ReLU(), nn.Linear(32, ACT), nn.Tanh(),
                           policies.DeterministicHead())
    rbuf = rbuf if rbuf is not None else ReplayBuffer(100)
    ex = explorers.AdditiveGaussian(0.1, -1, 1)
    adam = lambda m: torch.optim.Adam(m.parameters(), lr=1e-2, capturable=True)  # noqa: E731
    common = dict(gpu=0, replay_start_size=B, minibatch_size=B, phi=phi, cuda_graph=graph)
    if kind == "td3":
        q1, q2 = _qf(), _qf()
        kw.setdefault("max_grad_norm", 1.0)
        return agents.TD3(policy, q1, q2, adam(policy), adam(q1), adam(q2), rbuf, 0.95, ex,
                          **common, **kw)
    q = _qf()
    return agents.DDPG(policy, q, adam(policy), adam(q), rbuf, 0.95, ex, **common, **kw)


def _experiences(rng, n):
    return [[dict(state=rng.randn(OBS).astype(np.float32),
                  action=rng.uniform(-1, 1, ACT).astype(np.float32), reward=float(rng.randn()),
                  next_state=rng.randn(OBS).astype(np.float32),
                  is_state_terminal=bool(rng.rand() < 0.1), next_action=None)]
            for _ in range(n)]


def _state(agent):
    return {"%s.%s" % (n, k): v.detach().cpu().clone()
            for n, m in _module_attrs(agent) for k, v in m.state_dict().items()}


def _graphs(agent):
    if hasattr(agent, "_q_graph"):
        return (agent._q_graph, agent._full_graph)
    return (agent._graph,)


def _run(kind, graph, updates, change=None, at=None, **kw):
    """``updates`` seeded updates; ``change(agent)`` before update ``at``.  Returns the agent,
    its parameters and the graphs that existed just before the change."""
    rng = np.random.RandomState(1)
    batches = [_experiences(rng, B) for _ in range(updates)]
    agent = _make(kind, graph, **kw)
    torch.manual_seed(7)
    before = None
    for u, batch in enumerate(batches):
        if u == at:
            before = [s.graph for s in _graphs(agent)] if graph else None
            change(agent)
        agent.update(batch)
    return agent, _state(agent), before


def _assert_same(got, want):
    assert got.keys() == want.keys()
    for k in want:
        assert torch.equal(got[k], want[k]), k


@pytest.mark.parametrize("case", ["ddpg", "td3_identity"])
def test_graph_matches_eager_without_update_noise(case):
    kind = "ddpg" if case == "ddpg" else "td3"
    kw = {} if kind == "ddpg" else dict(target_policy_smoothing_func=lambda a: a)
    eager, s_eager, _ = _run(kind, False, 20, **kw)
    graphed, s_graph, _ = _run(kind, True, 20, **kw)
    _assert_same(s_graph, s_eager)
    assert all(s.graph is not None for s in _graphs(graphed))
    assert graphed.get_statistics() == eager.get_statistics()


def test_td3_graph_with_default_smoothing():
    eager, _, _ = _run("td3", False, 20)
    graphed, _, _ = _run("td3", True, 20)
    assert all(s.graph is not None for s in _graphs(graphed))
    assert graphed.policy_n_updates == eager.policy_n_updates == 10
    assert graphed.q_func_n_updates == eager.q_func_n_updates == 20
    for (name, v), (name_e, _) in zip(graphed.get_statistics(), eager.get_statistics()):
        assert name == name_e and np.isfinite(v), name


def _set_lr(agent):
    for opt in (getattr(agent, n) for n in agent.saved_attributes if n.endswith("optimizer")):
        for group in opt.param_groups:
            group["lr"] *= 0.01


CHANGES = {
    ("td3", "lr"): _set_lr,
    ("td3", "soft_update_tau"): lambda a: setattr(a, "soft_update_tau", 0.5),
    ("td3", "max_grad_norm"): lambda a: setattr(a, "max_grad_norm", 0.05),
    ("td3", "policy_update_delay"): lambda a: setattr(a, "policy_update_delay", 3),
    ("ddpg", "lr"): _set_lr,
    ("ddpg", "gamma"): lambda a: setattr(a, "gamma", 0.5),
}


@pytest.mark.parametrize("kind,change", list(CHANGES))
def test_graph_follows_changes(kind, change):
    """Both of TD3's graphs (and DDPG's one) are replayed before update 10; the change
    there drops them, and each is captured again within the next 14 updates."""
    kw = dict(target_policy_smoothing_func=lambda a: a) if kind == "td3" else {}
    _, s_eager, _ = _run(kind, False, 24, CHANGES[kind, change], 10, **kw)
    graphed, s_graph, before = _run(kind, True, 24, CHANGES[kind, change], 10, **kw)
    _assert_same(s_graph, s_eager)
    assert all(g is not None for g in before)
    after = [s.graph for s in _graphs(graphed)]
    assert all(g is not None for g in after)
    assert all(a is not b for a, b in zip(after, before))


@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("kind", ["td3", "ddpg"])
def test_update_on_device_replay_does_not_synchronise(kind, graph):
    from pfrl_b200.replay_buffers import ReplayBuffer
    from pfrl_b200.utils.phi import Identity

    rbuf = ReplayBuffer(1000, device=0)
    agent = _make(kind, graph, rbuf=rbuf, phi=Identity())
    rng = np.random.RandomState(0)
    for t in range(300):
        rbuf.append(state=rng.randn(OBS).astype(np.float32),
                    action=rng.uniform(-1, 1, ACT).astype(np.float32), reward=float(rng.randn()),
                    next_state=rng.randn(OBS).astype(np.float32), next_action=None,
                    is_state_terminal=t % 50 == 49)
    for _ in range(10):  # warm-up, and the captures (a capture synchronises)
        agent.update(rbuf.sample(B))
    before = _state(agent)
    for _ in range(2):  # TD3: a critic-only and a critic + policy update
        exps = rbuf.sample(B)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            agent.update(exps)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert any(not torch.equal(v, before[k]) for k, v in _state(agent).items())
