"""The whole A3C agent on cuda:0: the reference's seeded runs (tests/golden/
agent_trace_a3c_*.npz) with host-side sampling noise and the bounds of
tests/test_agent_traces_gpu.py; one kernel launch per update; an update-triggering observe
that never synchronises with the host; and the fused path against the reference formulation
on the same GPU."""
import os
import sys
from unittest import mock

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from oracle.gen_golden_a3c import A3C_KINDS, KINDS, make_a3c_agent, make_env, run  # noqa: E402
from test_a3c_cpu import check_trace  # noqa: E402
from test_agent_traces_gpu import TOL, host_rng  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = os.path.join(HERE, "golden")
DEV = torch.device("cuda:0")


def _count_kernel_calls():
    from pfrl_b200.ops import a3c as fused

    calls = []
    real = fused.loss_grads

    def counted(*args, **kwargs):
        calls.append(1)
        return real(*args, **kwargs)

    return calls, mock.patch.object(fused, "loss_grads", counted)


@pytest.fixture(autouse=True)
def _no_tf32():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


@pytest.mark.parametrize("kind", A3C_KINDS)
def test_a3c_on_cuda_reproduces_the_reference_run(kind):
    import pfrl_b200

    g = np.load(os.path.join(GOLD, "agent_trace_a3c_%s.npz" % kind))
    rtol, atol = TOL["ppo"]
    discrete = KINDS[kind][0]

    def check(t, a):
        if discrete:
            assert np.asarray(a).tolist() == g["actions"][t].tolist(), \
                "actions diverge at step %d" % t
        else:
            np.testing.assert_allclose(a, g["actions"][t], rtol=rtol, atol=atol,
                                       err_msg="actions diverge at step %d" % t)

    calls, patch = _count_kernel_calls()
    with host_rng(), patch:
        agent, got = run(pfrl_b200, kind, device=DEV, check=check, init=g)
    assert agent.device == DEV
    assert len(calls) == int(got["n_updates"])  # the fused path, once per update
    check_trace(g, got, rtol=rtol, atol=atol)


@pytest.mark.parametrize("kind", ["discrete_ff_t5", "discrete_lstm_t5", "gauss_ff_t5",
                                  "gauss_lstm_t1"])
def test_fused_path_equals_the_reference_formulation(kind):
    import pfrl_b200

    out = []
    for use_fused in (False, True):
        def setup(agent):
            agent.use_fused = use_fused

        calls, patch = _count_kernel_calls()
        with host_rng(), patch:
            agent, g = run(pfrl_b200, kind, device=DEV, setup=setup)
        assert len(calls) == (int(g["n_updates"]) if use_fused else 0)
        out.append(g)
    ref, got = out
    if KINDS[kind][0]:
        assert np.array_equal(ref["actions"], got["actions"])
    else:
        np.testing.assert_allclose(got["actions"], ref["actions"], rtol=1e-4, atol=1e-5)
    assert got["params"].shape == ref["params"].shape
    np.testing.assert_allclose(got["params"], ref["params"], rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(got["stats"], ref["stats"], rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize("kind", ["discrete_ff_clip", "discrete_lstm_t5", "gauss_ff_t5",
                                  "gauss_lstm_t1"])
@pytest.mark.parametrize("terminal", [True, False])
def test_updates_do_not_synchronise(kind, terminal):
    """A terminal observe (which makes the update), or an update bootstrapping from a state
    already on the device, under sync debug mode "error"."""
    import pfrl_b200

    torch.manual_seed(0)
    np.random.seed(0)
    agent = make_a3c_agent(pfrl_b200, kind, device=DEV, t_max=10 ** 6)
    env = make_env(pfrl_b200, kind)
    obs = env.reset()
    for _ in range(4):
        obs, r, done, _ = env.step(agent.act(obs))
        if done:
            break
        agent.observe(obs, r, False, False)
    agent.act(obs)
    statevar = agent.batch_states([obs], agent.device, agent.phi)
    before = [p.detach().clone() for p in agent.shared_model.parameters()]
    calls, patch = _count_kernel_calls()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        with patch:
            if terminal:
                agent.observe(obs, 1.0, True, False)
            else:
                agent.t += 1
                agent.past_rewards[agent.t - 1] = 0.5
                agent.update(statevar)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert len(calls) == 1 and agent.t_start == agent.t
    after = list(agent.shared_model.parameters())
    assert any(not torch.equal(x, y) for x, y in zip(before, after))
    for p, q in zip(agent.model.parameters(), agent.shared_model.parameters()):
        assert torch.equal(p, q)


def test_probs_categorical_takes_the_reference_formulation():
    import pfrl_b200
    from torch import nn

    class ProbsHead(nn.Module):
        def forward(self, x):
            return torch.distributions.Categorical(probs=torch.softmax(x, dim=1))

    torch.manual_seed(0)
    model = pfrl_b200.nn.Branched(nn.Sequential(nn.Linear(4, 3), ProbsHead()), nn.Linear(4, 1))
    model.to(DEV)
    agent = pfrl_b200.agents.A3C(model, torch.optim.SGD(model.parameters(), lr=0.1),
                                 t_max=3, gamma=0.9)
    calls, patch = _count_kernel_calls()
    rng = np.random.RandomState(0)
    with patch:
        for t in range(6):
            agent.act(rng.randn(4).astype(np.float32))
            agent.observe(rng.randn(4).astype(np.float32), float(rng.randn()), False, False)
    assert not calls and agent.t_start == 6
    for p, q in zip(agent.model.parameters(), agent.shared_model.parameters()):
        assert torch.equal(p, q)
