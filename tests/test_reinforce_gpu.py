"""The whole REINFORCE agent on cuda:0: the reference's seeded runs
(tests/golden/agent_trace_reinforce_*.npz) with host-side sampling noise and the bounds of
tests/test_agent_traces_gpu.py; the fused path against the reference formulation on the
same GPU; updates that never synchronise with the host; the kernel's launch count; and
the fast ABC cases of the reference's own test on the device."""
import os
import sys
import tempfile
import warnings
from unittest import mock

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from oracle.gen_golden_reinforce import (KINDS, REINFORCE_KINDS, make_env,  # noqa: E402
                                         make_model, make_reinforce_agent, run)
from test_agent_traces_gpu import TOL, host_rng  # noqa: E402
from test_reinforce_cpu import check_trace  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = os.path.join(HERE, "golden")
DEV = torch.device("cuda:0")


def _count_kernel_calls():
    from pfrl_b200.ops import reinforce as fused

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
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")  # the discarded episodes' warning
        yield


@pytest.mark.parametrize("kind", REINFORCE_KINDS)
def test_reinforce_on_cuda_reproduces_the_reference_run(kind):
    import pfrl_b200

    g = np.load(os.path.join(GOLD, "agent_trace_reinforce_%s.npz" % kind))
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
        agent, got = run(pfrl_b200, kind, gpu=0, check=check, init=g)
    assert agent.device == DEV and agent._fused_record
    # one launch per update, or per episode with backward_separately (the episodes of a
    # batch not yet complete at the end have had theirs)
    if KINDS[kind][3].get("backward_separately"):
        assert len(calls) == agent.batchsize * len(got["params"]) + agent.n_backward
    else:
        assert len(calls) == len(got["params"])
    check_trace(g, got, rtol=rtol, atol=atol)


@pytest.mark.parametrize("kind", ["discrete_ff_b10", "discrete_lstm_b10", "gauss_ff_b10_sep",
                                  "gauss_lstm_b10"])
def test_fused_path_equals_the_reference_formulation(kind):
    """Same seeds, same GPU: the fused and the reference formulation's updates give the
    same parameters and statistics."""
    import pfrl_b200

    out = []
    for use_fused in (False, True):
        def setup(agent):
            agent.use_fused = use_fused

        with host_rng():
            agent, g = run(pfrl_b200, kind, gpu=0, setup=setup)
        assert agent._fused_record == use_fused
        out.append(g)
    ref, got = out
    if KINDS[kind][0]:
        assert np.array_equal(ref["actions"], got["actions"])
    else:
        np.testing.assert_allclose(got["actions"], ref["actions"], rtol=1e-4, atol=1e-5)
    assert got["params"].shape == ref["params"].shape
    np.testing.assert_allclose(got["params"], ref["params"], rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(got["stats"], ref["stats"], rtol=1e-5, atol=1e-7)


def _collect(agent, env, n_episodes):
    """Act until ``n_episodes`` episodes are recorded, without letting the last one's
    terminal trigger the update."""
    obs, done_episodes = env.reset(), 0
    while True:
        obs2, r, done, _ = env.step(agent.act(obs))
        if done and done_episodes + 1 == n_episodes:
            return obs2, r
        agent.observe(obs2, r, done, False)
        if done:
            done_episodes += 1
            obs2 = env.reset()
        obs = obs2


@pytest.mark.parametrize("kind", ["discrete_ff_b10", "discrete_lstm_b10", "gauss_ff_b10_sep",
                                  "gauss_lstm_b10"])
def test_updates_do_not_synchronise(kind):
    import pfrl_b200

    torch.manual_seed(0)
    np.random.seed(0)
    agent = make_reinforce_agent(pfrl_b200, kind, gpu=0, max_grad_norm=1.0)
    separately = agent.backward_separately
    obs2, r = _collect(agent, make_env(pfrl_b200, kind), 1 if separately else agent.batchsize)
    if separately:
        agent.n_backward = agent.batchsize - 1  # this episode completes the batch
    before = [p.detach().clone() for p in agent.model.parameters()]
    calls, patch = _count_kernel_calls()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        with patch:
            agent.observe(obs2, r, True, False)  # the terminal: records and updates
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert len(calls) == 1 and agent.n_backward == 0
    after = list(agent.model.parameters())
    assert any(not torch.equal(x, y) for x, y in zip(before, after))


def test_train_mode_stochastic_layers_take_the_reference_formulation():
    import pfrl_b200
    from torch import nn

    model = nn.Sequential(nn.Linear(5, 20), nn.Dropout(0.1), nn.Linear(20, 2),
                          pfrl_b200.policies.SoftmaxCategoricalHead())
    agent = pfrl_b200.agents.REINFORCE(model, torch.optim.Adam(model.parameters()), gpu=0)
    agent.act(np.zeros(5, np.float32))
    assert not agent._fused_record and len(agent.log_prob_sequences[0]) == 1
    model.eval()
    agent2 = pfrl_b200.agents.REINFORCE(model, torch.optim.Adam(model.parameters()), gpu=0)
    agent2.act(np.zeros(5, np.float32))
    assert agent2._fused_record and len(agent2.obs_sequences[0]) == 1


def test_probs_categorical_takes_the_reference_formulation():
    """A Categorical built from probs keeps the probabilities in _param, which the kernel
    does not differentiate: on CUDA the agent records graphs and updates as the reference."""
    import pfrl_b200
    from torch import nn
    from test_reinforce_cpu import _ProbsHead

    torch.manual_seed(0)
    model = nn.Sequential(nn.Linear(4, 8), nn.Tanh(), nn.Linear(8, 3), _ProbsHead())
    agent = pfrl_b200.agents.REINFORCE(model, torch.optim.SGD(model.parameters(), lr=0.1),
                                       gpu=0, beta=0.1, batchsize=2)
    calls, patch = _count_kernel_calls()
    rng = np.random.RandomState(0)
    with patch:
        for t in range(8):
            agent.act(rng.randn(4).astype(np.float32))
            agent.observe(rng.randn(4).astype(np.float32), float(rng.randn()), t % 4 == 3,
                          False)
    assert not agent._fused_record and not agent._fused_distribution and not calls


@pytest.mark.parametrize("discrete", [True, False])
@pytest.mark.parametrize("use_lstm", [True, False])
@pytest.mark.parametrize("batchsize", [1, 10])
@pytest.mark.parametrize("backward_separately", [True, False])
def test_abc_fast_gpu(discrete, use_lstm, batchsize, backward_separately):
    """The reference test's fast case (tests/agents_tests/test_reinforce.py
    ``test_abc_fast_gpu``): ten training steps and five evaluation episodes on cuda:0."""
    import pfrl_b200
    from pfrl_b200.envs.abc import ABC
    from pfrl_b200.experiments import run_evaluation_episodes, train_agent_with_evaluation

    def env(test):
        return ABC(size=2, discrete=discrete, episodic=True, partially_observable=use_lstm,
                   deterministic=test)

    sample = env(False)
    out = sample.action_space.n if discrete else sample.action_space.low.size
    model = make_model(pfrl_b200, discrete, use_lstm, sample.observation_space.low.size, out)
    agent = pfrl_b200.agents.REINFORCE(
        model, torch.optim.Adam(model.parameters()), gpu=0, beta=1e-2, batchsize=batchsize,
        backward_separately=backward_separately, act_deterministically=True,
        recurrent=use_lstm)
    with tempfile.TemporaryDirectory() as outdir:
        train_agent_with_evaluation(agent=agent, env=env(False), eval_env=env(True),
                                    outdir=outdir, steps=10, train_max_episode_len=2,
                                    eval_interval=500, eval_n_steps=None, eval_n_episodes=5,
                                    successful_score=1)
    assert agent._fused_record
    returns, _ = run_evaluation_episodes(env(True), agent, n_steps=None, n_episodes=5)
    assert len(returns) == 5
