"""The whole ACER agent on cuda:0: the reference's seeded runs
(tests/golden/agent_trace_acer_*.npz) with host-side sampling noise and the bounds of
tests/test_agent_traces_gpu.py; the fused path against the reference formulation on the
same GPU; replay and online updates that never synchronise with the host; and seeded
ABC runs that reach the reference test's success criterion."""
import os
import sys
import tempfile
from unittest import mock

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from oracle.gen_golden_acer import ACER_KINDS, KINDS, make_acer_agent, make_model, run  # noqa: E402
from test_acer_cpu import check_trace  # noqa: E402
from test_agent_traces_gpu import TOL, host_rng  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = os.path.join(HERE, "golden")
DEV = torch.device("cuda:0")


def _count_kernel_calls():
    from pfrl_b200.ops import acer as fused

    calls = []
    real = fused.loss_grads

    def counted(*args, **kwargs):
        calls.append(1)
        return real(*args, **kwargs)

    return calls, mock.patch.object(fused, "loss_grads", counted)


@pytest.mark.parametrize("kind", ACER_KINDS)
def test_acer_on_cuda_reproduces_the_reference_run(kind):
    import pfrl_b200

    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    g = np.load(os.path.join(GOLD, "agent_trace_acer_%s.npz" % kind))
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
    rbuf = pfrl_b200.replay_buffers.EpisodicReplayBuffer(10 ** 4, device=0)
    with host_rng(), patch:
        agent, got = run(pfrl_b200, kind, device=DEV, rbuf=rbuf, check=check, init=g)
    assert agent.device == DEV
    assert (len(calls) > 0) == discrete  # the fused path ran for the categorical policies
    check_trace(g, got, rtol=rtol, atol=atol)


@pytest.mark.parametrize("kind", ["discrete_ff", "discrete_lstm", "discrete_ff_plain"])
def test_fused_path_equals_the_reference_formulation(kind):
    """Same seeds, same GPU: the fused and the reference formulation's online and replay
    updates give the same parameters and statistics."""
    import pfrl_b200

    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    out = []
    for use_fused in (False, True):
        def setup(agent):
            agent.use_fused = use_fused

        rbuf = pfrl_b200.replay_buffers.EpisodicReplayBuffer(10 ** 4, device=0)
        with host_rng():
            agent, g = run(pfrl_b200, kind, device=DEV, rbuf=rbuf, steps=60, setup=setup)
        out.append(g)
    ref, got = out
    assert np.array_equal(ref["actions"], got["actions"])
    np.testing.assert_allclose(got["stats"], ref["stats"], rtol=1e-4, atol=1e-6)
    for k in ref:
        if k.startswith("final_"):
            np.testing.assert_allclose(got[k], ref[k], rtol=1e-4, atol=1e-6, err_msg=k)


@pytest.mark.parametrize("kind", ["discrete_ff", "discrete_lstm"])
def test_replay_and_online_updates_do_not_synchronise(kind):
    import pfrl_b200
    from pfrl_b200.envs.abc import ABC
    from pfrl_b200.utils.batch_states import batch_states
    from pfrl_b200.utils.phi import Identity

    torch.manual_seed(0)
    np.random.seed(0)
    rbuf = pfrl_b200.replay_buffers.EpisodicReplayBuffer(10 ** 4, device=0)
    agent = make_acer_agent(pfrl_b200, kind, device=DEV, rbuf=rbuf, phi=Identity(),
                            t_max=10 ** 6, n_times_replay=0, replay_start_size=10)
    env = ABC(size=2, discrete=True, episodic=True, partially_observable=KINDS[kind][1])
    obs = env.reset()
    for _ in range(40):  # commit some episodes; the online history grows
        obs2, r, done, _ = env.step(agent.act(obs))
        agent.observe(obs2, r, done, False)
        obs = env.reset() if done else obs2
    agent.act(obs)
    obs2, r, done, _ = env.step(agent.last_action)
    agent.observe(obs2, r, False, True)  # reset: commits the episode (and updates online)
    for _ in range(3):
        obs2, r, done, _ = env.step(agent.act(obs2))
        agent.observe(obs2, r, False, False)
    statevar = batch_states([obs2], DEV, agent.phi)
    rbuf._flush()
    before = [p.detach().clone() for p in agent.shared_model.parameters()]
    calls, patch = _count_kernel_calls()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        with patch:
            agent.update_on_policy(statevar)  # first, as in observe(): acting kept its graph
            agent.update_from_replay()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert len(calls) == 2
    after = list(agent.shared_model.parameters())
    assert any(not torch.equal(x, y) for x, y in zip(before, after))


@pytest.mark.parametrize("lstm", [False, True])
def test_abc_reaches_the_reference_success_criterion(lstm):
    """The reference test's ABC setting, single-process, on cuda:0: 5 of 5 deterministic
    evaluation episodes return 1.  The same seed succeeds after 500 steps on the CPU;
    the budget is twice that."""
    import random

    import pfrl_b200
    from pfrl_b200.envs.abc import ABC
    from pfrl_b200.experiments import run_evaluation_episodes, train_agent_with_evaluation

    kind = "discrete_lstm" if lstm else "discrete_ff"
    torch.manual_seed(0)
    np.random.seed(0)
    random.seed(0)
    model = make_model(pfrl_b200, kind).to(DEV)
    opt = pfrl_b200.optimizers.SharedRMSpropEpsInsideSqrt(model.parameters(), lr=1e-3,
                                                          eps=1e-8, alpha=0.99)
    agent = pfrl_b200.agents.acer.ACER(
        model, opt, t_max=5 if lstm else 2, gamma=0.5, beta=1e-5,
        replay_buffer=pfrl_b200.replay_buffers.EpisodicReplayBuffer(10 ** 4, device=0),
        n_times_replay=2, act_deterministically=True, replay_start_size=100, recurrent=lstm)

    def make_env(test):
        return ABC(size=2, discrete=True, episodic=True, partially_observable=lstm,
                   deterministic=test)

    # single-process: training stops at the successful evaluation, with its parameters
    with tempfile.TemporaryDirectory() as outdir:
        train_agent_with_evaluation(agent=agent, env=make_env(False), eval_env=make_env(True),
                                    steps=1000, eval_n_steps=None, eval_n_episodes=5,
                                    eval_interval=500, outdir=outdir, successful_score=1)
    returns, _ = run_evaluation_episodes(make_env(True), agent, n_steps=None, n_episodes=5)
    assert np.sum(np.asarray(returns) >= 1) == 5, returns
