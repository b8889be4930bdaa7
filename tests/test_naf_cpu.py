"""CPU: NAF -- QuadraticActionValue, functions.lower_triangular_matrix and
q_functions.FCQuadraticStateQFunction against the reference's, bit for bit, and the DQN-family
agents' _compute_loss with a NAF Q-function against the reference's on fixed batches.

The six agents' seeded 260-step runs with 3-step prioritised replay and AdditiveOU exploration
on two continuous chain environments are replayed on the device PrioritizedReplayBuffer's host
logic over tests/fake_store.OracleBackedStore: actions at every step, n_updates / rlen,
average_q / average_loss, final parameters and the priority trees.

Fixtures: tests/golden/naf_values.npz, naf_losses.npz and agent_trace_naf_<kind>.npz
(oracle/gen_golden_naf.py, the reference on CPU)."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.gen_golden_losses import TRACE_PER  # noqa: E402
from oracle.gen_golden_naf import (BOUND_KINDS, LOSS_N, NAF_AGENTS, VALUE_N,  # noqa: E402
                                   VALUE_OBS, action_space, action_value_members, bounds,
                                   make_loss_agent, make_trace_agent, run_trace)

GOLD = os.path.join(os.path.dirname(__file__), "golden")
VALUES = np.load(os.path.join(GOLD, "naf_values.npz"))
LOSSES = np.load(os.path.join(GOLD, "naf_losses.npz"))


def _inputs(n):
    prefix = "n%d_" % n
    return {k: VALUES[prefix + k] for k in ("state", "actions", "actions2", "mu", "diag",
                                             "non_diag", "mat_raw", "v")}


def _assert_members(got, name):
    for k, v in got.items():
        np.testing.assert_array_equal(v, VALUES["%s_%s" % (name, k)], err_msg=k)


def load_naf_model(n, scale_mu):
    import pfrl_b200

    q = pfrl_b200.q_functions.FCQuadraticStateQFunction(VALUE_OBS, n, 16, 2, action_space(n),
                                                         scale_mu=bool(scale_mu))
    name = "n%d_s%d" % (n, scale_mu)
    q.load_state_dict({k: torch.tensor(VALUES["%s_param_%s" % (name, k)])
                       for k in q.state_dict()})
    return q, name


@pytest.mark.parametrize("scale_mu", [1, 0])
@pytest.mark.parametrize("n", VALUE_N)
def test_q_function_matches_the_reference(n, scale_mu):
    """The reference's weights load (same keys and shapes) and give the same mu, P, V and
    action-value members, bit for bit."""
    q, name = load_naf_model(n, scale_mu)
    ref_keys = sorted(k[len(name + "_param_"):] for k in VALUES.files
                      if k.startswith(name + "_param_"))
    assert sorted(q.state_dict()) == ref_keys
    for k, v in q.state_dict().items():
        assert tuple(v.shape) == VALUES["%s_param_%s" % (name, k)].shape
    assert ("mat_non_diag.weight" in ref_keys) == (n > 1)
    inp = _inputs(n)
    av = q(torch.tensor(inp["state"]))
    for k, v in zip(("mu", "mat", "v"), av.params):
        np.testing.assert_array_equal(v.detach().numpy(), VALUES["%s_%s" % (name, k)])
    _assert_members(action_value_members(av, inp), name)


def test_q_function_initialisation_and_buffers():
    import pfrl_b200
    from pfrl_b200.q_functions import FCQuadraticStateQFunction

    torch.manual_seed(0)
    q = FCQuadraticStateQFunction(4, 3, 8, 1, action_space(3))
    assert q is not None and pfrl_b200.q_functions.FCQuadraticStateQFunction is type(q)
    # chainer default: zero biases, LeCun-normal weights
    for mod in (q.v, q.mu, q.mat_diag, q.mat_non_diag, q.hidden_layers[0]):
        assert float(mod.bias.detach().abs().max()) == 0.0
    # the scale, mean and bounds are buffers that stay out of the state dict
    names = dict(q.named_buffers())
    assert {"mu_scale", "mu_mean", "min_action", "max_action"} <= set(names)
    assert not any(k in q.state_dict() for k in names)


@pytest.mark.parametrize("which", ["tril", "raw"])
@pytest.mark.parametrize("kind", BOUND_KINDS)
@pytest.mark.parametrize("n", VALUE_N)
def test_action_value_matches_the_reference(n, kind, which):
    """mu planted in and outside the box, bounds absent / scalar / array / lower only, a
    non-symmetric P: every member and a slice."""
    from pfrl_b200.action_value import QuadraticActionValue

    inp = _inputs(n)
    lo, hi = bounds(kind, n)
    mat = (torch.tensor(inp["mat_raw"]) if which == "raw"
           else torch.tensor(inp["diag"]).exp().diag_embed())
    av = QuadraticActionValue(torch.tensor(inp["mu"]), mat, torch.tensor(inp["v"]),
                              min_action=lo, max_action=hi)
    _assert_members(action_value_members(av, inp), "n%d_%s_%s" % (n, kind, which))
    assert repr(av).startswith("QuadraticActionValue greedy_actions:")
    assert len(av.params) == 3


def test_action_value_bounds_are_converted_once():
    from pfrl_b200.action_value import QuadraticActionValue

    lo = torch.tensor([-1.0, -2.0])
    av = QuadraticActionValue(torch.zeros(3, 2), torch.eye(2).expand(3, 2, 2), torch.zeros(3),
                              min_action=lo, max_action=np.array([1.0, 2.0]))
    assert av.min_action is lo  # already fp32 on the device: used as it is
    assert av.max_action.dtype == torch.float32
    assert av[1:].min_action is lo
    av = QuadraticActionValue(torch.zeros(3, 2), torch.eye(2).expand(3, 2, 2), torch.zeros(3),
                              min_action=-1, max_action=[1.0, 1.0])
    assert av.min_action.tolist() == [-1.0]


@pytest.mark.parametrize("n", [n for n in VALUE_N if n > 1])
def test_lower_triangular_matrix(n):
    from pfrl_b200.functions.lower_triangular_matrix import lower_triangular_matrix

    import pfrl_b200

    assert pfrl_b200.functions is not None
    inp = _inputs(n)
    got = lower_triangular_matrix(torch.tensor(inp["diag"]), torch.tensor(inp["non_diag"]))
    np.testing.assert_array_equal(got.numpy(), VALUES["n%d_tril" % n])


def check_fixed_batch_losses(kind, n, device, rtol=1e-5, use_fused_loss=True):
    """_compute_loss on the fixture's batch, with and without weights, against the reference's
    loss, per-sample errors and gradient norm (shared with the GPU test)."""
    import pfrl_b200

    G = LOSSES
    name = "%s_%d" % (kind, n)
    agent = make_loss_agent(pfrl_b200, kind, n, gpu=0 if device == "cuda" else None)
    agent.use_fused_loss = use_fused_loss
    for which, mod in (("model", agent.model), ("target", agent.target_model)):
        mod.load_state_dict({k: torch.tensor(G["%s_%s_%s" % (name, which, k)])
                             for k in mod.state_dict()})
    prefix = "batch%d_" % n
    batch = {k[len(prefix):]: torch.tensor(G[k]).to(device) for k in G.files
             if k.startswith(prefix)}
    out = {}
    for use_w in (1, 0):
        eb = dict(batch)
        if not use_w:
            del eb["weights"]
        agent.model.zero_grad()
        loss, delta = agent._compute_loss(eb, want_errors=True)
        loss.backward()
        gn = torch.sqrt(sum((p.grad ** 2).sum() for p in agent.model.parameters())).item()
        np.testing.assert_allclose(loss.item(), G["%s_w%d_loss" % (name, use_w)], rtol=rtol,
                                   atol=1e-6)
        np.testing.assert_allclose(delta.detach().cpu().numpy().reshape(-1),
                                   G["%s_w%d_errors" % (name, use_w)], rtol=rtol, atol=1e-5)
        np.testing.assert_allclose(gn, G["%s_w%d_gradnorm" % (name, use_w)], rtol=rtol)
        out[use_w] = (loss.item(), delta.detach().cpu().numpy().reshape(-1), gn)
    return agent, out


@pytest.mark.parametrize("n", LOSS_N)
@pytest.mark.parametrize("kind", list(NAF_AGENTS))
def test_fixed_batch_losses_match_the_reference(kind, n):
    check_fixed_batch_losses(kind, n, "cpu")


@pytest.mark.parametrize("cls_name", ["DPP", "DPPL"])
def test_dpp_and_dppl_refuse_a_naf_model_as_the_reference_does(cls_name):
    """DPP's L operator needs compute_expectation, DPPL's q_values: neither exists for a
    continuous action value, so the loss raises AttributeError (never computes another
    target)."""
    import pfrl_b200
    from pfrl_b200.agents import dpp

    cls = getattr(dpp, cls_name)
    qf = pfrl_b200.q_functions.FCQuadraticStateQFunction(4, 2, 8, 1, action_space(2))
    agent = cls(qf, torch.optim.SGD(qf.parameters(), lr=0.0),
                pfrl_b200.replay_buffers.HostReplayBuffer(100), 0.99,
                pfrl_b200.explorers.Greedy(), replay_start_size=10, minibatch_size=4)
    B = 4
    eb = dict(state=torch.randn(B, 4), next_state=torch.randn(B, 4), action=torch.randn(B, 2),
              reward=torch.zeros(B), discount=torch.full((B,), 0.99),
              is_state_terminal=torch.zeros(B))
    with pytest.raises(AttributeError):
        agent._compute_loss(eb)


def test_naf_agent_acts_and_updates_on_the_host():
    """DQN with a NAF Q-function: greedy continuous actions from act(), updates from a replay
    buffer (the reference's torch formulation on CPU)."""
    import pfrl_b200

    torch.manual_seed(0)
    qf = pfrl_b200.q_functions.FCQuadraticStateQFunction(3, 2, 8, 2, action_space(2))
    agent = pfrl_b200.agents.DoubleDQN(
        qf, torch.optim.Adam(qf.parameters(), lr=1e-2),
        pfrl_b200.replay_buffers.HostReplayBuffer(100), 0.9, pfrl_b200.explorers.Greedy(),
        replay_start_size=8, minibatch_size=4, target_update_interval=4)
    rng = np.random.RandomState(0)
    obs = rng.randn(3).astype(np.float32)
    before = [p.detach().clone() for p in qf.parameters()]
    for t in range(20):
        a = agent.act(obs)
        assert a.shape == (2,) and np.all(a >= action_space(2).low - 1e-6)
        obs = rng.randn(3).astype(np.float32)
        agent.observe(obs, float(rng.randn()), t % 7 == 6, False)
    assert agent.optim_t > 0
    assert any(not torch.equal(a, b) for a, b in zip(before, qf.parameters()))
    stats = dict(agent.get_statistics())
    assert np.isfinite(stats["average_q"]) and np.isfinite(stats["average_loss"])


def replay_trace(kind, device=None, rtol=1e-5, atol=1e-6):
    """Replays the reference's seeded run of ``kind`` (on CPU, ``device`` None, over
    tests/fake_store.OracleBackedStore).  Every step is compared up to the first update whose
    sampled indices differ from the reference's, and the whole run when there is none; returns
    that update's number (None) and the worst action deviation."""
    from unittest import mock

    import pfrl_b200
    from pfrl_b200.replay_buffers import PrioritizedReplayBuffer

    sys.path.insert(0, os.path.dirname(__file__))
    from fake_store import OracleBackedStore

    g = np.load(os.path.join(GOLD, "agent_trace_naf_%s.npz" % kind))
    patch = (mock.patch("pfrl_b200.replay_buffers.device_buffer.DeviceReplayStore",
                        OracleBackedStore) if device is None else mock.patch.dict({}))
    with patch:
        rbuf = PrioritizedReplayBuffer(150, device=0, **TRACE_PER)
        torch.manual_seed(3)
        q, agent = make_trace_agent(pfrl_b200, kind, rbuf, gpu=device)
        q.load_state_dict({k: torch.tensor(g["init_" + k]) for k in q.state_dict()})
        agent.target_model.load_state_dict(q.state_dict())
        sampled, sample = [], rbuf.sample

        def recording_sample(n):
            exps = sample(n)
            sampled.append(exps.index.cpu().tolist())
            return exps

        rbuf.sample = recording_sample
        np.random.seed(9)
        torch.manual_seed(9)
        actions, stats = run_trace(agent)
        rbuf._flush()
        info = rbuf.store.info()
    assert np.array_equal(stats[:, 2:], g["stats"][:, 2:])           # n_updates, rlen
    diverged = next((u for u, (a, b) in enumerate(zip(sampled, g["sampled"].tolist()))
                     if a != b), None)
    # steps whose actions and statistics come only from updates on the reference's indices
    upto = len(stats) if diverged is None else int(np.searchsorted(stats[:, 2], diverged + 1))
    np.testing.assert_allclose(actions[:upto], g["actions"][:upto], rtol=rtol, atol=atol)
    live = stats[:upto, 2] > 0
    np.testing.assert_allclose(stats[:upto][live, 0], g["stats"][:upto][live, 0], rtol=rtol,
                               atol=atol)
    np.testing.assert_allclose(stats[:upto][live, 1], g["stats"][:upto][live, 1], rtol=rtol,
                               atol=atol)
    worst = float(np.abs(actions[:upto] - g["actions"][:upto]).max())
    if diverged is not None:
        return diverged, worst
    for k, v in q.state_dict().items():
        np.testing.assert_allclose(v.cpu().numpy(), g["final_" + k], rtol=rtol, atol=atol,
                                   err_msg=k)
    np.testing.assert_allclose(info["total"], float(g["total"]), rtol=rtol)
    np.testing.assert_allclose(info["min"], float(g["min"]), rtol=rtol)
    np.testing.assert_allclose(info["max_priority"], float(g["max_priority"]), rtol=rtol)
    assert rbuf.beta == float(g["beta"])
    return None, worst


@pytest.mark.parametrize("kind", list(NAF_AGENTS))
def test_naf_agent_reproduces_the_reference_run(kind):
    """On CPU the run is the reference's to the end: same sampled indices at every update."""
    diverged, _ = replay_trace(kind)
    assert diverged is None
