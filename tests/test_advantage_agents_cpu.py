"""AL, PAL, DoublePAL and the DPP agents (DPP, DPPL, DPPGreedy) against the REAL reference on
CPU, in their torch formulation:

* seeded 260-step runs with 3-step prioritised replay on two chain environments
  (tests/golden/agent_trace_<kind>.npz, oracle/gen_golden_advantage.py; construction code
  shared by both sides), checked as tests/test_agent_traces_cpu.py checks the DQN family:
  actions at every step, n_updates / rlen, average_q / average_loss, final parameters and the
  priority trees.  A noisy-net DoublePAL run pins the order of the four network forwards;
* _compute_loss on fixed batches at nA = 4 and 18 (tests/golden/advantage_losses.npz):
  loss, per-sample errors and gradient norm within 1e-5.
"""
import os
import sys
from unittest import mock

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))
from fake_store import OracleBackedStore  # noqa: E402

from oracle.gen_golden_advantage import (ADV_AGENTS, ADV_TRACE_KINDS, LOSS_NA,  # noqa: E402
                                         _make_adv_trace_agent, make_loss_agent)
from oracle.gen_golden_losses import TRACE_PER, _run_trace  # noqa: E402

GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.mark.parametrize("kind", ADV_TRACE_KINDS)
def test_advantage_agent_reproduces_the_reference_run(kind):
    import pfrl_b200
    from pfrl_b200.replay_buffers import PrioritizedReplayBuffer

    g = np.load(os.path.join(GOLD, "agent_trace_%s.npz" % kind))
    with mock.patch("pfrl_b200.replay_buffers.device_buffer.DeviceReplayStore", OracleBackedStore):
        rbuf = PrioritizedReplayBuffer(150, device=0, **TRACE_PER)
        torch.manual_seed(3)
        q, agent = _make_adv_trace_agent(pfrl_b200, kind, rbuf)
        q.load_state_dict({k: torch.tensor(g["init_" + k]) for k in q.state_dict()})
        agent.target_model.load_state_dict(q.state_dict())
        np.random.seed(9)
        torch.manual_seed(9)

        def check(t, a):
            assert a == g["actions"][t].tolist(), "actions diverge at step %d" % t

        actions, stats = _run_trace(agent, rbuf, check=check)
        rbuf._flush()
        info = rbuf.store.info()
    assert np.array_equal(stats[:, 2:], g["stats"][:, 2:])           # n_updates, rlen
    live = stats[:, 2] > 0
    np.testing.assert_allclose(stats[live, 0], g["stats"][live, 0], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(stats[live, 1], g["stats"][live, 1], rtol=1e-5, atol=1e-7)
    for k, v in q.state_dict().items():
        np.testing.assert_allclose(v.numpy(), g["final_" + k], rtol=1e-5, atol=1e-6, err_msg=k)
    np.testing.assert_allclose(info["total"], float(g["total"]), rtol=1e-5)
    np.testing.assert_allclose(info["min"], float(g["min"]), rtol=1e-5)
    np.testing.assert_allclose(info["max_priority"], float(g["max_priority"]), rtol=1e-5)
    assert rbuf.beta == float(g["beta"])


LOSSES = np.load(os.path.join(GOLD, "advantage_losses.npz"))


def check_fixed_batch_losses(kind, nA, device, gradnorm_rtol=1e-5, use_fused_loss=True):
    """_compute_loss on the fixture's batch, with and without weights, against the
    reference's loss, per-sample errors and gradient norm (shared with the GPU test)."""
    import pfrl_b200

    G = LOSSES
    name = "%s_%d" % (kind, nA)
    agent = make_loss_agent(pfrl_b200, kind, nA, gpu=0 if device == "cuda" else None)
    agent.use_fused_loss = use_fused_loss
    for which, mod in (("model", agent.model), ("target", agent.target_model)):
        mod.load_state_dict({k: torch.tensor(G["%s_%s_%s" % (name, which, k)])
                             for k in mod.state_dict()})
    prefix = "batch%d_" % nA
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
        np.testing.assert_allclose(loss.item(), G["%s_w%d_loss" % (name, use_w)], rtol=1e-5,
                                   atol=1e-6)
        np.testing.assert_allclose(delta.cpu().numpy().reshape(-1),
                                   G["%s_w%d_errors" % (name, use_w)], rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(gn, G["%s_w%d_gradnorm" % (name, use_w)],
                                   rtol=gradnorm_rtol)
        out[use_w] = (loss.item(), delta.detach().cpu().numpy().reshape(-1), gn)
    return agent, out


@pytest.mark.parametrize("nA", LOSS_NA)
@pytest.mark.parametrize("kind", list(ADV_AGENTS))
def test_fixed_batch_losses_match_the_reference(kind, nA):
    check_fixed_batch_losses(kind, nA, "cpu")


def test_import_paths_and_defaults():
    import pfrl_b200
    from pfrl_b200.agents import AL, DPP, PAL, DoublePAL, dqn
    from pfrl_b200.agents.al import AL as AL2
    from pfrl_b200.agents.double_pal import DoublePAL as DoublePAL2
    from pfrl_b200.agents.dpp import DPPL, AbstractDPP, DPPGreedy
    from pfrl_b200.agents.pal import PAL as PAL2

    assert (AL, PAL, DoublePAL) == (AL2, PAL2, DoublePAL2)
    assert issubclass(DoublePAL, PAL) and issubclass(AL, dqn.DQN)
    assert all(issubclass(c, AbstractDPP) for c in (DPP, DPPL, DPPGreedy))
    with pytest.raises(TypeError):
        AbstractDPP(None, None, None, 0.9, None)

    def make(cls, **kw):
        q = pfrl_b200.q_functions.FCStateQFunctionWithDiscreteAction(3, 2, 8, 1)
        return cls(q, torch.optim.SGD(q.parameters(), lr=0.1),
                   pfrl_b200.replay_buffers.HostReplayBuffer(10), 0.9,
                   pfrl_b200.explorers.Greedy(), replay_start_size=5, minibatch_size=4, **kw)

    for cls in (AL, PAL, DoublePAL):
        assert make(cls).alpha == 0.9
        assert make(cls, alpha=0.5).alpha == 0.5
    for cls in (DPP, DPPL):
        assert make(cls).eta == 1.0
        assert make(cls, eta=3.0).eta == 3.0
    for cls in (AL, PAL, DoublePAL, DPP, DPPL, DPPGreedy):
        with pytest.raises(NotImplementedError):
            make(cls, recurrent=True)


def test_fused_mode_only_for_the_targets_the_kernel_restates():
    """A subclass that redefines the target (its own L operator, its own _compute_y_and_t)
    runs its torch formulation: the kernel computes only the six built-in targets."""
    from pfrl_b200.agents import AL, DPP, PAL, DoublePAL
    from pfrl_b200.agents._advantage import fused_mode
    from pfrl_b200.agents.dpp import DPPL, AbstractDPP, DPPGreedy

    class Tuned(DPP):  # a hyper-parameter subclass keeps the kernel
        pass

    class MeanDPP(AbstractDPP):
        def _l_operator(self, qout):
            return qout.q_values.mean(dim=1)

    class SharperDPP(DPP):
        def _l_operator(self, qout):
            return qout.compute_expectation(2 * self.eta)

    class MyPAL(PAL):
        def _compute_y_and_t(self, exp_batch):
            return super()._compute_y_and_t(exp_batch)

    modes = {cls: fused_mode(object.__new__(cls)) for cls in (
        AL, PAL, DoublePAL, DPP, DPPL, DPPGreedy, Tuned, MeanDPP, SharperDPP, MyPAL)}
    assert modes == {AL: "al", PAL: "pal", DoublePAL: "double_pal", DPP: "dpp", DPPL: "dppl",
                     DPPGreedy: "dpp_greedy", Tuned: "dpp", MeanDPP: None, SharperDPP: None,
                     MyPAL: None}
