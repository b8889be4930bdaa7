"""The whole TRPO agent on cuda:0 (fused policy update) against the reference's seeded
runs (tests/golden/agent_trace_trpo_*.npz), with host-side sampling noise and the
bounds of tests/test_agent_traces_gpu.py; and a fused policy update that never
synchronises with the host."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.gen_golden_trpo import TRPO_KINDS, line_search_arrays, make_trpo_agent, run  # noqa: E402
from test_agent_traces_gpu import TOL, host_rng  # noqa: E402
from test_trpo_cpu import check_trace  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.mark.parametrize("kind", TRPO_KINDS)
def test_trpo_on_cuda_reproduces_the_reference_run(kind):
    import pfrl_b200

    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    g = np.load(os.path.join(GOLD, "agent_trace_trpo_%s.npz" % kind))
    rtol, atol = TOL["ppo"]
    discrete = g["actions"].dtype.kind in "iu"

    def check(t, a):
        if discrete:
            assert a.tolist() == g["actions"][t].tolist(), "actions diverge at step %d" % t
        else:
            np.testing.assert_allclose(a, g["actions"][t], rtol=rtol, atol=atol,
                                       err_msg="actions diverge at step %d" % t)

    with host_rng():
        agent, got, updates = run(pfrl_b200, kind, gpu=0, check=check, init=g)
    assert agent._line_search_log is not None  # the fused path ran
    assert len(updates) == g["ls_accepted"].shape[0]
    check_trace(g, got, updates, rtol=rtol, atol=atol)
    cands, _ = line_search_arrays(updates, float(g["max_kl"]))
    want = g["ls_cands"]
    assert np.array_equal(np.isfinite(cands), np.isfinite(want))
    ok = np.isfinite(want)
    # every candidate's improvement and KL stay within a quarter of the fixture's decision
    # margin of the reference's values, so no accept / reject decision can flip
    m_imp, m_kl = g["margin"]
    d_imp = float(np.abs(cands[..., 1] - want[..., 1])[ok[..., 1]].max())
    d_kl = float(np.abs(cands[..., 2] - want[..., 2])[ok[..., 2]].max()) / float(g["max_kl"])
    print("\n[trpo %s on cuda] max |improve diff| %.3g (margin %.3g), max |kl diff| / max_kl "
          "%.3g (margin %.3g)" % (kind, d_imp, m_imp, d_kl, m_kl))
    assert d_imp < m_imp / 4 and d_kl < m_kl / 4


@pytest.mark.parametrize("kind", TRPO_KINDS)
def test_graphed_update_is_bit_equal_to_eager(kind):
    """cuda_graph=True (policy update and value-function steps replayed as graphs) gives
    the same parameters, statistics and actions, bit for bit, as the eager fused path with
    the same (capturable) optimizer."""
    import random

    import pfrl_b200
    from oracle.gen_golden_losses import _module_attrs, _run_more_trace

    results = []
    for graph in (False, True):
        torch.manual_seed(3)
        agent = make_trpo_agent(pfrl_b200, kind, gpu=0, cuda_graph=graph)
        for group in agent.vf_optimizer.param_groups:
            group["capturable"] = True
        np.random.seed(9)
        torch.manual_seed(9)
        random.seed(9)
        actions, stats = _run_more_trace(agent, "sac" if kind == "gauss" else "ppo", 260)
        for step in (agent._policy_graph, agent._vf_graph):
            assert (step is not None and step.graph is not None) == graph
        results.append((actions, stats, {"%s.%s" % (n, k): v.detach().cpu().clone()
                                         for n, m in _module_attrs(agent)
                                         for k, v in m.state_dict().items()}))
    (a0, s0, p0), (a1, s1, p1) = results
    assert np.array_equal(a0, a1)
    assert np.array_equal(s0, s1, equal_nan=True)
    for k in p0:
        assert torch.equal(p0[k], p1[k]), k


@pytest.mark.parametrize("kind", TRPO_KINDS)
def test_fused_policy_update_does_not_synchronise(kind):
    import pfrl_b200

    torch.manual_seed(0)
    agent = make_trpo_agent(pfrl_b200, kind, gpu=0)
    N = 300
    s = torch.randn(N, 5, device="cuda:0")
    with torch.no_grad():
        d = agent.policy(s)
        a = d.sample()
        lp_old = d.log_prob(a).float()
    adv = torch.randn(N, device="cuda:0")
    stats = torch.stack([adv.mean(), adv.std(unbiased=False)])
    before = [p.detach().clone() for p in agent.policy.parameters()]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        assert agent._update_policy_fused(s, a, lp_old, adv, stats)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    after = list(agent.policy.parameters())
    assert any(not torch.equal(x, y) for x, y in zip(before, after)) or \
        agent.policy_step_size_record.mean() == 0.0
