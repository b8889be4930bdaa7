"""TRPO on the CPU (the reference's formulation) against seeded runs of the
reference (tests/golden/agent_trace_trpo_*.npz, oracle/gen_golden_trpo.py),
utils.conjugate_gradient against an fp64 solve, and checkpoints exchanged with
the reference's TRPO."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.gen_golden_trpo import TRPO_KINDS, line_search_arrays, make_trpo_agent, run  # noqa: E402

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def check_trace(g, got, updates, rtol, atol):
    want = g["stats"]
    stats = got["stats"]
    both_nan = np.isnan(stats) & np.isnan(want)
    np.testing.assert_allclose(np.where(both_nan, 0.0, stats), np.where(both_nan, 0.0, want),
                               rtol=rtol, atol=atol)
    for k in g.files:
        if k.startswith("final_"):
            np.testing.assert_allclose(got[k], g[k], rtol=rtol, atol=atol, err_msg=k)
    _, accepted = line_search_arrays(updates, float(g["max_kl"]))
    assert accepted.tolist() == g["ls_accepted"].tolist()


@pytest.mark.parametrize("kind", TRPO_KINDS)
def test_trpo_reproduces_the_reference_run(kind):
    """Actions, statistics at every step, final parameters and every accepted step size."""
    import pfrl_b200

    g = np.load(os.path.join(GOLD, "agent_trace_trpo_%s.npz" % kind))
    discrete = g["actions"].dtype.kind in "iu"

    def check(t, a):
        if discrete:
            assert a.tolist() == g["actions"][t].tolist(), "actions diverge at step %d" % t
        else:
            np.testing.assert_allclose(a, g["actions"][t], rtol=1e-5, atol=2e-6,
                                       err_msg="actions diverge at step %d" % t)

    agent, got, updates = run(pfrl_b200, kind, check=check, init=g)
    assert [n for n, _ in agent.get_statistics()] == g["stat_names"].tolist()
    assert len(updates) == g["ls_accepted"].shape[0]
    # the bounds of the PPO CPU trace (tests/test_agent_traces_cpu.py)
    check_trace(g, got, updates, rtol=5e-5, atol=2e-6)


@pytest.mark.parametrize("n", [1, 5, 60])
def test_conjugate_gradient_agrees_with_an_fp64_solve(n):
    from pfrl_b200.utils import conjugate_gradient

    rng = np.random.RandomState(n)
    Q = rng.randn(n, n)
    A = Q @ Q.T + n * np.eye(n)
    b = rng.randn(n)
    want = np.linalg.solve(A, b)
    At = torch.tensor(A, dtype=torch.float64)
    x = conjugate_gradient(lambda v: At @ v, torch.tensor(b), max_iter=4 * n, tol=1e-12)
    np.testing.assert_allclose(x.numpy(), want, rtol=1e-8, atol=1e-10)
    x32 = conjugate_gradient(lambda v: At.float() @ v, torch.tensor(b, dtype=torch.float32),
                             max_iter=4 * n)
    np.testing.assert_allclose(x32.numpy(), want, rtol=2e-3, atol=2e-4)


def test_recurrent_trpo_is_refused():
    from torch import nn

    import pfrl_b200

    with pytest.raises(NotImplementedError, match="recurrent"):
        pfrl_b200.agents.TRPO(nn.Linear(2, 2), nn.Linear(2, 1), None, recurrent=True)


@pytest.mark.parametrize("head", ["gauss", "softmax"])
def test_fused_path_refuses_policies_that_are_not_fp32(head):
    """The kernels read fp32: the fused update is taken only when every policy parameter
    and every distribution parameter is fp32 on the agent's device."""
    from torch import nn

    import pfrl_b200
    from pfrl_b200.ops import trpo as fused
    from pfrl_b200.policies import (GaussianHeadWithStateIndependentCovariance,
                                    SoftmaxCategoricalHead)

    def agent_for(policy):
        return pfrl_b200.agents.TRPO(policy, nn.Linear(3, 1), None)

    def make(dtype=torch.float32):
        h = GaussianHeadWithStateIndependentCovariance(2, var_type="diagonal") \
            if head == "gauss" else SoftmaxCategoricalHead()
        return nn.Sequential(nn.Linear(3, 2), h).to(dtype)

    want = fused.GAUSSIAN if head == "gauss" else fused.CATEGORICAL
    s = torch.randn(4, 3)
    assert agent_for(make())._fused_kind(s) == want
    for dtype in (torch.float64, torch.float16, torch.bfloat16):
        assert agent_for(make(dtype))._fused_kind(s.to(dtype)) is False, dtype
    # fp32 parameters, fp64 distribution parameters
    cast = nn.Sequential(nn.Linear(3, 2), _Cast(torch.float64), make()[1])
    assert agent_for(cast)._fused_kind(s) is False
    # a policy converted after its first update is checked again
    agent = agent_for(make())
    assert agent._fused_kind(s) == want
    agent.policy.double()
    assert agent._fused_kind(s.double()) is False


class _Cast(torch.nn.Module):
    def __init__(self, dtype):
        super().__init__()
        self.dtype = dtype

    def forward(self, x):
        return x.to(self.dtype)


def test_checkpoints_interchange_with_the_reference(tmp_path):
    from oracle import refimport

    if not refimport.available():
        pytest.skip("the reference package is not available here")
    pfrl = refimport.import_reference()
    import pfrl_b200

    for kind in TRPO_KINDS:
        torch.manual_seed(0)
        ours = make_trpo_agent(pfrl_b200, kind)
        torch.manual_seed(1)
        ref = make_trpo_agent(pfrl, kind)
        ours.obs_normalizer.experience(torch.randn(7, 5))
        ours.save(str(tmp_path / ("ours_" + kind)))
        ref.load(str(tmp_path / ("ours_" + kind)))
        for name in ("policy", "vf", "obs_normalizer"):
            a, b = getattr(ours, name).state_dict(), getattr(ref, name).state_dict()
            assert a.keys() == b.keys()
            for k in a:
                assert torch.equal(a[k], b[k]), (name, k)
        assert ours.vf_optimizer.state_dict()["param_groups"] == \
            ref.vf_optimizer.state_dict()["param_groups"]
        ref.vf(torch.randn(3, 5)).sum().backward()
        ref.vf_optimizer.step()
        ref.save(str(tmp_path / ("ref_" + kind)))
        ours.load(str(tmp_path / ("ref_" + kind)))
        for name in ("policy", "vf", "obs_normalizer"):
            a, b = getattr(ours, name).state_dict(), getattr(ref, name).state_dict()
            for k in a:
                assert torch.equal(a[k], b[k]), (name, k)
        assert ours.vf_optimizer.state_dict()["state"].keys() == \
            ref.vf_optimizer.state_dict()["state"].keys()
