"""REINFORCE on the CPU: the fp64 closed form of the fused kernel
(oracle/reinforce_closed_form.py) against the reference formulation's autograd; the
recompute path (through the torch formulation of ops.reinforce) against the reference
formulation; the reference's seeded runs (tests/golden/agent_trace_reinforce_*.npz,
oracle/gen_golden_reinforce.py); and save / load."""
import os
import sys
import warnings
from unittest import mock

import numpy as np
import pytest
import torch
from torch import nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from oracle.gen_golden_reinforce import REINFORCE_KINDS, make_reinforce_agent, run  # noqa: E402
from oracle.reinforce_closed_form import (categorical_grads, gaussian_grads,  # noqa: E402
                                          reference_returns)

GOLD = os.path.join(HERE, "golden")


class _TablePolicy(nn.Module):
    """obs = a row index; the distribution's parameters are that row of a table.  Every
    distribution made while training is kept, with its parameters' gradients retained."""

    def __init__(self, table, discrete, scale=None):
        super().__init__()
        self.table = nn.Parameter(torch.as_tensor(table))
        self.scale = None if scale is None else nn.Parameter(torch.as_tensor(scale))
        self.discrete = discrete
        self.seen = []

    def forward(self, idx):
        rows = self.table[idx.long().reshape(-1)]
        D = torch.distributions
        if self.discrete:
            d = D.Categorical(logits=rows)
            d._param.retain_grad()
        else:
            scale = 1.0 if self.scale is None else self.scale[idx.long().reshape(-1)]
            d = D.Independent(D.Normal(loc=rows, scale=scale), 1)
            d.base_dist.loc.retain_grad()
            if self.scale is not None:
                d.base_dist.scale.retain_grad()
        self.seen.append(d)
        return d


def _episodes(rng, lens, reward_dtype):
    eps = []
    for n in lens:
        r = rng.randn(n)
        rewards = [reward_dtype(x) for x in r]
        eps.append(rewards)
    return eps


def _drive(agent, episodes, discard=()):
    """Act and observe the episodes (row index = observation); the episodes in
    ``discard`` end with a reset and no terminal.  Returns the row index of each step of
    the kept episodes and their reward records."""
    kept_rows, kept_records, row = [], [], 0
    for e, rewards in enumerate(episodes):
        rows = []
        for t, r in enumerate(rewards):
            agent.act(np.array(row, dtype=np.int64))
            last = t == len(rewards) - 1
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                agent.observe(np.array(row + 1, dtype=np.int64), r, last and e not in discard,
                              last and e in discard)
            rows.append(row)
            row += 1
        if e not in discard:
            kept_rows.append(rows)
            kept_records.append(list(rewards) + [rewards[-1]])
    return kept_rows, kept_records


CASES = {
    # name: (episode lengths, discarded episodes, reward dtype)
    "one_step_episodes": ([1, 1, 1], (), float),
    "mixed_lengths": ([3, 1, 5], (), float),
    "fp32_rewards": ([4, 2, 3], (), np.float32),
    "discarded_reset": ([2, 3, 4, 1], (1,), float),
}


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("policy", ["categorical", "gaussian", "gaussian_fixed_scale"])
def test_closed_form_equals_reference_autograd(case, policy):
    """One update through the reference formulation (fp64 policy, SGD with lr 0) against
    the closed form with fp64 coefficients, per row."""
    import pfrl_b200

    discrete, scale_grad = policy == "categorical", policy == "gaussian"
    lens, discard, rdtype = CASES[case]
    rng = np.random.RandomState(len(lens) * 10 + sum(lens))
    n_rows = sum(lens)
    K, A = 5, 3
    if discrete:
        model = _TablePolicy(rng.randn(n_rows + 1, K) * 3, True)
    else:
        model = _TablePolicy(rng.randn(n_rows + 1, A), False,
                             scale=rng.rand(n_rows + 1, A) + 0.2 if scale_grad else None)
    beta, bs = 0.37, len(lens) - len(discard)
    agent = pfrl_b200.agents.REINFORCE(model, torch.optim.SGD(model.parameters(), lr=0.0),
                                       beta=beta, batchsize=bs, batch_states=_idx_batch)
    rows, records = _drive(agent, _episodes(rng, lens, rdtype), discard)
    assert agent.n_backward == 0 and agent._record_is_empty()
    # the distributions made while acting, in step order; drop the discarded episodes'
    kept = [r for ep in rows for r in ep]
    dists = [model.seen[r] for r in kept]
    R = np.concatenate([reference_returns(rec) for rec in records])
    assert R.dtype == (np.float32 if rdtype is np.float32 else np.float64)
    if discrete:
        z = torch.cat([d._param.detach() for d in dists]).numpy()
        acts = np.concatenate([d._sampled for d in dists])
        want, _, _ = categorical_grads(z, acts, R, beta, bs, coef_dtype=np.float64)
        got = torch.cat([d._param.grad for d in dists]).numpy()
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-15)
    else:
        loc = torch.cat([d.base_dist.loc.detach() for d in dists]).numpy()
        scale = torch.cat([d.base_dist.scale.detach() for d in dists]).numpy()
        acts = np.concatenate([d._sampled for d in dists])
        g_loc, g_scale, _, _ = gaussian_grads(loc, scale, acts, R, beta, bs,
                                              coef_dtype=np.float64)
        np.testing.assert_allclose(torch.cat([d.base_dist.loc.grad for d in dists]).numpy(),
                                   g_loc, rtol=1e-12, atol=1e-15)
        if scale_grad:
            np.testing.assert_allclose(
                torch.cat([d.base_dist.scale.grad for d in dists]).numpy(), g_scale,
                rtol=1e-12, atol=1e-15)


def _idx_batch(states, device, phi):
    return torch.as_tensor(np.stack(states)).to(device)


@pytest.fixture(autouse=True)
def _remember_samples(monkeypatch):
    """Keep each distribution's sampled action on the distribution itself."""
    D = torch.distributions
    for cls in (D.Categorical, D.Independent):
        real = cls.sample

        def sample(self, sample_shape=torch.Size(), _real=real):
            x = _real(self, sample_shape)
            self._sampled = x.detach().numpy().copy()
            return x

        monkeypatch.setattr(cls, "sample", sample)


def reference_coefficients(R_seq, beta, batchsize, device="cpu"):
    """d loss / d log_prob and d loss / d entropy of every row, as torch's backward of the
    reference's fp32 loss (``-R * log_prob - beta * entropy`` per step, each a batch-1
    tensor, then ``torch.stack(losses).sum() / batchsize``) yields them."""
    lps = [torch.randn(1, device=device).requires_grad_() for _ in R_seq]
    hs = [torch.rand(1, device=device).requires_grad_() for _ in R_seq]
    losses = [-R * lp - beta * h for R, lp, h in zip(R_seq, lps, hs)]
    (torch.stack(losses).sum() / batchsize).backward()
    return (np.array([float(lp.grad) for lp in lps], np.float32),
            np.array([float(h.grad) for h in hs], np.float32))


@pytest.mark.parametrize("reward_dtype", [float, np.float32])
@pytest.mark.parametrize("beta,batchsize", [(1e-2, 10), (1e-4, 3), (0.37, 7), (0, 1)])
def test_coefficients_are_the_fp32_products_torch_yields(reward_dtype, beta, batchsize):
    """Per row, bit for bit: torch's backward of the fp32 reference loss hands log pi(a)
    fl32(fl32(1 / bs) * fl32(-R)) and H -fl32(fl32(1 / bs) * fl32(beta)), the products the
    kernel and the closed form (coef_dtype float32) form; fp64 products would differ."""
    from oracle.reinforce_closed_form import coefficients

    rng = np.random.RandomState(batchsize)
    R_seq = reference_returns([reward_dtype(x) for x in rng.randn(200) * 7] + [reward_dtype(1)])
    g_lp, g_h = reference_coefficients(R_seq, beta, batchsize)
    c_lp, c_h = coefficients(R_seq, batchsize, beta, np.float32)
    assert np.array_equal(g_lp.view(np.uint32), c_lp.astype(np.float32).view(np.uint32))
    assert np.array_equal(g_h, np.full_like(g_h, c_h)) and np.float32(c_h) == c_h
    if batchsize in (3, 7):  # 1 / bs is inexact: fp64 coefficients are distinguishable
        c64, _ = coefficients(R_seq, batchsize, beta, np.float64)
        assert (c64.astype(np.float32) != g_lp).any()


def test_returns_keep_the_reference_quirks():
    """The doubled terminal reward, the dropped first reward and numpy's dtype."""
    rec = [1.0, 2.0, 4.0, 4.0]  # rewards 1, 2, 4 and the terminal 4 again
    assert reference_returns(rec).tolist() == [10.0, 8.0, 4.0]
    assert reference_returns([np.float32(1), np.float32(1)]).dtype == np.float32
    assert reference_returns([0.5, 0.5]).tolist() == [0.5]


# ------------------------------------------------------------ recompute path
def test_only_logit_categoricals_and_gaussians_are_fused():
    """The kernel differentiates a Categorical's normalised logits: one built from probs
    (whose _param is the probabilities) is not the kernel's case."""
    from pfrl_b200.agents.reinforce import fused_distribution

    D = torch.distributions
    x = torch.randn(3, 4)
    assert fused_distribution(D.Categorical(logits=x))
    assert not fused_distribution(D.Categorical(probs=torch.softmax(x, 1)))
    assert not fused_distribution(D.Categorical(logits=x.double()))
    assert fused_distribution(D.Independent(D.Normal(x, 1.0), 1))
    assert not fused_distribution(D.Normal(x, 1.0))


def test_models_whose_forward_is_not_repeatable_are_not_fused():
    from pfrl_b200.agents.reinforce import recompute_equals_acting
    from pfrl_b200.nn import FactorizedNoisyLinear

    def net(*mid):
        return nn.Sequential(nn.Linear(4, 8), *mid, nn.Linear(8, 2))

    assert recompute_equals_acting(net())
    for layer, train_only in ((nn.Dropout(0.1), True), (nn.BatchNorm1d(8), True),
                              (FactorizedNoisyLinear(nn.Linear(8, 8)), False)):
        m = net(layer)
        assert not recompute_equals_acting(m)
        m.eval()
        # noisy layers draw fresh noise on every forward, in either mode
        assert recompute_equals_acting(m) == train_only


class _ProbsHead(nn.Module):
    def forward(self, x):
        return torch.distributions.Categorical(probs=torch.softmax(x, dim=1))


def test_probs_categorical_takes_the_reference_formulation():
    """A policy whose Categorical is built from probs, with the fused path allowed: the
    agent records graphs and updates as the reference does, bit for bit."""
    import pfrl_b200
    from pfrl_b200.agents.reinforce import REINFORCE

    out = []
    for allow in (False, True):
        torch.manual_seed(0)
        model = nn.Sequential(nn.Linear(4, 8), nn.Tanh(), nn.Linear(8, 3), _ProbsHead())
        agent = pfrl_b200.agents.REINFORCE(model, torch.optim.SGD(model.parameters(), lr=0.1),
                                           beta=0.1, batchsize=2)
        rng = np.random.RandomState(0)
        with mock.patch.object(REINFORCE, "_fused_ok", lambda self, f=allow: f):
            for t in range(8):
                agent.act(rng.randn(4).astype(np.float32))
                agent.observe(rng.randn(4).astype(np.float32), float(rng.randn()),
                              t % 4 == 3, False)
        assert not agent._fused_record and agent._fused_distribution == (not allow)
        out.append([p.detach().clone() for p in model.parameters()])
    for a, b in zip(*out):
        assert torch.equal(a, b)


@pytest.mark.parametrize("kind", REINFORCE_KINDS)
def test_recompute_path_equals_the_reference_formulation(kind):
    """The fused record and update, forced on the CPU through the torch formulation of
    ops.reinforce, against the reference formulation: same seeds, same actions, the same
    parameters after every update up to fp32 summation order."""
    import pfrl_b200
    from pfrl_b200.agents.reinforce import REINFORCE

    out = []
    for fused in (False, True):
        with warnings.catch_warnings(), \
                mock.patch.object(REINFORCE, "_fused_ok", lambda self, f=fused: f):
            warnings.simplefilter("ignore")
            agent, g = run(pfrl_b200, kind, steps=120)
        assert agent._fused_record == fused
        out.append(g)
    ref, got = out
    if ref["actions"].dtype.kind in "iu":
        assert np.array_equal(ref["actions"], got["actions"])
    else:
        np.testing.assert_allclose(got["actions"], ref["actions"], rtol=1e-5, atol=1e-6)
    assert got["params"].shape == ref["params"].shape
    np.testing.assert_allclose(got["params"], ref["params"], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(got["stats"], ref["stats"], rtol=1e-6, atol=1e-9)


# ------------------------------------------------------------ reference runs
def check_trace(g, got, rtol, atol):
    assert got["params"].shape == g["params"].shape
    np.testing.assert_allclose(got["params"], g["params"], rtol=rtol, atol=atol)
    np.testing.assert_allclose(got["stats"], g["stats"], rtol=rtol, atol=atol)


@pytest.mark.parametrize("kind", REINFORCE_KINDS)
def test_reinforce_reproduces_the_reference_run(kind):
    import pfrl_b200

    g = np.load(os.path.join(GOLD, "agent_trace_reinforce_%s.npz" % kind))
    discrete = g["actions"].dtype.kind in "iu"

    def check(t, a):
        if discrete:
            assert np.asarray(a).tolist() == g["actions"][t].tolist(), \
                "actions diverge at step %d" % t
        else:
            np.testing.assert_allclose(a, g["actions"][t], rtol=1e-5, atol=2e-6,
                                       err_msg="actions diverge at step %d" % t)

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        agent, got = run(pfrl_b200, kind, check=check, init=g)
    assert [n for n, _ in agent.get_statistics()] == g["stat_names"].tolist()
    assert len(got["actions"]) == len(g["actions"])
    check_trace(g, got, rtol=5e-5, atol=2e-6)


def test_save_and_load_round_trip(tmp_path):
    import pfrl_b200

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        a, g = run(pfrl_b200, "discrete_ff_b10", steps=60)
    assert len(g["params"]) > 0 and a.optimizer.state_dict()["state"]
    a.save(str(tmp_path / "agent"))
    assert sorted(os.listdir(tmp_path / "agent")) == ["model.pt", "optimizer.pt"]
    torch.manual_seed(1)
    b = make_reinforce_agent(pfrl_b200, "discrete_ff_b10")
    b.load(str(tmp_path / "agent"))
    for (ka, va), (kb, vb) in zip(a.model.state_dict().items(), b.model.state_dict().items()):
        assert ka == kb and torch.equal(va, vb)
    sa, sb = a.optimizer.state_dict(), b.optimizer.state_dict()
    assert sa["param_groups"] == sb["param_groups"]
    for k in sa["state"]:
        for name, v in sa["state"][k].items():
            assert torch.equal(torch.as_tensor(v), torch.as_tensor(sb["state"][k][name]))
