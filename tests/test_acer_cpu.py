"""ACER on the CPU: the fp64 closed form of the fused kernel (oracle/acer_closed_form.py)
against the reference formulation's autograd; the device EpisodicReplayBuffer's mu ring
(over the host-logic fake store) against HostEpisodicReplayBuffer; the reference's
seeded runs (tests/golden/agent_trace_acer_*.npz, oracle/gen_golden_acer.py); and
checkpoints exchanged with the reference's ACER."""
import os
import sys
from unittest import mock

import numpy as np
import pytest
import torch
from torch import nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from oracle.acer_closed_form import acer_loss_grads  # noqa: E402
from oracle.gen_golden_acer import ACER_KINDS, make_acer_agent, run  # noqa: E402

GOLD = os.path.join(HERE, "golden")

# (truncation_threshold, use_trust_region, on_policy)
COMBOS = [(c, tr, on) for c in (None, 0, 1, 10, np.inf) for tr in (False, True)
          for on in (False, True)]


def reference_grads(z, q, avg, mu, actions, rewards, R, *, dtype=torch.float64, **cfg):
    """(g_z, g_q, average_kl) by autograd through the reference formulation
    (ACER.compute_loss), with z = each step's Categorical._param."""
    import pfrl_b200
    from pfrl_b200.action_value import DiscreteActionValue

    T = z.shape[0]
    net = nn.Linear(1, 1)
    agent = pfrl_b200.agents.ACER(
        net, torch.optim.SGD(net.parameters(), lr=0.0), t_max=T, gamma=cfg["gamma"],
        replay_buffer=None, beta=cfg["beta"], pi_loss_coef=cfg["pi_loss_coef"],
        Q_loss_coef=cfg["Q_loss_coef"], use_trust_region=cfg["use_trust_region"],
        trust_region_delta=cfg["delta"], truncation_threshold=cfg["truncation_threshold"],
        normalize_loss_by_steps=cfg["normalize_loss_by_steps"], use_Q_opc=cfg["use_Q_opc"],
        average_kl_decay=cfg["average_kl_decay"])
    agent.average_kl = cfg["average_kl"]
    D = torch.distributions
    ds = [D.Categorical(logits=torch.tensor(z[t:t + 1], dtype=dtype, requires_grad=True))
          for t in range(T)]
    qs = [torch.tensor(q[t:t + 1], dtype=dtype, requires_grad=True) for t in range(T)]
    avs = [D.Categorical(logits=torch.tensor(avg[t:t + 1], dtype=dtype)) for t in range(T)]
    mus = None if mu is None else {
        t: D.Categorical(logits=torch.tensor(mu[t:t + 1], dtype=dtype)) for t in range(T)}
    values = {t: (ds[t].probs * qs[t]).sum(1) for t in range(T)}
    # the Q loss's target is torch.tensor(Q_ret), of the default dtype
    previous = torch.get_default_dtype()
    torch.set_default_dtype(dtype)
    try:
        loss = agent.compute_loss(
            t_start=0, t_stop=T, R=R, actions={t: int(actions[t]) for t in range(T)},
            rewards={t: float(rewards[t]) for t in range(T)}, values=values,
            action_values={t: DiscreteActionValue(qs[t]) for t in range(T)},
            action_distribs=dict(enumerate(ds)), action_distribs_mu=mus,
            avg_action_distribs=dict(enumerate(avs)))
    finally:
        torch.set_default_dtype(previous)
    grads = torch.autograd.grad(loss.squeeze(), [d._param for d in ds] + qs)
    g_z = torch.cat(grads[:T]).double().numpy()
    g_q = torch.cat(grads[T:]).double().numpy()
    return g_z, g_q, agent.average_kl


def _case(rng, T, K, degenerate=False):
    z = rng.randn(T, K) * 2
    if degenerate:
        z[0, :2] = [1e10, 1e-10]
        z[-1, :2] = [1e-10, 1e10]
    z = z - np.log(np.exp(z - z.max(1, keepdims=True)).sum(1, keepdims=True)) - \
        z.max(1, keepdims=True)  # the normalised logits Categorical keeps
    q = rng.randn(T, K)
    avg = z + 0.3 * rng.randn(T, K)
    mu = z + 0.5 * rng.randn(T, K)
    return (z.astype(np.float32), q.astype(np.float32), avg.astype(np.float32),
            mu.astype(np.float32), rng.randint(K, size=T), rng.randn(T))


def _cfg(c, tr, **over):
    cfg = dict(gamma=0.9, beta=0.01, pi_loss_coef=1.0, Q_loss_coef=0.5, use_trust_region=tr,
               delta=0.1, truncation_threshold=c, normalize_loss_by_steps=True,
               use_Q_opc=False, average_kl=0.25, average_kl_decay=0.9)
    cfg.update(over)
    return cfg


def _closed(z, q, avg, mu, a, r, R, cfg):
    return acer_loss_grads(z, q, a, r, avg_z=avg, mu_z=mu, bootstrap=R, gamma=cfg["gamma"],
                           truncation_threshold=cfg["truncation_threshold"],
                           use_trust_region=cfg["use_trust_region"], delta=cfg["delta"],
                           beta=cfg["beta"], pi_loss_coef=cfg["pi_loss_coef"],
                           Q_loss_coef=cfg["Q_loss_coef"],
                           normalize_loss_by_steps=cfg["normalize_loss_by_steps"],
                           use_Q_opc=cfg["use_Q_opc"], average_kl=cfg["average_kl"],
                           average_kl_decay=cfg["average_kl_decay"])


@pytest.mark.parametrize("c,tr,on", COMBOS)
@pytest.mark.parametrize("T,K", [(1, 2), (5, 4), (7, 18)])
def test_closed_form_equals_reference_autograd(c, tr, on, T, K):
    rng = np.random.RandomState(T * 100 + K)
    z, q, avg, mu, a, r = _case(rng, T, K)
    for R, over in ((None, {}), (0.7, dict(use_Q_opc=True)),
                    (-0.3, dict(normalize_loss_by_steps=False, delta=1.0))):
        cfg = _cfg(c, tr, **over)
        mu_in = None if on else mu
        want = reference_grads(z, q, avg, mu_in, a, r, 0 if R is None else R, **cfg)
        got = _closed(z, q, avg, mu_in, a, r, R, cfg)
        np.testing.assert_allclose(got[0], want[0], rtol=1e-9, atol=1e-12)
        # the closed form rounds the Q target to fp32 as an fp32 model does; this fp64
        # run does not
        np.testing.assert_allclose(got[1], want[1], rtol=1e-9, atol=1e-6)
        assert got[2] == pytest.approx(want[2], rel=1e-10, abs=1e-14)


@pytest.mark.parametrize("c,tr,on", COMBOS)
def test_closed_form_on_degenerate_rows(c, tr, on):
    """The reference test's degenerate logits [1e10, 1e-10] and flat logits [0, 0], as pi
    and as mu in all four pairings (one per step), action 0 and Q = [1, 3]: fp32 autograd,
    NaN exactly where the reference gives NaN (0 * inf in the full correction, c = 0)."""
    deg, flat = [1e10, 1e-10], [0.0, 0.0]
    pairs = [(deg, deg), (deg, flat), (flat, deg), (flat, flat)]
    z = np.array([p for p, _ in pairs], dtype=np.float32)
    mu = np.array([m for _, m in pairs], dtype=np.float32)
    q = np.tile(np.array([[1.0, 3.0]], dtype=np.float32), (4, 1))
    a = np.zeros(4, dtype=np.int64)
    r = np.array([0.5, -1.0, 0.0, 1.0])
    cfg = _cfg(c, tr)
    mu_in = None if on else mu
    want = reference_grads(z, q, flat + z * 0, mu_in, a, r, 0.5, dtype=torch.float32, **cfg)
    got = _closed(z, q, flat + z * 0, mu_in, a, r, 0.5, cfg)
    for g, w in zip(got[:2], want[:2]):
        assert np.array_equal(np.isnan(g), np.isnan(w))
        np.testing.assert_allclose(np.nan_to_num(g), np.nan_to_num(w), rtol=2e-5, atol=2e-6)
    assert got[2] == pytest.approx(want[2], rel=2e-5, abs=1e-6, nan_ok=True)


# ------------------------------------------------------------------ the mu ring
@pytest.fixture
def fake_store():
    from fake_episodic_store import EpisodicOracleStore

    with mock.patch("pfrl_b200.replay_buffers.device_buffer.DeviceReplayStore",
                    EpisodicOracleStore), \
            mock.patch("torch.cuda.current_device", return_value=0):
        yield


def _mu(kind, rng):
    D = torch.distributions
    if kind == "categorical":
        return D.Categorical(logits=torch.tensor(rng.randn(1, 3), dtype=torch.float32))
    return D.Independent(D.Normal(loc=torch.tensor(rng.randn(1, 2), dtype=torch.float32),
                                  scale=torch.tensor(rng.rand(1, 2) + 0.1,
                                                     dtype=torch.float32)), 1)


def _fill(bufs, rng, kind, n=60):
    for t in range(n):
        term = bool(rng.rand() < 0.15)
        reset = bool(rng.rand() < 0.1)
        kw = dict(state=rng.randn(4).astype(np.float32), action=int(rng.randint(3)),
                  reward=float(rng.randn()), next_state=rng.randn(4).astype(np.float32),
                  is_state_terminal=term, mu=_mu(kind, rng))
        for b in bufs:
            b.append(**kw)
            if term or reset:
                b.stop_current_episode()


def _same_mu(a, b, exact=True):
    """``a`` is ``b`` rebuilt from its parameters as deepcopy_distribution rebuilds it
    (a Categorical normalises its logits again, which may move their last bit)."""
    from pfrl_b200.agents.acer import deepcopy_distribution

    b = deepcopy_distribution(b)
    assert type(a) is type(b)
    same = torch.equal if exact else (lambda x, y: torch.allclose(x, y, rtol=1e-6, atol=1e-6))
    if isinstance(a, torch.distributions.Categorical):
        assert same(a.logits, b.logits)
    else:
        assert same(a.base_dist.loc, b.base_dist.loc)
        assert same(a.base_dist.scale, b.base_dist.scale)
        assert a.reinterpreted_batch_ndims == b.reinterpreted_batch_ndims


@pytest.mark.parametrize("kind", ["categorical", "gaussian"])
@pytest.mark.parametrize("capacity", [None, 25])
def test_device_buffer_keeps_mu_like_the_host_buffer(fake_store, tmp_path, kind, capacity):
    from pfrl_b200.replay_buffers import EpisodicReplayBuffer, HostEpisodicReplayBuffer

    dev, host = EpisodicReplayBuffer(capacity), HostEpisodicReplayBuffer(capacity)
    _fill([dev, host], np.random.RandomState(1), kind)
    assert len(dev) == len(host) and dev.n_episodes == host.n_episodes
    for seed in range(5):
        np.random.seed(seed)
        de = dev.sample_episodes(1, 4)
        np.random.seed(seed)
        he = host.sample_episodes(1, 4)
        for td, th in zip(de[0], he[0]):
            _same_mu(td["mu"], th["mu"])
            assert td["reward"] == th["reward"]
        assert bool(de.last_terminal[0]) == bool(he[0][-1]["is_state_terminal"])
        if kind == "categorical":
            rows = dev.mu_rows(de)
            assert torch.equal(rows, torch.cat([t["mu"].logits for t in he[0]]))
        rew = dev._rewards_f64_device(de)
        assert rew.dtype == torch.float64
        assert rew.tolist() == [t["reward"] for t in he[0]]
    dev.save(str(tmp_path / "buf.pkl"))
    back = EpisodicReplayBuffer(capacity)
    back.load(str(tmp_path / "buf.pkl"))
    for ea, eb in zip(dev._all_episodes(), back._all_episodes()):
        for ta, tb in zip(ea, eb):
            _same_mu(ta["mu"], tb["mu"], exact=False)


def test_buffer_refuses_other_distributions_and_layout_changes(fake_store):
    from pfrl_b200.replay_buffers import EpisodicReplayBuffer

    buf = EpisodicReplayBuffer(100)
    kw = dict(state=np.zeros(2, np.float32), action=0, reward=0.0,
              next_state=np.zeros(2, np.float32))
    with pytest.raises(NotImplementedError, match="Categorical"):
        buf.append(mu=torch.distributions.Normal(torch.zeros(1), torch.ones(1)), **kw)
    buf.append(mu=torch.distributions.Categorical(logits=torch.zeros(1, 3)), **kw)
    with pytest.raises(AssertionError, match="layout"):
        buf.append(mu=torch.distributions.Categorical(logits=torch.zeros(1, 4)), **kw)


def test_buffer_without_mu_is_unchanged(fake_store):
    from pfrl_b200.replay_buffers import EpisodicReplayBuffer

    buf = EpisodicReplayBuffer(100)
    for t in range(5):
        buf.append(state=np.full(2, t, np.float32), action=t, reward=float(t),
                   next_state=np.full(2, t + 1, np.float32), is_state_terminal=t == 4)
    assert buf._mu_ring is None
    ep = buf.sample_episodes(1)
    assert all("mu" not in t for t in ep[0])
    assert bool(ep.last_terminal[0])


# ------------------------------------------------------------ reference runs
def check_trace(g, got, rtol, atol):
    np.testing.assert_allclose(got["stats"], g["stats"], rtol=rtol, atol=atol)
    for k in g.files:
        if k.startswith("final_"):
            np.testing.assert_allclose(got[k], g[k], rtol=rtol, atol=atol, err_msg=k)


@pytest.mark.parametrize("kind", ACER_KINDS)
def test_acer_reproduces_the_reference_run(kind):
    import pfrl_b200

    g = np.load(os.path.join(GOLD, "agent_trace_acer_%s.npz" % kind))
    discrete = g["actions"].dtype.kind in "iu"

    def check(t, a):
        if discrete:
            assert np.asarray(a).tolist() == g["actions"][t].tolist(), \
                "actions diverge at step %d" % t
        else:
            np.testing.assert_allclose(a, g["actions"][t], rtol=1e-5, atol=2e-6,
                                       err_msg="actions diverge at step %d" % t)

    rbuf = pfrl_b200.replay_buffers.HostEpisodicReplayBuffer(10 ** 4)
    agent, got = run(pfrl_b200, kind, rbuf=rbuf, check=check, init=g)
    assert [n for n, _ in agent.get_statistics()] == g["stat_names"].tolist()
    assert len(got["actions"]) == len(g["actions"])
    # the bounds of the PPO / TRPO CPU traces
    check_trace(g, got, rtol=5e-5, atol=2e-6)


def test_checkpoints_interchange_with_the_reference(tmp_path):
    from oracle import refimport

    if not refimport.available():
        pytest.skip("the reference package is not available here")
    pfrl = refimport.import_reference()
    import pfrl_b200

    torch.manual_seed(0)
    ours = make_acer_agent(pfrl_b200, "discrete_ff")
    torch.manual_seed(1)
    ref = make_acer_agent(pfrl, "discrete_ff")
    ours.save(str(tmp_path / "ours"))
    ref.load(str(tmp_path / "ours"))
    for name in ("model", "shared_model"):
        a, b = ours.model.state_dict(), getattr(ref, name).state_dict()
        assert a.keys() == b.keys()
        for k in a:
            assert torch.equal(a[k], b[k]), (name, k)
    ref.save(str(tmp_path / "ref"))
    ours.load(str(tmp_path / "ref"))
    for name in ("model", "shared_model"):
        a, b = getattr(ours, name).state_dict(), ref.model.state_dict()
        for k in a:
            assert torch.equal(a[k], b[k]), (name, k)
    assert ours.optimizer.state_dict()["state"].keys() == \
        ref.optimizer.state_dict()["state"].keys()
    assert ours.optimizer.state_dict()["param_groups"] == \
        ref.optimizer.state_dict()["param_groups"]
