"""A3C on the CPU: the reference's seeded runs (tests/golden/agent_trace_a3c_*.npz,
oracle/gen_golden_a3c.py) replayed exactly; the loss factors; the torch formulation of the
fused kernel (ops.a3c) against the reference's expression and autograd; the public
attributes; save / load; and the eval-mode act."""
import os
import sys
from unittest import mock

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from oracle.gen_golden_a3c import A3C_KINDS, make_a3c_agent, run  # noqa: E402
from oracle.gen_golden_acer import share_memory  # noqa: E402

GOLD = os.path.join(HERE, "golden")


def check_trace(g, got, rtol, atol):
    assert int(got["n_updates"]) == int(g["n_updates"])
    assert got["params"].shape == g["params"].shape
    np.testing.assert_allclose(got["params"], g["params"], rtol=rtol, atol=atol)
    np.testing.assert_allclose(got["stats"], g["stats"], rtol=rtol, atol=atol)


@pytest.mark.parametrize("kind", A3C_KINDS)
def test_a3c_reproduces_the_reference_run(kind):
    import pfrl_b200

    g = np.load(os.path.join(GOLD, "agent_trace_a3c_%s.npz" % kind))

    def check(t, a):
        assert np.array_equal(np.asarray(a), g["actions"][t]), "actions diverge at step %d" % t

    agent, got = run(pfrl_b200, kind, check=check, init=g)
    assert [n for n, _ in agent.get_statistics()] == g["stat_names"].tolist()
    assert len(got["actions"]) == len(g["actions"])
    if agent.max_grad_norm is None:
        check_trace(g, got, rtol=0, atol=0)
    else:
        # the reference clips with a numpy norm on the CPU, utils.clip_l2_grad_norm_ with
        # torch's: the norms differ in the last bits
        check_trace(g, got, rtol=5e-5, atol=2e-6)


def reference_loss(dist, v, actions, rewards, bootstrap, gamma, beta, pf, vf):
    """pfrl/agents/a3c.py:177-204 on given rows: the Python scan, the fp32 returns and the
    loss, with the factors applied as there."""
    import torch.nn.functional as F

    R = 0 if bootstrap is None else float(bootstrap)
    rev = []
    for r in reversed(rewards):
        R *= gamma
        R += r
        rev.append(R)
    ret = torch.as_tensor(list(reversed(rev)), dtype=torch.float, device=v.device)
    adv = ret - v.detach().squeeze(-1)
    pi_loss = torch.sum(-adv * dist.log_prob(actions) - beta * dist.entropy(), dim=0)
    v_loss = F.mse_loss(v, ret[..., None], reduction="sum") / 2
    if pf != 1.0:
        pi_loss *= pf
    if vf != 1.0:
        v_loss *= vf
    return ret, torch.squeeze(pi_loss) + torch.squeeze(v_loss)


def make_rows(rng, N, D, discrete, device="cpu", scale=True):
    D_ = torch.distributions
    v = torch.tensor(rng.randn(N, 1) * 2, dtype=torch.float32, device=device,
                     requires_grad=True)
    if discrete:
        z = torch.tensor(rng.randn(N, D) * 3, dtype=torch.float32, device=device,
                         requires_grad=True)
        dist = D_.Categorical(logits=z)
        dist._param.retain_grad()
        actions = torch.as_tensor(rng.randint(0, D, N), device=device)
        return dist, [dist._param], v, actions
    loc = torch.tensor(rng.randn(N, D), dtype=torch.float32, device=device, requires_grad=True)
    leaves = [loc]
    if scale:
        s = torch.tensor(rng.rand(N, D) + 0.3, dtype=torch.float32, device=device,
                         requires_grad=True)
        leaves.append(s)
        dist = D_.Independent(D_.Normal(loc, s), 1)
    else:
        dist = D_.Independent(D_.Normal(loc, 1.0), 1)
    actions = torch.tensor(rng.randn(N, D), dtype=torch.float32, device=device)
    return dist, leaves, v, actions


def fused_call(dist, v, actions, rewards, bootstrap, gamma, beta, pf, vf, **kw):
    from pfrl_b200.ops import a3c as fused

    dev = v.device
    r = torch.as_tensor(np.asarray(rewards, np.float64), device=dev)
    boot = None if bootstrap is None else torch.tensor([bootstrap], dtype=torch.float32,
                                                       device=dev)
    if type(dist) is torch.distributions.Categorical:
        return fused.loss_grads(v, r, boot, gamma, beta, pf, vf, z=dist._param,
                                actions=actions, **kw)
    base = dist.base_dist
    return fused.loss_grads(v, r, boot, gamma, beta, pf, vf, loc=base.loc, scale=base.scale,
                            action_values=actions, **kw)


@pytest.mark.parametrize("discrete", [True, False])
@pytest.mark.parametrize("bootstrap", [None, 0.7310586])
@pytest.mark.parametrize("gamma", [0.0, 0.99, 1.0])
def test_torch_formulation_equals_the_reference(discrete, bootstrap, gamma):
    """Returns bit for bit; g_v bit for bit (its fp32 chain is the reference's); the
    policy's gradients within fp32 rounding of the reference's autograd."""
    rng = np.random.RandomState(int(gamma * 100) + (bootstrap is None))
    N, D = 7, 5
    rewards = list(rng.randn(N) * 3)
    dist, leaves, v, actions = make_rows(rng, N, D, discrete)
    pf, vf = 5 / 3, 0.5 * 5 / 3
    ret, loss = reference_loss(dist, v, actions, rewards, bootstrap, gamma, 0.37, pf, vf)
    loss.backward()
    grads, g_v, R, pi_loss, v_loss = fused_call(dist, v, actions, rewards, bootstrap, gamma,
                                                0.37, pf, vf, want_loss=True)
    assert np.array_equal(R.numpy().view(np.uint32), ret.numpy().view(np.uint32))
    assert np.array_equal(g_v.numpy(), v.grad.reshape(-1).numpy())
    for leaf, g in zip(leaves, grads):
        np.testing.assert_allclose(g.numpy(), leaf.grad.numpy(), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(float(pi_loss + v_loss), float(loss), rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("keep,norm,n,t_max", [(False, False, 3, 5), (True, False, 3, 5),
                                               (True, False, 5, 5), (False, True, 3, 5),
                                               (True, True, 2, 7)])
def test_loss_factors_match_the_reference(keep, norm, n, t_max):
    """The factors of pfrl/agents/a3c.py:149-160, in its operation order (the traces with
    keep_loss_scale_same and normalize_grad_by_t_max check them through whole runs)."""
    import pfrl_b200

    model = pfrl_b200.nn.Branched(
        torch.nn.Sequential(torch.nn.Linear(2, 2), pfrl_b200.policies.SoftmaxCategoricalHead()),
        torch.nn.Linear(2, 1))
    a = pfrl_b200.agents.A3C(model, torch.optim.SGD(model.parameters(), lr=0), t_max=t_max,
                             gamma=0.9, pi_loss_coef=1.3, v_loss_coef=0.7,
                             keep_loss_scale_same=keep, normalize_grad_by_t_max=norm)
    a.t, a.t_start = 10 + n, 10
    pi, v = 1.3, 0.7
    if keep and n < t_max:
        pi *= t_max / n
        v *= t_max / n
    if norm:
        pi /= n
        v /= n
    assert a._loss_factors() == (pi, v)


def test_public_attributes_match_the_reference():
    from oracle.refimport import import_reference

    pfrl = import_reference()
    import pfrl_b200

    for name in ("process_idx", "saved_attributes"):
        assert getattr(pfrl_b200.agents.A3C, name) == getattr(pfrl.agents.A3C, name)
    agents = [make_a3c_agent(lib, "discrete_ff_t5") for lib in (pfrl, pfrl_b200)]
    for a in agents:
        share_memory(a)
        a.assert_shared_memory()
    assert agents[0].shared_attributes == agents[1].shared_attributes
    assert [n for n, _ in agents[0].get_statistics()] == \
        [n for n, _ in agents[1].get_statistics()]
    assert agents[1].process_idx is None


def test_assert_shared_memory_refuses_an_unshared_model():
    import pfrl_b200

    agent = make_a3c_agent(pfrl_b200, "discrete_ff_t5")
    with pytest.raises(AssertionError):
        agent.assert_shared_memory()


def test_save_then_load_gives_shared_model_equal_to_model(tmp_path):
    import pfrl_b200

    a, g = run(pfrl_b200, "discrete_ff_t5", steps=40)
    assert len(g["params"]) > 0
    a.save(str(tmp_path / "agent"))
    assert sorted(os.listdir(tmp_path / "agent")) == ["model.pt", "optimizer.pt"]
    torch.manual_seed(1)
    b = make_a3c_agent(pfrl_b200, "discrete_ff_t5")
    b.load(str(tmp_path / "agent"))
    for (ka, va), (kb, vb), (ks, vs) in zip(a.model.state_dict().items(),
                                            b.model.state_dict().items(),
                                            b.shared_model.state_dict().items()):
        assert ka == kb == ks and torch.equal(va, vb) and torch.equal(vb, vs)


@pytest.mark.parametrize("kind", ["discrete_ff_t5", "gauss_lstm_t1"])
def test_eval_act_is_deterministic(kind):
    """With act_deterministically, the eval-mode act of an episode is a function of its
    observations: the same episode twice gives the same actions."""
    import pfrl_b200
    from oracle.gen_golden_a3c import make_env

    agent = make_a3c_agent(pfrl_b200, kind)
    env = make_env(pfrl_b200, kind, test=True)
    episode = [env.reset()] + [env.step(env.action_space.sample())[0] for _ in range(3)]
    out = []
    for _ in range(2):
        with agent.eval_mode():
            acts = []
            for obs in episode:
                acts.append(np.asarray(agent.act(obs)))
                agent.observe(obs, 0.0, False, False)
            agent.observe(obs, 0.0, False, True)
        out.append(acts)
    for x, y in zip(*out):
        assert np.array_equal(x, y)


def test_forced_fused_path_on_the_cpu_equals_the_reference_formulation():
    """The fused record and update, forced on the CPU through the torch formulation of
    ops.a3c, against the reference formulation: same actions, and the parameters after
    every update up to fp32 summation order."""
    import pfrl_b200
    from pfrl_b200.agents.a3c import A3C

    out = []
    for forced in (False, True):
        with mock.patch.object(A3C, "_fused_ok", lambda self, f=forced: f):
            agent, g = run(pfrl_b200, "discrete_ff_t5", steps=80)
        out.append(g)
    ref, got = out
    assert np.array_equal(ref["actions"], got["actions"])
    np.testing.assert_allclose(got["params"], ref["params"], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(got["stats"], ref["stats"], rtol=1e-6, atol=1e-9)
