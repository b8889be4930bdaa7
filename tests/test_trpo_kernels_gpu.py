"""TRPO kernels (csrc/trpo.cu) against fp64 torch of the reference's expressions.

Bounds: the kernels read fp32 inputs exactly, compute in fp64 and round each output
to fp32 once, so an output differs from the fp64 value by at most one fp32 rounding
(2^-24 relative) plus fp64 round-off; the bounds below are 4 fp32 ulps relative plus
an absolute floor for values that cancel (KL near 0).

The categorical reference is evaluated in fp64 except for one decision: whether a
probability is zero.  torch takes that from the fp32 probabilities of the fp32
Categorical the policy returns (the KL's inf where q = 0 and 0 where p = 0, the entropy's
clamped logits), so the restatement does too; e^l is 0 in fp32 below l = -103.97."""
import numpy as np
import pytest
import torch
from torch import distributions as D
from torch import nn

from pfrl_b200.ops import trpo as fused

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RT = 4 * 2.0 ** -24


def ref_objective(kind, params, old, actions, lp_old, adv, stats, c):
    """trpo.py:415-420 and mean KL(old || new) in fp64, with the fp32 standardisation."""
    if stats is not None:
        adv = (adv - stats[0]) / (stats[1] + 1e-8)
    p = [x.double().requires_grad_() for x in params]
    if kind == fused.GAUSSIAN:
        d = D.Independent(D.Normal(p[0], p[1]), 1)
        do = D.Independent(D.Normal(old[0].double(), old[1].double()), 1)
        lp = d.log_prob(actions.double())
    else:
        d = D.Categorical(logits=p[0])
        lp = d.log_prob(actions)
    if kind == fused.GAUSSIAN:
        ent, kl = d.entropy(), D.kl_divergence(do, d)
    else:
        ent, kl = categorical_entropy_kl(p[0], old[0].double(), params[0], old[0])
    gain = torch.mean(torch.exp(lp - lp_old.double()) * adv.double()) + c * torch.mean(ent)
    kl = torch.mean(kl)
    grads = torch.autograd.grad(gain, p)
    return gain.detach(), kl.detach(), ent.mean().detach(), grads


def categorical_entropy_kl(z, zo, z32, zo32):
    """Categorical.entropy and _kl_categorical_categorical(old, new) per row in fp64 (z, zo),
    with p == 0 decided on the fp32 probabilities of the fp32 logits (z32, zo32)."""
    nz = D.Categorical(logits=z32.float()).probs != 0
    nzo = D.Categorical(logits=zo32.float()).probs != 0
    l = z - torch.logsumexp(z, -1, keepdim=True)
    lo = zo - torch.logsumexp(zo, -1, keepdim=True)
    zero = torch.zeros((), dtype=torch.float64)
    l_nz = torch.where(nz, l, zero)  # no -inf * 0 in the gradient of a masked term
    ent = -torch.where(nz, l.exp() * l_nz, zero).sum(-1)
    lo_nz = torch.where(nzo, lo, zero)
    kl = torch.where(nzo, torch.where(nz, lo.exp() * (lo_nz - l_nz), float("inf")), zero)
    return ent, kl.detach().sum(-1)


def plant_underflow(z, zo, actions, rows=None):
    """Rows whose normalised logits are 0 at the action, -80 elsewhere and -120 at one
    other category: -120 only on the new side (torch: q = 0 in fp32, KL inf), only on the
    old side (p = 0 in fp32, the term is 0), and on both.  -80 and -120 lie well inside
    fp32's normal range and well below its smallest subnormal (e^-103.3)."""
    K = z.shape[1]
    rows = range(min(3, z.shape[0])) if rows is None else rows
    for r in rows:
        a = int(actions[r])
        other = (a + 1) % K
        for t in (z, zo):
            t[r] = -80.0
            t[r, a] = 0.0
        if r % 3 in (0, 2):
            z[r, other] = -120.0
        if r % 3 in (1, 2):
            zo[r, other] = -120.0


def make_case(kind, N, A, seed, extreme=False, zero_adv=False, neg_inf=False,
              underflow=False):
    g = torch.Generator().manual_seed(seed)
    if kind == fused.GAUSSIAN:
        loc = torch.randn(N, A, generator=g)
        lsd = torch.randn(N, A, generator=g) * (3.0 if extreme else 0.5)
        params = [loc, torch.exp(lsd)]
        # the old mean moves by a tenth of a standard deviation, so that extreme scales
        # give extreme densities without overflowing the ratio
        old = [loc + 0.1 * params[1] * torch.randn(N, A, generator=g),
               torch.exp(lsd + 0.1 * torch.randn(N, A, generator=g))]
        actions = loc + params[1] * torch.randn(N, A, generator=g)
        lp_old = D.Independent(D.Normal(old[0].double(), old[1].double()), 1).log_prob(
            actions.double()).float()
    else:
        z = torch.randn(N, A, generator=g) * (20.0 if extreme else 1.0)
        zo = z + 0.3 * torch.randn(N, A, generator=g)
        actions = torch.randint(A, (N,), generator=g)
        if neg_inf:
            # p = 0 on the new side only, on the old side only, and on both
            rows = torch.arange(N)
            other = (actions + 1) % A
            z[rows[0::3], other[0::3]] = -float("inf")
            zo[rows[1::3], other[1::3]] = -float("inf")
            z[rows[2::3], other[2::3]] = -float("inf")
            zo[rows[2::3], other[2::3]] = -float("inf")
        if underflow:
            plant_underflow(z, zo, actions, range(0, N, 7))
        params, old = [z], [zo]
        lp_old = D.Categorical(logits=zo.double()).log_prob(actions).float()
    adv = torch.zeros(N) if zero_adv else torch.randn(N, generator=g)
    return params, old, actions, lp_old, adv


def run_case(kind, N, A, seed, stats=True, **kw):
    params, old, actions, lp_old, adv = make_case(kind, N, A, seed, **kw)
    st = torch.stack([adv.mean(), adv.std(unbiased=False)]) if stats else None
    c = 0.01
    want = ref_objective(kind, params, old, actions, lp_old, adv, st, c)
    cu = lambda xs: [x.to(DEV) for x in xs]  # noqa: E731
    pr = [x.to(DEV).requires_grad_() for x in params]
    gain, out = fused.gain(kind, pr, cu(old), actions.to(DEV), lp_old.to(DEV), adv.to(DEV),
                           None if st is None else st.to(DEV), c)
    grads = torch.autograd.grad(gain, pr)
    out = out.double().cpu()
    for got, w, name in ((out[0], want[0], "gain"), (out[1], want[1], "kl"),
                         (out[2], want[2], "entropy")):
        w = float(w)
        if not np.isfinite(w):
            assert float(got) == w or (np.isnan(w) and np.isnan(float(got))), (name, got, w)
        else:
            assert abs(float(got) - w) <= RT * abs(w) + 1e-12, (name, float(got), w)
    for gg, w in zip(grads, want[3]):
        gg = gg.double().cpu()
        # fp64 values beyond the fp32 range (ratios of extreme scales) round to inf
        big = w.abs() > torch.finfo(torch.float32).max
        assert bool((gg[big] == torch.sign(w[big]) * float("inf")).all())
        gg, w = gg[~big], w[~big]
        err = (gg - w).abs()
        assert bool((err <= RT * w.abs() + 1e-12 * max(1.0, float(w.abs().max()))).all()), \
            float(err.max())
    # the forward-only entry point gives the same scalars
    out2 = fused.objective(kind, cu(params), cu(old), actions.to(DEV), lp_old.to(DEV),
                           adv.to(DEV), None if st is None else st.to(DEV), c)
    assert torch.equal(out2.cpu(), out.float())


@pytest.mark.parametrize("N", [1, 255, 256, 257, 5000])
@pytest.mark.parametrize("A", [1, 6, 17])
def test_gaussian_objective_matches_fp64(N, A):
    run_case(fused.GAUSSIAN, N, A, seed=N * 31 + A)


@pytest.mark.parametrize("N", [1, 255, 256, 257, 5000])
@pytest.mark.parametrize("K", [2, 18])
def test_categorical_objective_matches_fp64(N, K):
    run_case(fused.CATEGORICAL, N, K, seed=N * 17 + K)


@pytest.mark.parametrize("kind,A", [(fused.GAUSSIAN, 6), (fused.CATEGORICAL, 18)])
def test_objective_edges(kind, A):
    run_case(kind, 300, A, seed=1, extreme=True)
    run_case(kind, 300, A, seed=2, zero_adv=True, stats=False)
    run_case(kind, 300, A, seed=3, stats=False)


def test_categorical_zero_probabilities():
    """-inf logits: p_old = 0 adds 0 to the KL, p_new = 0 with p_old > 0 makes it inf."""
    run_case(fused.CATEGORICAL, 301, 4, seed=4, neg_inf=True)
    params, old, actions, lp_old, adv = make_case(fused.CATEGORICAL, 9, 4, 5, neg_inf=True)
    # only p_old = 0 entries: KL finite
    z, zo = params[0].clone(), old[0].clone()
    z[torch.isinf(z)] = 0.0
    out = fused.objective(fused.CATEGORICAL, [z.to(DEV)], [zo.to(DEV)], actions.to(DEV),
                          lp_old.to(DEV), adv.to(DEV), None, 0.01)
    assert torch.isfinite(out).all()


@pytest.mark.parametrize("K", [3, 18])
def test_categorical_underflow_is_decided_on_fp32_probabilities(K):
    """A probability that is nonzero in fp64 but 0 in fp32 is 0, as torch decides it: KL
    inf where the new side underflows, no term where the old side does."""
    run_case(fused.CATEGORICAL, 301, K, seed=6, underflow=True)
    params, old, actions, lp_old, adv = make_case(fused.CATEGORICAL, 30, K, 7)
    z, zo = params[0], old[0]
    plant_underflow(z, zo, actions)
    lp_old = D.Categorical(logits=zo.double()).log_prob(actions).float()
    dev = lambda t: t.to(DEV)  # noqa: E731
    out = fused.objective(fused.CATEGORICAL, [dev(z)], [dev(zo)], dev(actions), dev(lp_old),
                          dev(adv), None, 0.01).cpu()
    # the reference's fp32 KL is inf; the fp64 rule alone would give e^-80 * 40 / 30
    assert float(D.kl_divergence(D.Categorical(logits=zo), D.Categorical(logits=z)).mean()) \
        == float("inf")
    assert float(out[1]) == float("inf")
    # without the new-side row: finite, and equal to the fp64 restatement
    keep = list(range(1, 30))
    zk, zok, ak, lpk, advk = (t[keep] for t in (z, zo, actions, lp_old, adv))
    out = fused.objective(fused.CATEGORICAL, [dev(zk)], [dev(zok)], dev(ak), dev(lpk),
                          dev(advk), None, 0.01).cpu().double()
    want = ref_objective(fused.CATEGORICAL, [zk], [zok], ak, lpk, advk, None, 0.01)
    assert np.isfinite(float(want[1]))
    for got, w in zip(out, want[:3]):
        assert abs(float(got) - float(w)) <= RT * abs(float(w)) + 1e-12, (float(got), float(w))


def test_line_search_backtracks_from_a_kl_that_is_inf_in_fp32():
    """Candidate 0 puts probability e^-120 (0 in fp32) where the old policy has e^-80: the
    reference's KL is inf there and it backtracks to candidate 1 (theta_old, KL 0)."""
    K, N = 5, 40
    params, old, actions, _, _ = make_case(fused.CATEGORICAL, N, K, 8)
    z, zo = params[0], old[0]
    plant_underflow(z, zo, actions, rows=[0])
    zo = z.clone()
    zo[0, (int(actions[0]) + 1) % K] = -80.0
    lp_old = D.Categorical(logits=zo.double()).log_prob(actions).float()
    adv = torch.zeros(N)
    dev = lambda t: t.to(DEV)  # noqa: E731
    cand = torch.stack([
        fused.objective(fused.CATEGORICAL, [dev(x)], [dev(zo)], dev(actions), dev(lp_old),
                        dev(adv), None, 0.0) for x in (z, zo)])
    gain0 = fused.objective(fused.CATEGORICAL, [dev(zo)], [dev(zo)], dev(actions), dev(lp_old),
                            dev(adv), None, 0.0)
    ref_kl = [float(D.kl_divergence(D.Categorical(logits=zo), D.Categorical(logits=x)).mean())
              for x in (z, zo)]
    assert ref_kl == [float("inf"), 0.0]
    theta_old = torch.randn(50, device=DEV)
    full = torch.randn(50, device=DEV)
    theta, rec = fused.line_search(cand, gain0, 0.01, theta_old, full)
    assert rec.cpu().tolist() == [0.0, 0.5, 1.0]
    assert torch.equal(theta, theta_old + 0.5 * full)


def _mlp_policy(kind, obs, A):
    from pfrl_b200.policies import (GaussianHeadWithStateIndependentCovariance,
                                    SoftmaxCategoricalHead)

    head = GaussianHeadWithStateIndependentCovariance(A, var_type="diagonal") \
        if kind == fused.GAUSSIAN else SoftmaxCategoricalHead()
    return nn.Sequential(nn.Linear(obs, 64), nn.Tanh(), nn.Linear(64, 64), nn.Tanh(),
                         nn.Linear(64, A), head)


@pytest.mark.parametrize("kind", [fused.GAUSSIAN, fused.CATEGORICAL])
def test_fisher_vector_product_matches_double_backward_hvp(kind):
    """J^T M J v + damping v (fp32 kernels) vs the reference's Hessian of mean
    KL(old || new) by double backward, at theta_old, in fp64.  Bound: fp32 forward and
    backward passes through a 64-64 tanh MLP, 1e-4 relative to |Fv|."""
    import pfrl_b200
    from pfrl_b200.agents.trpo import (_distribution_params, _flatten_and_concat_variables,
                                       _hessian_vector_product)

    torch.manual_seed(0)
    A = 6 if kind == fused.GAUSSIAN else 5
    policy = _mlp_policy(kind, 11, A)
    states = torch.randn(500, 11)
    pol64 = _mlp_policy(kind, 11, A).double()
    pol64.load_state_dict({k: v.double() for k, v in policy.state_dict().items()})
    params64 = list(pol64.parameters())
    d = pol64(states.double())
    with torch.no_grad():
        d_old = pol64(states.double())
    kl = torch.mean(D.kl_divergence(d_old, d))
    flat = _flatten_and_concat_variables(torch.autograd.grad(kl, params64, create_graph=True))

    agent = pfrl_b200.agents.TRPO(policy, nn.Linear(11, 1), None, gpu=0,
                                  conjugate_gradient_damping=0.1)
    s = states.to(DEV)
    kind_got, dparams = _distribution_params(agent.policy(s))
    assert kind_got == kind
    fvp = agent._fisher_vector_product(s, kind, dparams, [x.detach() for x in dparams])
    for seed in range(3):
        v = torch.randn(flat.numel(), generator=torch.Generator().manual_seed(seed))
        want = _hessian_vector_product(flat, params64, v.double()) + 0.1 * v.double()
        got = fvp(v.to(DEV)).double().cpu()
        err = float((got - want).abs().max() / want.abs().max())
        assert err < 1e-4, err


def fp64_cg(A, b, tol, max_iter):
    x = np.zeros_like(b)
    r = b.copy()
    p = r.copy()
    rr = r @ r
    for _ in range(max_iter):
        Ap = A @ p
        alpha = rr / (p @ Ap)
        x = x + alpha * p
        r = r - alpha * Ap
        rr1 = r @ r
        if np.sqrt(rr1) < tol:
            return x
        p = r + (rr1 / rr) * p
        rr = rr1
    return x


@pytest.mark.parametrize("n", [1, 5, 10000])
def test_cg_kernel_matches_fp64_cg(n):
    from pfrl_b200.utils import conjugate_gradient

    rng = np.random.RandomState(n)
    if n <= 5:
        Q = rng.randn(n, n)
        A = Q @ Q.T + n * np.eye(n)
    else:  # SPD, well conditioned and cheap to apply
        Q = rng.randn(n, 50) / np.sqrt(n)
        A = Q @ Q.T + np.diag(1.0 + rng.rand(n))
    A = A.astype(np.float32).astype(np.float64)
    A = (A + A.T) / 2
    b = rng.randn(n).astype(np.float32).astype(np.float64)
    At = torch.tensor(A, dtype=torch.float32, device=DEV)
    iters = min(n, 10)
    x = conjugate_gradient(lambda v: At @ v, torch.tensor(b, dtype=torch.float32, device=DEV),
                           max_iter=iters).double().cpu().numpy()
    want = fp64_cg(A, b, 1e-10, iters)
    np.testing.assert_allclose(x, want, rtol=1e-4, atol=1e-4 * np.abs(want).max())
    # b = 0: 0 / 0 in the first alpha, as in the reference
    x0 = conjugate_gradient(lambda v: At @ v, torch.zeros(n, device=DEV), max_iter=3)
    assert torch.isnan(x0).all()


def test_cg_kernel_stops_at_tol_like_the_reference():
    """A diagonal system with 2 distinct eigenvalues is solved in 2 iterations: the
    residual is then below tol and later iterations leave x as it is."""
    from pfrl_b200.utils import conjugate_gradient

    d = torch.tensor([1.0, 1.0, 3.0, 3.0, 3.0], device=DEV)
    b = torch.tensor([1.0, -2.0, 0.5, 3.0, 1.0], device=DEV)
    calls = []

    def A(v):
        calls.append(1)
        return d * v

    x = conjugate_gradient(A, b, tol=1e-5, max_iter=10)
    assert len(calls) == 10
    np.testing.assert_allclose(x.cpu().numpy(), (b / d).cpu().numpy(), rtol=1e-6)
    x2 = conjugate_gradient(A, b, tol=1e-5, max_iter=2)
    assert torch.equal(x, x2)


def _ls(cand, gain0, max_kl=0.01, n=1000):
    g = torch.Generator().manual_seed(0)
    theta_old = torch.randn(n, generator=g).to(DEV)
    full = torch.randn(n, generator=g).to(DEV)
    theta, rec = fused.line_search(torch.tensor(cand, dtype=torch.float32, device=DEV),
                                   torch.tensor([gain0, 0, 0], dtype=torch.float32, device=DEV),
                                   max_kl, theta_old, full)
    return theta_old, full, theta, rec.cpu().tolist()


def test_line_search_all_rejected_restores_theta_bit_for_bit():
    theta_old, _, theta, rec = _ls([[0.5, 0.02, 0], [-1.0, 0.001, 0], [float("nan"), 0.0, 0]],
                                   0.1)
    assert torch.equal(theta.view(torch.int32), theta_old.view(torch.int32))
    assert rec == [0.0, 0.0, 0.0]


def test_line_search_nan_gain_at_candidate_0():
    theta_old, full, theta, rec = _ls([[float("nan"), 0.001, 0], [0.2, 0.005, 0]], 0.1)
    assert rec[1] == 0.5 and rec[2] == 1.0
    assert rec[0] == np.float32(0.005)
    assert torch.equal(theta, theta_old + 0.5 * full)


def test_line_search_kl_equal_to_max_kl_and_zero_improve_are_accepted():
    max_kl = float(np.float32(0.01))
    theta_old, full, theta, rec = _ls([[0.3, max_kl, 0]], 0.1, max_kl=max_kl)
    assert rec[1] == 1.0 and torch.equal(theta, theta_old + 1.0 * full)
    theta_old, full, theta, rec = _ls([[0.1, 0.02, 0], [0.1, 0.001, 0]], 0.1)
    assert rec[1] == 0.5 and torch.equal(theta, theta_old + 0.5 * full)
    # the KL is compared in double: a KL whose float32 equals float32(max_kl) but which
    # lies above max_kl as a double is rejected
    kl32 = float(np.float32(0.01))               # 0.009999999776...
    max_kl = kl32 - 1e-12
    assert float(np.float32(max_kl)) == kl32
    _, _, _, rec = _ls([[0.3, kl32, 0], [0.3, kl32 / 4, 0]], 0.1, max_kl=max_kl)
    assert rec[1] == 0.5 and rec[0] == np.float32(kl32 / 4)


def test_line_search_non_finite_kl_with_finite_gain_is_rejected():
    for bad in (float("inf"), float("nan")):
        theta_old, full, theta, rec = _ls([[0.5, bad, 0], [0.4, 0.002, 0]], 0.1)
        assert rec == [np.float32(0.002), 0.5, 1.0]
        assert torch.equal(theta, theta_old + 0.5 * full)
