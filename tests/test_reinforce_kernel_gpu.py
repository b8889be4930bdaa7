"""b2rl_reinforce_loss (csrc/reinforce.cu) against the fp64 closed form
(oracle/reinforce_closed_form.py), per element.

Both sides read the same fp32 inputs, form the two per-row coefficients as the same fp32
products, and compute the rest in fp64; the kernel stores fp32.  So an element may differ
by the fp32 rounding of the result (2^-24 relative, bounded here by 2^-23, or 2^-150
absolute for a subnormal result) plus fp64
reassociation and libm differences (exp, log) in the terms that make it up.  For a
Categorical those terms are bounded by |c_lp| [j = a] + |c_H| p_j (1 + |c_j| + |H| +
sum_k p_k |c_k|) for element j (p_j carries the row's entropy error too; an element whose
p_j is 0, a -inf logit, must come out exactly 0); for a Gaussian by
|c_lp| (d^2 / s^3 + 1 / s) + |c_H| / s.  1e-12 of that bound covers the fp64 part.  The per-row loss and entropy are checked in sum against the closed
form's, within fp32 storage of each row's term."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.reinforce_closed_form import (FP32_MIN, categorical_grads,  # noqa: E402
                                          coefficients, gaussian_grads)

pytestmark = pytest.mark.gpu
EPS32 = 2.0 ** -23
TINY32 = 2.0 ** -150  # the fp32 rounding of a result in the subnormal range
DEV = torch.device("cuda:0")


def _close(got, want, terms):
    assert np.array_equal(np.isnan(got), np.isnan(want))
    ok = ~np.isnan(want)
    bound = EPS32 * np.abs(want) + TINY32 + 1e-12 * terms
    err = np.abs(got - want)
    assert (err[ok] <= bound[ok]).all(), float(np.max((err - bound)[ok]))


def _returns(rng, N):
    return (rng.randn(N) * 3).astype(np.float32)


def check_categorical(N, K, seed, extreme=False, beta=0.01, bs=10):
    from pfrl_b200.ops import reinforce as fused

    rng = np.random.RandomState(seed)
    logits = (rng.randn(N, K) * (30 if extreme else 2)).astype(np.float32)
    if extreme:
        logits[0, :2] = [1e10, 1e-10]
        if N > 1:
            logits[-1, :] = 0
            logits[-1, 0] = 1e10
        # a masked action: z = -inf, where torch's entropy clamps to finfo.min and passes
        # no gradient through the clamp
        logits[1:, -1] = -np.inf
    z = torch.distributions.Categorical(logits=torch.tensor(logits)).logits.numpy()
    a = rng.randint(K - 1 if extreme and K > 1 else K, size=N)
    R = _returns(rng, N)
    g_z, loss, ent = fused.loss_grads(
        torch.tensor(R, device=DEV), bs, beta, z=torch.tensor(z, device=DEV),
        actions=torch.tensor(a, device=DEV), want_loss=True)
    want, want_loss, want_ent = categorical_grads(z, a, R, beta, bs)
    c_lp, c_h = coefficients(R, bs, beta)
    zc = np.maximum(z.astype(np.float64), FP32_MIN)
    with np.errstate(over="ignore", under="ignore"):
        p = np.exp(z.astype(np.float64))
    pc = np.sum(p * np.abs(zc), axis=1, keepdims=True)
    terms = abs(c_h) * p * (1 + np.abs(zc) + 2 * pc)
    terms[np.arange(N), a] += np.abs(c_lp)
    got = g_z.double().cpu().numpy()
    _close(got, want, terms)
    if extreme and N > 1:
        assert (got[1:, -1] == 0).all() and np.isfinite(got).all()
    assert float(loss) == pytest.approx(want_loss, rel=1e-5, abs=1e-6 * (1 + abs(want_loss)))
    assert float(ent) == pytest.approx(want_ent, rel=1e-5, abs=1e-6 * N)


def check_gaussian(N, A, seed, tiny_scale=False, scale_kind="learned", beta=0.01, bs=10):
    from pfrl_b200.ops import reinforce as fused

    rng = np.random.RandomState(seed)
    loc = rng.randn(N, A).astype(np.float32)
    if scale_kind == "none":
        scale = None
    else:
        scale = (rng.rand(N, A) + 0.1).astype(np.float32)
        if tiny_scale:
            scale[0] = 1e-4
            scale[-1, 0] = 1e-6
    s = np.ones_like(loc) if scale is None else scale
    act = (loc + s * rng.randn(N, A)).astype(np.float32)
    R = _returns(rng, N)
    scale_grad = scale_kind == "learned"
    g_loc, g_scale, loss, ent = fused.loss_grads(
        torch.tensor(R, device=DEV), bs, beta, loc=torch.tensor(loc, device=DEV),
        scale=None if scale is None else torch.tensor(scale, device=DEV),
        action_values=torch.tensor(act, device=DEV), scale_grad=scale_grad, want_loss=True)
    w_loc, w_scale, w_loss, w_ent = gaussian_grads(loc, scale, act, R, beta, bs)
    c_lp, c_h = coefficients(R, bs, beta)
    d = act.astype(np.float64) - loc
    s64 = s.astype(np.float64)
    terms = np.abs(c_lp)[:, None] * (d * d / s64 ** 3 + 1 / s64) + abs(c_h) / s64
    _close(g_loc.double().cpu().numpy(), w_loc, terms)
    if scale_grad:
        _close(g_scale.double().cpu().numpy(), w_scale, terms)
    else:
        assert g_scale is None
    assert float(loss) == pytest.approx(w_loss, rel=1e-5, abs=1e-6 * (1 + abs(w_loss)))
    assert float(ent) == pytest.approx(w_ent, rel=1e-5, abs=1e-6 * N * A)


@pytest.mark.parametrize("K", [2, 3, 18, 1000])
@pytest.mark.parametrize("N", [1, 7, 1025])
def test_categorical_shapes(N, K):
    check_categorical(N, K, seed=N * 31 + K)


@pytest.mark.parametrize("A", [1, 6, 17])
@pytest.mark.parametrize("N", [1, 7, 1025])
@pytest.mark.parametrize("scale_kind", ["learned", "fixed", "none"])
def test_gaussian_shapes(N, A, scale_kind):
    check_gaussian(N, A, seed=N * 17 + A, scale_kind=scale_kind)


@pytest.mark.parametrize("K", [3, 18])
def test_categorical_many_rows(K):
    check_categorical(100003, K, seed=K)


@pytest.mark.parametrize("A", [1, 6])
def test_gaussian_many_rows(A):
    check_gaussian(100003, A, seed=A)


@pytest.mark.parametrize("K", [2, 3, 18, 1000])
def test_categorical_extreme_logits(K):
    check_categorical(9, K, seed=K, extreme=True)


@pytest.mark.parametrize("A", [1, 6, 17])
def test_gaussian_tiny_scale(A):
    check_gaussian(9, A, seed=A, tiny_scale=True)


@pytest.mark.parametrize("beta,bs", [(0.0, 1), (1e-4, 3), (0.5, 7)])
def test_beta_and_batchsize(beta, bs):
    check_categorical(33, 18, seed=5, beta=beta, bs=bs)
    check_gaussian(33, 6, seed=6, beta=beta, bs=bs)


@pytest.mark.parametrize("reward_dtype", [float, np.float32])
@pytest.mark.parametrize("beta,bs", [(1e-2, 10), (1e-4, 3), (0.37, 7), (0.0, 1)])
def test_kernel_coefficients_are_torch_backward_bit_for_bit(reward_dtype, beta, bs):
    """With loc = 0, action 1 and scale 1, the kernel's d/d loc is c_lp exactly and its
    d/d scale is c_lp (1 - 1) + c_H = c_H exactly: both must equal, bit for bit, what
    torch's backward of the fp32 reference loss hands log_prob and entropy on this GPU."""
    from pfrl_b200.ops import reinforce as fused
    from test_reinforce_cpu import reference_coefficients

    rng = np.random.RandomState(bs)
    R_seq = np.cumsum([reward_dtype(x) for x in rng.randn(300) * 7])[::-1]
    want_lp, want_h = reference_coefficients(R_seq, beta, bs, device=DEV)
    N = len(R_seq)
    g_loc, g_scale = fused.loss_grads(
        torch.tensor(np.ascontiguousarray(R_seq, np.float32), device=DEV), bs, beta,
        loc=torch.zeros(N, 1, device=DEV), scale=None,
        action_values=torch.ones(N, 1, device=DEV))
    assert np.array_equal(g_loc[:, 0].cpu().numpy().view(np.uint32), want_lp.view(np.uint32))
    assert np.array_equal(g_scale[:, 0].cpu().numpy(), want_h)


def test_kernel_gradient_equals_torch_backward_of_the_reference_loss():
    """The fp32 reference loss's autograd on the same rows, on the same GPU: agreement
    within fp32 arithmetic (torch's backward rounds every intermediate to fp32)."""
    from pfrl_b200.ops import reinforce as fused

    rng = np.random.RandomState(0)
    N, K, bs, beta = 40, 6, 4, 0.01
    logits = torch.tensor(rng.randn(N, K).astype(np.float32), device=DEV)
    logits[::3, 0] = -float("inf")  # masked actions: torch gives them a zero gradient
    z = torch.distributions.Categorical(logits=logits).logits.detach().requires_grad_()
    a = torch.tensor(rng.randint(1, K, size=N), device=DEV)
    R = rng.randn(N)
    d = torch.distributions.Categorical(logits=z)
    d._param.retain_grad()
    losses = [-R[i] * d.log_prob(a)[i] - beta * d.entropy()[i] for i in range(N)]
    (torch.stack(losses).sum() / bs).backward()
    (g_z,) = fused.loss_grads(torch.tensor(R, dtype=torch.float32, device=DEV), bs, beta,
                              z=d._param.detach(),
                              actions=a)
    torch.testing.assert_close(g_z, d._param.grad, rtol=1e-5, atol=1e-6)
    assert (d._param.grad[::3, 0] == 0).all() and (g_z[::3, 0] == 0).all()


def test_invalid_arguments_are_refused():
    from pfrl_b200 import _lib

    L = _lib.load()
    assert L.b2rl_reinforce_loss(0, 4, *([None] * 6), 1, 0.0, *([None] * 6)) != 0
