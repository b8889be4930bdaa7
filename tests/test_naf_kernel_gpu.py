"""GPU: the NAF kernels (csrc/naf.cu) per element against fp64.

* head: P = L L^T and its backward, against fp64 autograd of the reference's expression
  (exp, lower_triangular_matrix, matmul; mat_diag**2 when n = 1);
* loss: y, t, |y - t| and the loss of every mode, against the reference's QuadraticActionValue
  arithmetic in fp64; the gradients of mu, P and V against fp64 autograd of evaluate_actions.

Each bound is derived per element: (n + c) units of fp32 rounding times the sum of the
magnitudes of the terms that make the element."""
import numpy as np
import pytest
import torch

from pfrl_b200.action_value import QuadraticActionValue
from pfrl_b200.functions.lower_triangular_matrix import lower_triangular_matrix
from pfrl_b200.ops import naf

pytestmark = pytest.mark.gpu

U = 2.0 ** -23
SIZES_B = (1, 255, 256, 257, 5000)
SIZES_N = (1, 2, 3, 17, 33, 65)


def _cases():
    for B in SIZES_B:
        for n in SIZES_N:
            if B * n * n <= 5000 * 33 * 33:
                yield B, n


def _head64(dp, nd):
    d = torch.exp(dp)
    if nd is None:
        return torch.unsqueeze(d ** 2, 2), d[:, :, None]
    L = torch.zeros(dp.shape[0], dp.shape[1], dp.shape[1], dtype=dp.dtype, device=dp.device)
    rows, cols = torch.tril_indices(dp.shape[1], dp.shape[1], -1, device=dp.device)
    L[:, rows, cols] = nd
    idx = torch.arange(dp.shape[1], device=dp.device)
    L[:, idx, idx] = d
    return L @ L.transpose(1, 2), L


@pytest.mark.parametrize("B,n", list(_cases()))
def test_head_forward_and_backward_against_fp64(B, n):
    g = torch.Generator(device="cuda").manual_seed(B * 100 + n)
    m = n * (n - 1) // 2
    dp = torch.randn(B, n, device="cuda", generator=g) * 0.5
    nd = torch.randn(B, m, device="cuda", generator=g) if n > 1 else None
    dp.requires_grad_()
    if nd is not None:
        nd.requires_grad_()
    mat = naf.head(dp, nd)
    dp64 = dp.detach().double().requires_grad_()
    nd64 = None if nd is None else nd.detach().double().requires_grad_()
    mat64, L64 = _head64(dp64, nd64)
    La = L64.detach().abs()
    tol = (n + 8) * U * (La @ La.transpose(1, 2)) + 1e-30
    assert bool(((mat.detach().double() - mat64.detach()).abs() <= tol).all())
    G = torch.randn(B, n, n, device="cuda", generator=g)  # not symmetric
    mat.backward(G)
    mat64.backward(G.double())
    Gs = G.double().abs() + G.double().abs().transpose(1, 2)
    gl_tol = (n + 8) * U * (Gs @ La)  # |grad_L| majorant
    d_tol = torch.diagonal(gl_tol, dim1=1, dim2=2) * torch.exp(dp64.detach()) * 2
    assert bool(((dp.grad.double() - dp64.grad).abs() <= d_tol + 1e-30).all())
    if nd is not None:
        rows, cols = torch.tril_indices(n, n, -1, device="cuda")
        assert bool(((nd.grad.double() - nd64.grad).abs() <= gl_tol[:, rows, cols] + 1e-30).all())


def test_head_n1_equals_the_reference_square():
    dp = torch.randn(300, 1, device="cuda")
    got = naf.head(dp, None)
    assert torch.equal(got, torch.unsqueeze(torch.exp(dp) ** 2, 2))


def test_head_overflow_places_inf_and_nan_where_the_reference_does():
    n = 4
    dp = torch.randn(8, n, device="cuda")
    dp[1, 2] = 100.0  # exp overflows
    dp[5, 0] = 200.0
    nd = torch.randn(8, n * (n - 1) // 2, device="cuda")
    nd[3, 0] = 0.0
    got = naf.head(dp, nd)
    tril = lower_triangular_matrix(torch.exp(dp), nd)
    want = torch.matmul(tril, tril.transpose(1, 2))
    assert torch.equal(torch.isnan(got), torch.isnan(want))
    assert torch.equal(torch.isinf(got), torch.isinf(want))
    fin = torch.isfinite(want)
    assert torch.allclose(got[fin], want[fin], rtol=1e-5, atol=1e-6)


# ----------------------------------------------------------------------------- loss
def _qav(mu, mat, v, lo, hi):
    return QuadraticActionValue(mu, mat, v, min_action=lo, max_action=hi)


def _abs_q(av, actions):
    """Majorant of |evaluate_actions|: |v| + 1/2 |d|^T |P| |d|."""
    d = (actions - av.mu).abs()
    return av.v.reshape(-1).abs() + 0.5 * (d[:, None, :] @ av.mat.abs() @ d[:, :, None])[:, 0, 0]


def _abs_max(av):
    if av.min_action is None and av.max_action is None:
        return av.v.reshape(-1).abs()
    return _abs_q(av, av.greedy_actions)


def target64(mode, batch, q, tq, tnq, nq, alpha):
    """t and a majorant of the magnitudes that make it, in fp64 (the reference's targets)."""
    r, disc, term = batch["reward"], batch["discount"], batch["is_state_terminal"]
    a = batch["action"]
    c = disc * (1.0 - term)
    if mode in ("double_dqn", "double_pal"):
        g = nq.greedy_actions
        next_v, next_m = tnq.evaluate_actions(g), _abs_q(tnq, g)
    else:
        next_v, next_m = tnq.max, _abs_max(tnq)
    bell, bell_m = r + c * next_v, r.abs() + c.abs() * next_m
    if mode in ("dqn", "double_dqn"):
        return bell, bell_m
    tq_a, tq_a_m = tq.evaluate_actions(a), _abs_q(tq, a)
    tq_max, tq_max_m = tq.max, _abs_max(tq)
    if mode == "dpp_greedy":
        return tq_a + bell - tq_max, tq_a_m + bell_m + tq_max_m
    adv, adv_m = tq_a - tq_max, tq_a_m + tq_max_m
    if mode != "al":
        adv2 = tnq.evaluate_actions(a) - tnq.max
        adv = torch.max(adv, adv2)
        adv_m = adv_m + _abs_q(tnq, a) + _abs_max(tnq)
    return bell + alpha * adv, bell_m + abs(alpha) * adv_m


def make_problem(B, n, seed, bounds="array", scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)

    def r(*s):
        return torch.randn(*s, device="cuda", generator=g)

    def net():
        L = torch.tril(r(B, n, n) * 0.3 * scale)
        return r(B, n) * 1.5, L @ L.transpose(1, 2) + 0.1 * torch.eye(n, device="cuda"), r(B, 1)

    lo = hi = None
    if bounds == "array":
        lo, hi = -torch.rand(n, device="cuda", generator=g) - 0.1, torch.rand(n, device="cuda",
                                                                             generator=g) + 0.1
    elif bounds == "scalar":
        lo, hi = torch.tensor([-0.5], device="cuda"), torch.tensor([0.75], device="cuda")
    batch = dict(action=r(B, n) * 1.5, reward=r(B), discount=torch.full((B,), 0.97, device="cuda"),
                 is_state_terminal=(torch.rand(B, device="cuda", generator=g) < 0.2).float(),
                 weights=torch.rand(B, device="cuda", generator=g))
    batch["weights"][::7] = 0.0  # zero weights
    return [net() for _ in range(4)], lo, hi, batch


LOSS_CASES = [(B, n) for B in SIZES_B for n in SIZES_N if B <= 257 or n <= 3]


@pytest.mark.parametrize("mode", list(naf.NAF_MODES))
@pytest.mark.parametrize("B,n", LOSS_CASES)
def test_loss_forward_and_backward_against_fp64(mode, B, n):
    nets, lo, hi, batch = make_problem(B, n, seed=B * 7 + n + len(mode))
    _loss_case(mode, nets, lo, hi, batch, clip_delta=(B + n) % 2 == 0, mean=B % 2 == 1,
               use_w=n != 2)


@pytest.mark.parametrize("mode", list(naf.NAF_MODES))
@pytest.mark.parametrize("bounds", ["none", "scalar"])
def test_loss_without_or_with_scalar_bounds(mode, bounds):
    nets, lo, hi, batch = make_problem(257, 3, seed=5, bounds=bounds)
    for clip in (True, False):
        _loss_case(mode, nets, lo, hi, batch, clip_delta=clip, mean=True, use_w=True)


def _loss_case(mode, nets, lo, hi, batch, clip_delta, mean, use_w, alpha=0.7):
    (mu, mat, v), (tmu, tmat, tv), (tnmu, tnmat, tnv), (nmu, nmat, nv) = nets
    mu = mu.clone().requires_grad_()
    mat = mat.clone().requires_grad_()
    v = v.clone().requires_grad_()
    q = _qav(mu, mat, v, lo, hi)
    tq, tnq, nq = _qav(tmu, tmat, tv, lo, hi), _qav(tnmu, tnmat, tnv, lo, hi), _qav(nmu, nmat,
                                                                                    nv, lo, hi)
    w = batch["weights"] if use_w else None
    loss, delta, y, t = naf.td_loss(
        q, batch["action"], tnq, batch["reward"], batch["discount"], batch["is_state_terminal"],
        w, mode, target=tq, next_online=nq, alpha=alpha, clip_delta=clip_delta, mean=mean)
    d64 = {k: x.double() for k, x in batch.items()}
    lo64 = None if lo is None else lo.double()
    hi64 = None if hi is None else hi.double()

    def q64(m, p, vv):
        return _qav(m.detach().double(), p.detach().double(), vv.detach().double(), lo64, hi64)

    Q, TQ, TNQ, NQ = q64(mu, mat, v), q64(tmu, tmat, tv), q64(tnmu, tnmat, tnv), q64(nmu, nmat,
                                                                                    nv)
    n = mu.shape[1]
    y64 = Q.evaluate_actions(d64["action"])
    y_tol = (n + 16) * U * _abs_q(Q, d64["action"])
    t64, t_m = target64(mode, d64, Q, TQ, TNQ, NQ, alpha)
    t_tol = (n + 32) * U * t_m
    assert bool(((y.double() - y64).abs() <= y_tol).all())
    assert bool(((t.double() - t64).abs() <= t_tol).all())
    assert bool(((delta.double() - (y64 - t64).abs()).abs() <= y_tol + t_tol + 1e-30).all())
    B = y.shape[0]
    e = y64 - t64
    if clip_delta:
        lv = torch.where(e.abs() < 1, 0.5 * e * e, e.abs() - 0.5)
        lv_tol = (e.abs().clamp(max=1) + 1) * (y_tol + t_tol)
    else:
        lv = 0.5 * e * e
        lv_tol = (e.abs() + 1) * (y_tol + t_tol)
    wv = d64["weights"] if use_w else torch.ones_like(lv)
    div = B if mean else 1
    loss64 = (lv * wv).sum() / div
    loss_tol = ((lv_tol + lv.abs() * (B + 4) * U) * wv).sum() / div + 1e-30
    assert abs(loss.item() - loss64.item()) <= loss_tol.item()
    # gradients: fp64 autograd of the reference's evaluate_actions, with d loss / d y taken at
    # the kernel's own y and t (checked above)
    loss.backward()
    ek = (y - t).double()
    gy = (ek.clamp(-1, 1) if clip_delta else ek) * wv / div
    mu64 = mu.detach().double().requires_grad_()
    mat64 = mat.detach().double().requires_grad_()
    v64 = v.detach().double().requires_grad_()
    (QuadraticActionValue(mu64, mat64, v64).evaluate_actions(d64["action"]) * gy).sum().backward()
    dabs = (d64["action"] - mu64.detach()).abs()
    Pabs = mat64.detach().abs()
    mu_tol = (n + 16) * U * gy.abs()[:, None] * ((Pabs + Pabs.transpose(1, 2)) @ dabs[:, :, None])[:, :, 0]
    mat_tol = 8 * U * gy.abs()[:, None, None] * dabs[:, :, None] * dabs[:, None, :]
    assert bool(((mu.grad.double() - mu64.grad).abs() <= mu_tol + 1e-30).all())
    assert bool(((mat.grad.double() - mat64.grad).abs() <= mat_tol + 1e-30).all())
    assert bool(((v.grad.double() - v64.grad).abs() <= 6 * U * gy.abs()[:, None] + 1e-30).all())


@pytest.mark.parametrize("mean", [True, False])
def test_huber_boundary_terminal_samples_and_zero_weights(mean):
    """P = 0, terminal samples: y = v and t = r exactly, |y - t| = 1 on the Huber boundary."""
    B, n = 300, 3
    mu = torch.zeros(B, n, device="cuda", requires_grad=True)
    mat = torch.zeros(B, n, n, device="cuda", requires_grad=True)
    v = torch.full((B, 1), 1.5, device="cuda", requires_grad=True)
    tn = QuadraticActionValue(torch.zeros(B, n, device="cuda"), torch.zeros(B, n, n, device="cuda"),
                              torch.full((B, 1), 9.0, device="cuda"))
    r = torch.full((B,), 0.5, device="cuda")
    r[1::2] = 2.5
    w = torch.rand(B, device="cuda")
    w[::5] = 0.0
    loss, delta, y, t = naf.td_loss(
        QuadraticActionValue(mu, mat, v), torch.randn(B, n, device="cuda"), tn, r,
        torch.full((B,), 0.99, device="cuda"), torch.ones(B, device="cuda"), w, "dqn",
        clip_delta=True, mean=mean)
    assert torch.equal(delta, torch.ones(B, device="cuda"))
    y_ref = v.detach().reshape(-1).clone().requires_grad_()
    ref = torch.nn.functional.smooth_l1_loss(y_ref, r, reduction="none")
    ref = (ref * w).sum() / (B if mean else 1)
    ref.backward()
    assert abs(loss.item() - ref.item()) <= 1e-6 * max(1.0, abs(ref.item()))
    loss.backward()
    assert torch.allclose(v.grad.reshape(-1), y_ref.grad, rtol=1e-6, atol=0)
    assert bool((v.grad.reshape(-1)[::5] == 0).all())


def test_mu_outside_the_bounds_is_clamped_for_max_only():
    """mu far outside the box: max' is Q' at the clamped mu (below V'), as the reference."""
    B, n = 64, 2
    (mu, mat, v), (tmu, tmat, tv), (tnmu, tnmat, tnv), nxt, = make_problem(B, n, 3)[0]
    lo, hi = torch.tensor([-0.1, -0.2], device="cuda"), torch.tensor([0.1, 0.2], device="cuda")
    tnmu = tnmu * 10
    batch = dict(action=torch.zeros(B, n, device="cuda"), reward=torch.zeros(B, device="cuda"),
                 discount=torch.ones(B, device="cuda"),
                 is_state_terminal=torch.zeros(B, device="cuda"))
    tnq = _qav(tnmu, tnmat, tnv, lo, hi)
    _, _, _, t = naf.td_loss(_qav(mu, mat, v, lo, hi), batch["action"], tnq, batch["reward"],
                             batch["discount"], batch["is_state_terminal"], None, "dqn")
    want = tnq.max
    assert torch.allclose(t, want, rtol=1e-5, atol=1e-5)
    assert bool((t <= tnv.reshape(-1) + 1e-6).all())


def test_non_symmetric_p_given_directly():
    B, n = 257, 5
    nets, lo, hi, batch = make_problem(B, n, 11)
    g = torch.Generator(device="cuda").manual_seed(1)
    nets = [(m, torch.randn(B, n, n, device="cuda", generator=g), vv) for m, _, vv in nets]
    for mode in ("dqn", "pal", "double_pal"):
        _loss_case(mode, nets, lo, hi, batch, clip_delta=False, mean=True, use_w=True)
