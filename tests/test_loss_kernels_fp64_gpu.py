"""GPU: the loss, GAE and PPO kernels (csrc/losses.cu, csrc/ppo.cu) against restatements of
the reference's expressions, at the agents' shapes, across the 256-thread block boundaries and
at the points where a gradient changes branch.

The references are the reference's torch expressions, written out below with the reference's
line numbers, and evaluated two ways:

* in fp64 on the fp32 inputs.  This is the accuracy yardstick for values everywhere and for
  gradients away from branch points;
* in fp32 with torch autograd on the same device.  pfrl runs exactly this fp32 code, so this
  evaluation fixes what the reference does at ties and on clip bounds, where the fp64
  evaluation may take the other branch.  It is used for the planted edge elements.

Tolerances (U = 2**-24, the fp32 unit roundoff):

* Element-wise outputs (delta, y, t, the projected target, the gradients):
  |x - x64| <= k U S + (the error carried in from an earlier output), where S is the sum of
  the magnitudes of the rounded terms -- the input scale, not the result, because y - t
  cancels -- and k counts the fp32 roundings in the chain.
* fp32 batch reductions (finish_sum: a strided sum per thread, a 256-thread tree, the
  division): |L - L64| <= (ceil(B / 256) + log2(256) + 2) U sum|term_i| / divisor, plus the
  element terms' own error carried through the sum.
* fp64-accumulated sums (the GAE moments, the PPO partial losses) are rounded to fp32 once:
  2**-23 relative, plus, for PPO, the fp32 element terms' own error.
* Planted edge elements match the fp32 autograd reference to 4 U relative: kernel and torch
  round the same products in different orders, but a gradient that is 0 where the reference
  passes half misses by far more.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = "cuda"
U = 2.0 ** -24
BLOCK = 256  # threads per CTA of k_td_fwd, k_qh_fwd, k_c51_fwd and k_ppo_loss


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def check(what, got, want, bound):
    """Element-wise |got - want| <= bound, in fp64."""
    got = torch.as_tensor(got).double().reshape(-1)
    want = torch.as_tensor(want).double().to(got.device).reshape(-1)
    bound = torch.as_tensor(bound, dtype=torch.float64).to(got.device).reshape(-1)
    bound = bound.expand_as(got) if bound.numel() == 1 else bound
    err = (got - want).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        i = int(torch.nonzero(bad)[0])
        raise AssertionError("%s: %d of %d outside the bound; first at %d: got %r, want %r, "
                             "bound %r" % (what, int(bad.sum()), got.numel(), i, got[i].item(),
                                           want[i].item(), bound[i].item()))


def finish_sum_bound(n, abs_sum, divisor):
    """fp32 error of finish_sum over n terms whose magnitudes sum to abs_sum."""
    return (math.ceil(n / BLOCK) + math.log2(BLOCK) + 2) * U * abs_sum / divisor


def spread_rows(B, k):
    """Up to k distinct rows spread over [0, B), first and last included."""
    return sorted(set(int(round(x)) for x in np.linspace(0, B - 1, min(B, k))))


# ---------------------------------------------------------------------------
# Reference expressions
# ---------------------------------------------------------------------------
def td_ref(q, action, next_q, reward, discount, terminal, weights, clip, mean):
    """pfrl/agents/dqn.py:388-470 (target, y, |y - t| errors) and :44-104 (value loss)."""
    B = q.shape[0]
    acc = "mean" if mean else "sum"
    y = q.gather(1, action[:, None])
    t = (reward + discount * (1.0 - terminal) * next_q).reshape(B, 1)
    if weights is None:
        loss = (F.smooth_l1_loss(y, t, reduction=acc) if clip
                else F.mse_loss(y, t, reduction=acc) / 2)
    else:
        losses = (F.smooth_l1_loss(y, t, reduction="none") if clip
                  else F.mse_loss(y, t, reduction="none") / 2).reshape(-1)
        loss = torch.sum(losses * weights)
        if mean:
            loss = loss / B
    return loss, torch.abs(y - t)[:, 0], y[:, 0], t[:, 0]


def categorical_projection(y, y_probs, z):
    """pfrl/agents/categorical_dqn.py:7-57."""
    batch_size, n_atoms = y.shape
    delta_z = z[1] - z[0]
    v_min, v_max = z[0], z[-1]
    y = torch.clamp(y, v_min, v_max)
    bj = torch.clamp((y - v_min) / delta_z, 0, n_atoms - 1)
    l, u = torch.floor(bj), torch.ceil(bj)
    z_probs = torch.zeros((batch_size, n_atoms), dtype=y.dtype, device=y.device)
    z_probs.scatter_add_(1, l.long(), y_probs * (1 - (bj - l)))
    z_probs.scatter_add_(1, u.long(), y_probs * (bj - l))
    return z_probs, bj


def c51_ref(y, next_p, reward, discount, terminal, weights, z, mean):
    """pfrl/agents/categorical_dqn.py:178-204 (target: :147-152, projection: :7-57)."""
    B = y.shape[0]
    Tz = reward[..., None] + (1.0 - terminal[..., None]) * discount[..., None] * z[None]
    t, bj = categorical_projection(Tz, next_p, z)
    eltwise_loss = -t * torch.log(torch.clamp(y, 1e-10, 1.0))
    per = eltwise_loss.sum(dim=1)
    if weights is not None:
        loss = torch.matmul(per, weights)
        if mean:
            loss = loss / B
    else:
        loss = per.mean() if mean else eltwise_loss.sum()
    return loss, per, t, Tz, bj


def qh_ref(y, t, taus, weights, mean):
    """pfrl/agents/iqn.py:176-250, errors of :385-389."""
    yb, tb, tab = torch.broadcast_tensors(y.unsqueeze(2), t.unsqueeze(1), taus.unsqueeze(2))
    I_delta_lt_0 = (tb < yb).to(y.dtype)
    eltwise_loss = torch.abs(tab - I_delta_lt_0) * F.smooth_l1_loss(yb, tb, reduction="none")
    if weights is not None:
        loss = torch.matmul(eltwise_loss.mean(2).sum(1), weights)
        if mean:
            loss = loss / y.shape[0]
    elif mean:
        loss = eltwise_loss.mean((0, 2)).sum()
    else:
        loss = eltwise_loss.mean(2).sum()
    return loss, eltwise_loss.mean((1, 2)), eltwise_loss


def gae_ref(reward, nonterminal, v, v_next, cut, valid, gamma, lambd):
    """pfrl/agents/ppo.py:36-53 over the episode segments of a [T, E] rollout (a segment ends
    at cut; an invalid slot holds no transition), in fp64.  Also returns the magnitude S of
    the terms each advantage sums, for the error bound."""
    r, nt, vv, vn = (np.asarray(x, dtype=np.float64) for x in (reward, nonterminal, v, v_next))
    T, E = r.shape
    adv, S = np.zeros(E), np.zeros(E)
    out, mag = np.zeros((T, E)), np.zeros((T, E))
    for t in range(T - 1, -1, -1):
        ok = valid[t]
        start = cut[t] | ~ok
        adv[start], S[start] = 0.0, 0.0
        td_err = r[t] + gamma * nt[t] * vn[t] - vv[t]
        adv = np.where(ok, td_err + gamma * lambd * adv, 0.0)
        S = np.where(ok, np.abs(r[t]) + gamma * np.abs(nt[t] * vn[t]) + np.abs(vv[t])
                     + gamma * lambd * S, 0.0)
        out[t], mag[t] = adv, S
    return out, out + np.where(valid, vv, 0.0), mag


def ppo_ref(log_probs, entropy, vs_pred, log_probs_old, vs_pred_old, advs, vs_teacher, stats,
            clip_eps, clip_eps_vf, value_coef, entropy_coef):
    """pfrl/agents/ppo.py:495 (advantage standardisation, stats from :476-478) and
    :634-671 (_lossfun), with _elementwise_clip of :28-33."""
    if stats is not None:
        advs = (advs - stats[0]) / (stats[1] + 1e-8)
    prob_ratio = torch.exp(log_probs - log_probs_old)
    loss_policy = -torch.mean(torch.min(
        prob_ratio * advs, torch.clamp(prob_ratio, 1 - clip_eps, 1 + clip_eps) * advs))
    if clip_eps_vf is None:
        loss_value_func = F.mse_loss(vs_pred, vs_teacher)
    else:
        clipped_vs_pred = torch.min(torch.max(vs_pred, vs_pred_old - clip_eps_vf),
                                    vs_pred_old + clip_eps_vf)
        loss_value_func = torch.mean(torch.max(
            F.mse_loss(vs_pred, vs_teacher, reduction="none"),
            F.mse_loss(clipped_vs_pred, vs_teacher, reduction="none")))
    loss_entropy = -torch.mean(entropy)
    loss = loss_policy + value_coef * loss_value_func + entropy_coef * loss_entropy
    return loss, loss_policy, loss_value_func, loss_entropy, advs, prob_ratio


def grads(fn, inputs, dtype):
    """Evaluate fn on copies of inputs in dtype; returns (outputs, d out[0] / d input) for
    the inputs given as (tensor, True)."""
    xs = [None if x is None else
          (x[0].detach().to(dtype).requires_grad_(True) if isinstance(x, tuple)
           else (x.to(dtype) if x.is_floating_point() else x)) for x in inputs]
    out = fn(*xs)
    leaves = [x for x, i in zip(xs, inputs) if isinstance(i, tuple)]
    g = torch.autograd.grad(out[0], leaves)
    return [o.detach() if torch.is_tensor(o) else o for o in out], g


# ---------------------------------------------------------------------------
# TD loss (k_td_fwd / k_td_bwd)
# ---------------------------------------------------------------------------
def td_inputs(B, nA, seed):
    g = gen(seed)
    q = torch.randn(B, nA, device=DEV, generator=g) * 2
    action = torch.randint(0, nA, (B,), device=DEV, generator=g)
    next_q = torch.randn(B, device=DEV, generator=g) * 2
    reward = torch.randn(B, device=DEV, generator=g)
    discount = torch.where(torch.rand(B, device=DEV, generator=g) < 0.5,
                           torch.tensor(0.99, device=DEV), torch.tensor(0.99 ** 3, device=DEV))
    terminal = (torch.rand(B, device=DEV, generator=g) < 0.1).float()
    weights = torch.rand(B, device=DEV, generator=g) + 0.05
    # planted rows: d = 0, d = +1 and d = -1 exactly (t = r: next_q = 0), a terminal row
    rows = spread_rows(B, 4)
    plants = [(0.5, 0.5), (0.75, -0.25), (0.25, 1.25)]  # (q[i, a_i], r): d = 0, 1, -1
    for k, i in enumerate(rows[:3]):
        q[i, action[i]], reward[i], next_q[i] = plants[k][0], plants[k][1], 0.0
    terminal[rows[-1]] = 1.0
    return q, action, next_q, reward, discount, terminal, weights, rows[:3]


@pytest.mark.parametrize("B", [1, 255, 256, 257, 512, 4099])
@pytest.mark.parametrize("nA", [1, 18])
@pytest.mark.parametrize("clip", [True, False])
@pytest.mark.parametrize("mean", [True, False])
@pytest.mark.parametrize("use_w", [True, False])
def test_td_loss(B, nA, clip, mean, use_w):
    from pfrl_b200.ops.losses import td_loss

    q, action, next_q, reward, discount, terminal, weights, planted = td_inputs(B, nA, B + nA)
    w = weights if use_w else None
    qk = q.clone().requires_grad_(True)
    loss, delta, y, t = td_loss(qk, action, next_q, reward, discount, terminal, w, clip, mean)
    loss.backward()

    def fn(q_, nq, r, d, term, w_):
        return td_ref(q_, action, nq, r, d, term, w_, clip, mean)

    args = [(q, True), next_q, reward, discount, terminal, w]
    (L64, d64, y64, t64), (g64,) = grads(fn, args, torch.float64)
    _, (g32,) = grads(fn, args, torch.float32)

    assert torch.equal(y, q[torch.arange(B, device=DEV), action])
    S_t = reward.double().abs() + (discount.double() * (1 - terminal.double()) * next_q.double()).abs()
    check("t", t, t64, 3 * U * S_t)
    S_d = y.double().abs() + S_t
    err_d = 4 * U * S_d
    check("delta", delta, d64, err_d)
    dd = d64  # |y - t|
    slope = dd.clamp(max=1.0) if clip else dd  # |h'(d)|
    lval = torch.where(dd < 1, 0.5 * dd * dd, dd - 0.5) if clip else 0.5 * dd * dd
    wd = weights.double() if use_w else torch.ones_like(dd)
    div = B if mean else 1
    elem = (wd * (slope * err_d + 3 * U * lval)).sum() / div
    check("loss", loss, L64, elem + finish_sum_bound(B, (wd * lval).sum(), div) + U * L64.abs())
    c = (wd / div)[:, None]
    check("grad_q", qk.grad, g64, c * err_d[:, None] + 4 * U * g64.abs())
    off = torch.ones_like(q, dtype=torch.bool)
    off[torch.arange(B, device=DEV), action] = False
    assert torch.all(qk.grad[off] == 0)
    # planted d = 0 / |d| = 1 rows against fp32 autograd
    assert len(planted) > 0
    p = torch.tensor(planted, device=DEV)
    assert torch.all(delta[p] == torch.tensor([0.0, 1.0, 1.0], device=DEV)[:len(planted)])
    check("grad_q at d = 0, |d| = 1", qk.grad[p], g32[p], 4 * U * g32[p].abs())


# ---------------------------------------------------------------------------
# Categorical projection + cross entropy (k_c51_fwd / k_c51_bwd)
# ---------------------------------------------------------------------------
def c51_inputs(B, n, seed):
    g = gen(seed)
    z = torch.from_numpy(np.linspace(-10, 10, num=n, dtype=np.float32)).to(DEV)
    y = torch.softmax(torch.randn(B, n, device=DEV, generator=g), 1)
    next_p = torch.softmax(torch.randn(B, n, device=DEV, generator=g), 1)
    reward = torch.randn(B, device=DEV, generator=g) * 3
    discount = torch.full((B,), 0.99, device=DEV)
    terminal = (torch.rand(B, device=DEV, generator=g) < 0.1).float()
    weights = torch.rand(B, device=DEV, generator=g) + 0.05
    rows = spread_rows(B, 6)
    dz = float(z[1] - z[0])
    # row plants, in order of priority for the small batches
    for k, i in enumerate(rows):
        if k == 0:  # discount 1, r a multiple of dz: bj on integers
            reward[i], discount[i], terminal[i] = dz, 1.0, 0.0
        elif k == 1:
            reward[i], terminal[i] = 50.0, 0.0  # every Tz past v_max
        elif k == 2:
            reward[i], terminal[i] = -50.0, 0.0  # every Tz past v_min
        elif k == 3:
            terminal[i] = 1.0
        elif k == 4:
            reward[i], discount[i], terminal[i] = 0.0, 1.0, 0.0
    # the clamp edges of log(clamp(y, 1e-10, 1)) and of its gradient
    edges = torch.tensor([0.0, 1e-12, 1e-10, 1.0], device=DEV)[:n]
    y[rows[-1], :len(edges)] = edges
    return z, y, next_p, reward, discount, terminal, weights, rows


def c51_bounds(z, y, next_p, reward, discount, terminal, t64, Tz64, bj64, n):
    """Per-atom bound on the fp32 projected target and the per-sample loss."""
    z64 = z.double()
    dz = z64[1] - z64[0]
    s = ((1 - terminal.double()) * discount.double())[:, None]
    err_tz = 3 * U * (reward.double().abs()[:, None] + (s * z64[None]).abs())
    err_bj = (err_tz + U * (Tz64.clamp(z64[0], z64[-1]) - z64[0]).abs()) / dz + 3 * U * bj64
    move = 2 * (next_p.double() * err_bj).sum(1, keepdim=True)  # mass between neighbours
    lo, up = bj64.floor().long(), bj64.ceil().long()
    m = torch.zeros_like(t64)
    one = torch.ones_like(t64)
    m.scatter_add_(1, lo, one)
    m.scatter_add_(1, up, one)
    bound_t = move + (m + 4) * U * t64
    logy = torch.log(torch.clamp(y.double(), 1e-10, 1.0)).abs()
    bound_per = ((bound_t * logy).sum(1)
                 + (math.ceil(n / 32) + 5 + 3) * U * (t64 * logy).sum(1))
    return bound_t, bound_per, logy


@pytest.mark.parametrize("n", [2, 32, 33, 51, 256])
@pytest.mark.parametrize("B", [1, 7, 9, 512, 4099])
@pytest.mark.parametrize("mean,use_w", [(True, True), (True, False), (False, True),
                                        (False, False)])
def test_c51_loss(n, B, mean, use_w):
    from pfrl_b200.ops.losses import c51_loss

    z, y, next_p, reward, discount, terminal, weights, rows = c51_inputs(B, n, 10 * n + B)
    w = weights if use_w else None
    yk = y.clone().requires_grad_(True)
    loss, delta, t = c51_loss(yk, next_p, reward, discount, terminal, w, mean=mean, z=z,
                              return_target=True)
    loss.backward()

    def fn(y_, p, r, d, term, w_, z_):
        return c51_ref(y_, p, r, d, term, w_, z_, mean)

    args = [(y, True), next_p, reward, discount, terminal, w, z]
    (L64, per64, t64, Tz64, bj64), (g64,) = grads(fn, args, torch.float64)
    (_, _, t32, _, bj32), (g32,) = grads(fn, args, torch.float32)

    bound_t, bound_per, logy = c51_bounds(z, y, next_p, reward, discount, terminal, t64, Tz64,
                                          bj64, n)
    check("projected target", t, t64, bound_t)
    check("per-sample loss", delta, per64, bound_per)
    wd = weights.double() if use_w else torch.ones(B, dtype=torch.float64, device=DEV)
    div = B if mean else 1
    check("loss", loss, L64, (wd * bound_per).sum() / div
          + finish_sum_bound(B, (wd * per64.abs()).sum(), div) + U * L64.abs())
    c = (wd / div)[:, None]
    y64 = y.double()
    inside = (y >= np.float32(1e-10)) & (y <= 1.0)
    g_bound = torch.where(inside, c * bound_t / y64.clamp(min=1e-10) + 5 * U * g64.abs(),
                          torch.zeros_like(g64))
    check("grad_y", yk.grad, g64, g_bound)
    # planted: bj on integers (l = u), the y clamp edges; against fp32 autograd, which
    # computes bj with the kernel's fp32 operations: only the accumulation order differs
    i = rows[0]
    assert bool((bj32[i] == bj32[i].floor()).any()), "no bj landed on an integer"
    m32 = torch.zeros_like(t32[i]).scatter_add_(0, bj32[i].floor().long(), torch.ones_like(t32[i]))
    m32.scatter_add_(0, bj32[i].ceil().long(), torch.ones_like(t32[i]))
    check("t where bj is an integer", t[i], t32[i], 2 * (m32 + 2) * U * t32[i].abs())
    r = rows[-1]
    k = min(n, 4)
    check("grad_y at y in {0, 1e-12, 1e-10, 1}", yk.grad[r, :k], g32[r, :k],
          (c[r] * bound_t[r, :k] / y64[r, :k].clamp(min=1e-10)) + 5 * U * g32[r, :k].abs())
    assert torch.all(yk.grad[r, :min(n, 2)] == 0)  # y = 0, 1e-12: clamped, no gradient
    assert torch.equal(yk.grad[r, 2:k] != 0, t[r, 2:k] != 0)  # y = 1e-10, 1: passed


@pytest.mark.parametrize("n", [1, 257])
def test_c51_atom_count_out_of_range_is_an_error(n):
    from pfrl_b200._lib import B2rlError
    from pfrl_b200.ops.losses import c51_loss

    z = torch.linspace(-10, 10, n, device=DEV)
    y = torch.full((4, n), 1.0 / n, device=DEV)
    r = torch.zeros(4, device=DEV)
    with pytest.raises(B2rlError):
        c51_loss(y, y, r, r + 0.99, r, None, z=z)


# ---------------------------------------------------------------------------
# Quantile Huber loss (k_qh_fwd / k_qh_bwd)
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("B,N,Np", [(1, 1, 1), (32, 64, 64), (32, 8, 200), (3, 200, 8),
                                    (512, 32, 32)])
@pytest.mark.parametrize("mean,use_w", [(True, True), (True, False), (False, True),
                                        (False, False)])
def test_quantile_huber_loss(B, N, Np, mean, use_w):
    from pfrl_b200.ops.losses import quantile_huber_loss

    g = gen(B * N + Np)
    y = torch.randn(B, N, device=DEV, generator=g) * 1.5
    t = torch.randn(B, Np, device=DEV, generator=g) * 1.5
    taus = torch.rand(B, N, device=DEV, generator=g)
    weights = torch.rand(B, device=DEV, generator=g) + 0.05
    # plants: a tie t = y in row 0, |t - y| = 1 exactly in the last row
    y[0, 0], t[0, 0] = 0.5, 0.5
    y[-1, -1], t[-1, -1] = 0.25, 1.25
    if Np > 1:
        t[-1, 0] = -0.75
    w = weights if use_w else None
    yk = y.clone().requires_grad_(True)
    loss, delta = quantile_huber_loss(yk, t, taus, w, mean)
    loss.backward()

    def fn(y_, t_, tau_, w_):
        return qh_ref(y_, t_, tau_, w_, mean)

    args = [(y, True), t, taus, w]
    (L64, d64, elt64), (g64,) = grads(fn, args, torch.float64)
    _, (g32,) = grads(fn, args, torch.float32)

    P = N * Np
    per_sum = elt64.sum((1, 2))
    bound_s = (math.ceil(P / BLOCK) + 8 + 6 + 2) * U * per_sum
    check("delta", delta, d64, bound_s / P)
    wd = weights.double() if use_w else torch.ones(B, dtype=torch.float64, device=DEV)
    div = B if mean else 1
    check("loss", loss, L64, (wd * bound_s / Np).sum() / div
          + finish_sum_bound(B, (wd * per_sum / Np).sum(), div) + U * L64.abs())
    d = (t.double()[:, None, :] - y.double()[:, :, None])
    I = (d < 0).double()
    terms = ((taus.double()[:, :, None] - I).abs() * d.clamp(-1, 1)).abs().sum(2)
    c = (wd / (Np * div))[:, None]
    check("grad_y", yk.grad, g64, c * (Np + 4) * U * terms + 4 * U * g64.abs())
    # planted tie and |d| = 1 elements against fp32 autograd
    for i, j in ((0, 0), (B - 1, N - 1)):
        check("grad_y at a tie / |t - y| = 1", yk.grad[i, j], g32[i, j],
              c[i, 0] * (Np + 4) * U * terms[i, j] + 4 * U * g32[i, j].abs())


# ---------------------------------------------------------------------------
# GAE (k_gae)
# ---------------------------------------------------------------------------
def gae_inputs(T, E, seed, with_valid, offset=0.0):
    rng = np.random.RandomState(seed)
    r = (offset + rng.randn(T, E)).astype(np.float32)
    v = rng.randn(T, E).astype(np.float32)
    vn = rng.randn(T, E).astype(np.float32)
    nt = (rng.rand(T, E) > 0.02).astype(np.float32)
    nt[rng.rand(T, E) < 0.01] = 0.0
    cut = (nt == 0) | (rng.rand(T, E) < 0.01)
    cut[-1] = True
    valid = rng.rand(T, E) > 0.05 if with_valid else np.ones((T, E), dtype=bool)
    if with_valid:
        valid[0, 0] = T * E == 1  # a hole, unless it is the only slot
        valid[-1, -1] = True
    return r, nt, v, vn, cut, valid


def check_gae(T, E, gamma, lambd, with_valid, offset, seed):
    from pfrl_b200.ops.ppo import gae

    r, nt, v, vn, cut, valid = gae_inputs(T, E, seed, with_valid, offset)
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)  # noqa: E731
    adv, vt, stats = gae(cu(r), cu(nt), cu(v), cu(vn), cu(cut.astype(np.uint8)), gamma, lambd,
                         valid=cu(valid.astype(np.uint8)) if with_valid else None)
    a64, vt64, S = gae_ref(r, nt, v, vn, cut, valid, gamma, lambd)
    fp64 = (T + 8) * 2.0 ** -53 * S
    check("adv", adv, a64, U * np.abs(a64) + fp64)
    check("v_teacher", vt, vt64, U * np.abs(vt64) + fp64 + 2.0 ** -53 * np.abs(v))
    if with_valid:
        assert not bool(adv[cu(~valid)].any()) and not bool(vt[cu(~valid)].any())
    av = adv.cpu().numpy()[valid].astype(np.float64)
    m, s = av.mean(), av.std()
    n_blocks = -(-E // 128)
    acc64 = (T + 5 + 4 + n_blocks) * 2.0 ** -53 * np.abs(av).mean()
    got = stats.cpu().numpy().astype(np.float64)
    check("stats mean", got[0], m, 2.0 ** -23 * abs(m) + acc64)
    check("stats std", got[1], s, 2.0 ** -23 * s + 1e-30)


@pytest.mark.parametrize("T,E", [(1, 1), (8, 256), (2048, 256), (5, 129), (3, 1000)])
@pytest.mark.parametrize("lambd", [0.0, 0.95, 1.0])
@pytest.mark.parametrize("gamma", [0.99, 1.0])
@pytest.mark.parametrize("with_valid", [False, True])
def test_gae(T, E, lambd, gamma, with_valid):
    check_gae(T, E, gamma, lambd, with_valid, 0.0, T + E)


@pytest.mark.parametrize("offset", [1e3, 1e4])
@pytest.mark.parametrize("lambd", [0.0, 0.95])
def test_gae_stats_with_reward_offset(offset, lambd):
    """The advantages sit far from 0 relative to their spread: the moments must not lose
    the spread to cancellation."""
    check_gae(2048, 256, 0.99, lambd, True, offset, 7)


# ---------------------------------------------------------------------------
# PPO loss (k_ppo_loss)
# ---------------------------------------------------------------------------
def f32_bounds(eps):
    """The reference's clamp bounds: Python floats 1 - eps, 1 + eps rounded once to fp32."""
    return float(np.float32(1 - eps)), float(np.float32(1 + eps))


def exp_preimages(targets):
    """fp32 x near log(b) with torch.exp(x) == b exactly on the device, for the targets b
    that exp reaches (the kernel's expf is the same libdevice function; the build does not
    use fast math).  expf does not reach every fp32 value below 1."""
    out = {}
    for b in targets:
        x0 = np.float32(np.log(np.float64(b)))
        xs = (np.array([x0]).view(np.int32) + np.arange(-4096, 4097, dtype=np.int32))
        xs = xs.view(np.float32)
        r = torch.exp(torch.from_numpy(xs).to(DEV)).cpu().numpy()
        hit = np.nonzero(r == np.float32(b))[0]
        if len(hit):
            out[b] = float(xs[hit[len(hit) // 2]])
    return out


def ppo_plants(eps, eps_vf, stats, g):
    """Planted elements: ratios exactly on the fp32 clip bounds and one ulp either side, min
    ties outside the clip range, v_pred exactly on v_old -+ eps_vf.  Returns columns
    (lp, adv, v, v_old, v_teacher) and the index sets of each kind."""
    lo, hi = f32_bounds(eps)
    f = np.float32
    edge = [lo, float(np.nextafter(f(lo), f(0))), float(np.nextafter(f(lo), f(2))),
            hi, float(np.nextafter(f(hi), f(0))), float(np.nextafter(f(hi), f(2)))]
    outside = ([float(x) for x in f(hi) + np.arange(1, 9, dtype=np.float32) * np.spacing(f(hi))]
               + [float(x) for x in f(lo) - np.arange(1, 9, dtype=np.float32)
                  * np.spacing(f(lo))])
    pre = exp_preimages(edge + outside)
    assert all(b in pre for b in edge), "exp reaches no ratio on / next to %r" % [lo, hi]
    outside = [b for b in outside if b in pre]
    m, s = (0.0, 1.0) if stats is None else (float(stats[0]), float(stats[1]))
    std = lambda a: a if stats is None else (a - stats[0]) / (stats[1] + 1e-8)  # noqa: E731
    lp, adv = [], []
    for b in edge:  # both advantage signs on each bound ratio
        lp += [pre[b], pre[b]]
        adv += [m + 1.5 * s, m - 0.7 * s]
    n_edge = len(lp)
    # ties: s1 == s2 in fp32 with the ratio outside [lo, hi] and adv != 0
    cand = (torch.randn(8192, device=DEV, generator=g) * s + m)
    a = std(cand)
    n_tie = {}
    for b in outside:
        bound = hi if b > hi else lo
        ratio = torch.exp(torch.tensor([pre[b]], device=DEV))
        assert float(ratio) == np.float32(b)
        tie = (ratio * a == torch.tensor(bound, device=DEV) * a) & (a != 0)
        idx = torch.nonzero(tie)[:2, 0]
        side = "hi" if b > hi else "lo"
        n_tie[side] = n_tie.get(side, 0) + len(idx)
        lp += [pre[b]] * len(idx)
        adv += cand[idx].tolist()
    n_pol = len(lp)
    assert n_tie.get("hi", 0) > 0 and n_tie.get("lo", 0) > 0, n_tie
    # value: v exactly on v_old -+ eps_vf, computed in fp32 on the device as the reference does
    vo = torch.tensor([0.3, -1.1, 0.7, 2.0], device=DEV)
    v, vt = [], []
    if eps_vf is not None:
        v = [float(vo[0] - eps_vf), float(vo[1] + eps_vf), float(vo[2] - eps_vf),
             float(vo[3] + eps_vf)]
        vt = [0.9, -0.2, -1.5, 1.0]
    return (lp, adv, v, vo.tolist()[:len(v)], vt), n_edge, len(lp)


@pytest.mark.parametrize("M", [1, 64, 255, 256, 257, 4096, 1 << 20])
@pytest.mark.parametrize("eps", [0.1, 0.18, 0.2, 0.33])
@pytest.mark.parametrize("eps_vf", [None, 0.0, 0.2])
@pytest.mark.parametrize("use_stats", [False, True])
def test_ppo_loss(M, eps, eps_vf, use_stats):
    from pfrl_b200.ops.ppo import ppo_loss

    seed = M + int(eps * 100) + (7 if eps_vf is None else int(eps_vf * 10)) + use_stats
    g = gen(seed)
    lp = torch.randn(M, device=DEV, generator=g) * 0.3
    lp_old = torch.randn(M, device=DEV, generator=g) * 0.3
    ent = torch.rand(M, device=DEV, generator=g) * 2
    v = torch.randn(M, device=DEV, generator=g)
    v_old = v + torch.randn(M, device=DEV, generator=g) * 0.3
    vt = v + torch.randn(M, device=DEV, generator=g) * 0.5
    adv = torch.randn(M, device=DEV, generator=g) * 2 + 0.3
    stats = torch.tensor([0.3, 2.1], device=DEV) if use_stats else None
    planted = M >= 64
    if planted:
        (p_lp, p_adv, p_v, p_vo, p_vt), n_edge, n_pol = ppo_plants(eps, eps_vf, stats, g)
        n_val = len(p_v)
        pos = torch.randperm(M, device=DEV, generator=g)[:n_pol]
        lp[pos] = torch.tensor(p_lp, device=DEV)
        lp_old[pos] = 0.0
        adv[pos] = torch.tensor(p_adv, device=DEV)
        if n_val:
            v[pos[:n_val]] = torch.tensor(p_v, device=DEV)
            v_old[pos[:n_val]] = torch.tensor(p_vo, device=DEV)
            vt[pos[:n_val]] = torch.tensor(p_vt, device=DEV)
    vc, ec = 0.5, 0.01
    lpk, entk, vk = (x.clone().requires_grad_(True) for x in (lp, ent, v))
    total, parts = ppo_loss(lpk, entk, vk, lp_old, v_old, adv, vt, stats, eps, eps_vf, vc, ec)
    total.backward()

    def fn(lp_, ent_, v_, lpo, vo, a, vt_, st):
        return ppo_ref(lp_, ent_, v_, lpo, vo, a, vt_, st, eps, eps_vf, vc, ec)

    args = [(lp, True), (ent, True), (v, True), lp_old, v_old, adv, vt, stats]
    (L64, P64, V64, E64, a64, r64), (glp64, gent64, gv64) = grads(fn, args, torch.float64)
    (_, _, _, _, a32, r32), (glp32, gent32, gv32) = grads(fn, args, torch.float32)

    # error budget of the fp32 element terms
    x = (lp.double() - lp_old.double()).abs()
    rel_r = (x + 3) * U
    if use_stats:
        da = U * (adv.double().abs() + 0.3) / 2.1 + 3 * U * a64.abs()
    else:
        da = torch.zeros_like(a64)
    ds = a64.abs() * r64 * rel_r + r64 * da + U * (r64 * a64).abs()
    check("policy loss", parts[1], P64, ds.sum() / M + 2.0 ** -23 * P64.abs())
    d = v.double() - vt.double()
    if eps_vf is None:
        dv = 3 * U * d * d
        ddc = torch.zeros_like(d)
    else:
        vo = v_old.double()
        ddc = U * (vo.abs() + eps_vf) * 2 + U * eps_vf + 2 * U * (vo.abs() + vt.double().abs()
                                                                  + eps_vf)
        dc = torch.min(torch.max(v.double(), vo - eps_vf), vo + eps_vf) - vt.double()
        dv = 3 * U * d * d + 2 * dc.abs() * ddc + 3 * U * dc * dc
    check("value loss", parts[2], V64, dv.sum() / M + 2.0 ** -23 * V64.abs())
    check("entropy loss", parts[3], E64, 2.0 ** -23 * E64.abs() + 1e-30)
    check("total loss", total, L64, ds.sum() / M + vc * dv.sum() / M
          + 3 * U * (P64.abs() + vc * V64.abs() + ec * E64.abs()) + 2.0 ** -23 * L64.abs())
    check("grad entropy", entk.grad, gent64, 3 * U * gent64.abs())

    # gradients away from branch points against fp64
    lo32, hi32 = f32_bounds(eps)
    near = torch.zeros(M, dtype=torch.bool, device=DEV)
    for b in (lo32, hi32, 1 - eps, 1 + eps):
        near |= ((r64 - b).abs() <= 1e-6 * b) | ((r32.double() - b).abs() <= 1e-6 * b)
    away = ~near
    check("grad log_prob (fp64, away from the clip bounds)", lpk.grad[away], glp64[away],
          ((r64 * da + a64.abs() * r64 * rel_r) / M + 4 * U * glp64.abs())[away])
    vscale = v.double().abs() + vt.double().abs() + v_old.double().abs() + (eps_vf or 0.0)
    vaway = torch.ones(M, dtype=torch.bool, device=DEV)
    if eps_vf is not None:
        vo = v_old.double()
        for b in (vo - eps_vf, vo + eps_vf, v_old - eps_vf, v_old + eps_vf):
            vaway &= (v.double() - b.double()).abs() > 1e-6 * vscale
        vaway &= (d.abs() - dc.abs()).abs() > 1e-6 * vscale
    check("grad v_pred (fp64, away from branch points)", vk.grad[vaway], gv64[vaway],
          (vc / M * 2 * (U * d.abs() + ddc + 2 * U * vscale) + 4 * U * gv64.abs())[vaway])

    if not planted:
        return
    # planted elements against fp32 autograd.  Every set is non-empty, and every set is
    # checked before the test fails, so a failure names each deviating kind.
    failures = []

    def planted_check(what, idx, got, want):
        try:
            check(what, got[idx], want[idx], 4 * U * want[idx].abs())
        except AssertionError as e:
            failures.append(str(e))

    edge = pos[:n_edge]
    r_e, a_e = r32[edge], a32[edge]
    on_bound = (r_e == lo32) | (r_e == hi32)
    # one ulp outside a bound, s1 and s2 may also round to a tie: those count as ties
    tie_e = ((r_e < lo32) | (r_e > hi32)) & (r_e * a_e == torch.clamp(r_e, lo32, hi32) * a_e)
    next_to = ~on_bound & ~tie_e
    assert bool(on_bound.any()) and bool(next_to.any())
    planted_check("grad log_prob at ratios exactly on the clip bounds", edge[on_bound],
                  lpk.grad, glp32)
    planted_check("grad log_prob at ratios one ulp from the clip bounds", edge[next_to],
                  lpk.grad, glp32)
    assert n_pol > n_edge
    tie = torch.cat([pos[n_edge:n_pol], edge[tie_e]])
    s1, s2 = r32[tie] * a32[tie], torch.clamp(r32[tie], lo32, hi32) * a32[tie]
    assert bool((s1 == s2).all()) and bool(((r32[tie] < lo32) | (r32[tie] > hi32)).all())
    planted_check("grad log_prob at min ties outside the clip range", tie, lpk.grad, glp32)
    if eps_vf is not None:
        assert n_val > 0
        vb = pos[:n_val]
        on = (v[vb] == v_old[vb] - eps_vf) | (v[vb] == v_old[vb] + eps_vf)
        assert bool(on.all())
        planted_check("grad v_pred exactly on v_old -+ eps_vf", vb, vk.grad, gv32)
    planted_check("grad v_pred at the other planted elements", pos[n_val:n_pol], vk.grad, gv32)
    assert not failures, "\n".join(failures)


# ---------------------------------------------------------------------------
# Agent level: the fused C51 loss uses the model's atoms
# ---------------------------------------------------------------------------
def test_categorical_dqn_fused_loss_matches_torch_path(monkeypatch):
    from pfrl_b200 import agents, explorers, q_functions
    from pfrl_b200.ops import losses as fused
    from pfrl_b200.replay_buffers import HostReplayBuffer

    torch.backends.cuda.matmul.allow_tf32 = False
    torch.manual_seed(0)
    OBS, NA, B = 10, 4, 512
    qf = q_functions.DistributionalFCStateQFunctionWithDiscreteAction(OBS, NA, 51, -10, 10, 32, 2)
    agent = agents.CategoricalDQN(qf, torch.optim.SGD(qf.parameters(), lr=0.0),
                                  HostReplayBuffer(2 * B), 0.99, explorers.Greedy(), gpu=0,
                                  replay_start_size=B, minibatch_size=B)
    g = gen(3)
    batch = dict(
        state=torch.randn(B, OBS, device=DEV, generator=g) * 3,
        next_state=torch.randn(B, OBS, device=DEV, generator=g) * 3,
        action=torch.randint(0, NA, (B,), device=DEV, generator=g),
        reward=torch.randn(B, device=DEV, generator=g) * 2,
        discount=torch.full((B,), 0.99, device=DEV),
        is_state_terminal=(torch.rand(B, device=DEV, generator=g) < 0.1).float(),
        weights=torch.rand(B, device=DEV, generator=g) + 0.1)
    seen = {}
    real = fused.c51_loss

    def spy(*a, **k):
        k["return_target"] = True
        loss, delta, t = real(*a, **k)
        seen["t"] = t
        return loss, delta

    monkeypatch.setattr(fused, "c51_loss", spy)
    agent.use_fused_loss = True
    loss_f, delta_f = agent._compute_loss(batch, want_errors=True)
    agent.use_fused_loss = False
    loss_t, delta_t = agent._compute_loss(batch, want_errors=True)
    with torch.no_grad():
        t_torch = agent._compute_target_values(batch)
        next_p, z = agent._next_distribution(batch)
        y = agent.model(batch["state"]).evaluate_actions_as_distribution(batch["action"])
        Tz = (batch["reward"][:, None] + (1.0 - batch["is_state_terminal"][:, None])
              * batch["discount"][:, None] * z[None])
        _, bj = categorical_projection(Tz, next_p, z)
    # both paths accumulate the same fp32 contributions, in different orders
    m = torch.zeros_like(t_torch)
    one = torch.ones_like(t_torch)
    m.scatter_add_(1, bj.floor().long(), one)
    m.scatter_add_(1, bj.ceil().long(), one)
    bound_t = 2 * (m + 2) * U * t_torch.double()
    check("projected target (fused vs torch path)", seen["t"], t_torch, bound_t)
    logy = torch.log(torch.clamp(y.double(), 1e-10, 1.0)).abs()
    tl = (t_torch.double() * logy).sum(1)
    bound_per = (bound_t * logy).sum(1) + (2 + 2 * 8) * U * tl
    check("per-sample errors (fused vs torch path)", delta_f, delta_t, bound_per)
    w = batch["weights"].double()
    check("loss (fused vs torch path)", loss_f, loss_t,
          (w * bound_per).sum() / B + 2 * finish_sum_bound(B, (w * tl).sum(), B))


# ---------------------------------------------------------------------------
# Completion tickets: back-to-back launches of mixed grid sizes wrap the 256 counters
# ---------------------------------------------------------------------------
def test_reduction_tickets_wrap():
    from pfrl_b200.ops.losses import c51_loss, quantile_huber_loss, td_loss
    from pfrl_b200.ops.ppo import gae, ppo_loss

    calls = []
    for B in (3, 300, 4099):
        q, action, next_q, reward, discount, terminal, weights, _ = td_inputs(B, 6, B)
        calls.append(("td", lambda q=q, a=action, n=next_q, r=reward, d=discount, t=terminal,
                      w=weights: td_loss(q, a, n, r, d, t, w, True, True)[0]))
    for B in (9, 700):
        z, y, next_p, reward, discount, terminal, weights, _ = c51_inputs(B, 51, B)
        calls.append(("c51", lambda z=z, y=y, p=next_p, r=reward, d=discount, t=terminal,
                      w=weights: c51_loss(y, p, r, d, t, w, z=z)[0]))
    for B in (2, 600):
        g = gen(B)
        y, t = torch.randn(B, 8, device=DEV, generator=g), torch.randn(B, 8, device=DEV, generator=g)
        taus = torch.rand(B, 8, device=DEV, generator=g)
        calls.append(("qh", lambda y=y, t=t, tau=taus: quantile_huber_loss(y, t, tau, None)[0]))
    for E in (5, 700):
        r, nt, v, vn, cut, valid = gae_inputs(16, E, E, True)
        cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)  # noqa: E731
        args = [cu(r), cu(nt), cu(v), cu(vn), cu(cut.astype(np.uint8))]
        vmask = cu(valid.astype(np.uint8))
        calls.append(("gae", lambda args=args, vmask=vmask: gae(*args, 0.99, 0.95,
                                                                valid=vmask)[2]))
    for M in (100, 5000):
        g = gen(M)
        xs = [torch.randn(M, device=DEV, generator=g) for _ in range(7)]
        calls.append(("ppo", lambda xs=xs: ppo_loss(*xs, None, 0.2, 0.2, 0.5, 0.01)[1]))
    alone = []
    for _, fn in calls:
        torch.cuda.synchronize()
        alone.append(fn().clone())
        torch.cuda.synchronize()
    order = [k % len(calls) for k in range(300)]
    outs = [calls[k][1]() for k in order]
    torch.cuda.synchronize()
    for k, out in zip(order, outs):
        kind, want = calls[k][0], alone[k]
        if kind == "c51":  # shared-memory float atomics: the target's order may change
            check("c51 loss in a back-to-back launch", out, want, 64 * U * want.abs())
        else:
            assert torch.equal(out, want), (kind, k, out, want)
