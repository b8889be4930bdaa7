"""GPU: k_adv_td_fwd (csrc/losses.cu, ops.losses.adv_td_loss), the targets of AL, PAL,
DoublePAL, DPP, DPPL and DPPGreedy fused with the scalar TD loss, against restatements of the
reference's expressions (pfrl/agents/al.py:69-80, pal.py:60-78, double_pal.py:48-70,
dpp.py:34-105, action_value.py:60-79), evaluated as in tests/test_loss_kernels_fp64_gpu.py:

* in fp32 with torch on the device -- what pfrl computes;
* in fp64 on the fp32 inputs.  For DPP and DPPL the reference first forms z = fp32(eta) * Q'
  in fp32 (``eta * q_values``); kernel and torch round that product identically, so the fp64
  evaluation starts from the same fp32 z and measures the rest.

Tolerances (U = 2**-24):

* AL, PAL, DOUBLE_PAL, DPP_GREEDY: y, t and delta are gathers, row maxima and element-wise
  fp32 operations in the reference's order, with alpha rounded to fp32 once as torch rounds a
  Python float factor.  They are bit-equal to torch fp32.
* DPP: L(x) = sum_j softmax(z)_j x_j.  exp(z_j - max z) carries the subtraction's rounding
  (|z_j - m| U relative, times the weight e^-(m - z_j) <= 1/e per term) and expf's 2 ulp; the
  sum over nA terms adds nA U relative; the normalisation and the products a few U.  So
  |dL| <= (2 nA + 8) U max|x|.  The target t = (Q'(s,a) + r + c L(s')) - L(s), c <= 1, adds
  its own roundings of magnitude <= U (|Q'(s,a)| + |r| + |L|) each.  Bound per row:
  (4 nA + 16) U M, with M = max|Q'(s)| + max|Q'(s')| + |r|.
* DPPL: L(x) = (log sum_j e^(z_j - m) + m) / eta.  The sum S in [1, nA] is good to
  (2 nA + 4) U relative, logf adds 1 ulp of log S <= 8 U, the addition of m and the
  multiplication by fp32(1 / fp32(eta)) (torch's x / eta on CUDA) 3 U |L|.  Bound per row:
  (4 nA + 16) U M + 4 (nA + 8) U / eta.
  The same bounds hold against torch fp32, which rounds the same quantities in another order.
* Loss: the finish_sum bound (ceil(B / 256) + 10) U sum|term| / divisor, plus 5 U per term for
  the term's own roundings (d, d*d or the Huber branch, the weight).
* Gradient: b2rl_td_loss_bwd on the kernel's y and t, bit for bit.
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = "cuda"
U = 2.0 ** -24
MODES = ("al", "pal", "double_pal", "dpp", "dppl", "dpp_greedy")
EXACT = ("al", "pal", "double_pal", "dpp_greedy")
ALPHAS = (0.0, 0.9, 0.99, 1.0 / 3)
ETAS = (0.1, 1.0, 2.0, 10.0)


def gather(x, a):
    return x.gather(1, a.long()[:, None])[:, 0]


def row_max(x):  # DiscreteActionValue.max: the value at argmax (first maximal index)
    return gather(x, x.argmax(dim=1))


def l_operator(mode, x32, eta, dtype):
    """dpp.py:80-105 on fp32 action values x32, evaluated in dtype after z = fp32(eta) x."""
    x = x32.to(dtype)
    if mode == "dpp_greedy":
        return row_max(x)
    z = (eta * x32).to(dtype)
    if mode == "dpp":
        return torch.sum(F.softmax(z, dim=1) * x, dim=1)
    return torch.logsumexp(z, dim=1) / eta


def target_ref(mode, tq, tnq, nq, action, reward, discount, terminal, alpha, eta, dtype):
    """The reference's _compute_y_and_t targets, in dtype."""
    r, d, term = (v.to(dtype) for v in (reward, discount, terminal))
    if mode in ("al", "pal", "double_pal"):
        tq_, tnq_ = tq.to(dtype), tnq.to(dtype)
        next_v = gather(tnq_, nq.argmax(dim=1)) if mode == "double_pal" else row_max(tnq_)
        t_q = r + d * (1.0 - term) * next_v
        cur = gather(tq_, action) - row_max(tq_)
        if mode == "al":
            return t_q + alpha * cur
        nxt = gather(tnq_, action) - row_max(tnq_)
        return t_q + alpha * torch.max(cur, nxt)
    batch_q_target = r + d * (1 - term) * l_operator(mode, tnq, eta, dtype)
    return gather(tq.to(dtype), action) + batch_q_target - l_operator(mode, tq, eta, dtype)


def value_loss(y, t, weights, clip, mean):
    """pfrl/agents/dqn.py:44-104."""
    acc = "mean" if mean else "sum"
    y, t = y.reshape(-1, 1), t.reshape(-1, 1)
    if weights is None:
        return F.smooth_l1_loss(y, t, reduction=acc) if clip else F.mse_loss(y, t, reduction=acc) / 2
    losses = (F.smooth_l1_loss(y, t, reduction="none") if clip
              else F.mse_loss(y, t, reduction="none") / 2).reshape(-1)
    loss = torch.sum(losses * weights.to(losses.dtype))
    return loss / y.shape[0] if mean else loss


def t_bound(mode, tq, tnq, reward, eta):
    nA = tq.shape[1]
    M = tq.abs().amax(1).double() + tnq.abs().amax(1).double() + reward.abs().double()
    b = (4 * nA + 16) * U * M
    if mode == "dppl":
        b = b + 4 * (nA + 8) * U / eta
    return b


def check(what, got, want, bound=None):
    got, want = got.double().reshape(-1), want.double().reshape(-1)
    if bound is None:
        bad = ~((got == want) | (torch.isnan(got) & torch.isnan(want)))
    else:
        bound = torch.as_tensor(bound, dtype=torch.float64, device=got.device).reshape(-1)
        bad = ~((got - want).abs() <= bound)
    if bool(bad.any()):
        i = int(torch.nonzero(bad)[0])
        raise AssertionError("%s: %d of %d differ; first at %d: got %r, want %r%s" % (
            what, int(bad.sum()), got.numel(), i, got[i].item(), want[i].item(),
            "" if bound is None else ", bound %r" % bound.reshape(-1)[i].item()))


def inputs(B, nA, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    rnd = lambda *s: torch.randn(*s, device=DEV, generator=g)  # noqa: E731
    q, tq, tnq, nq = rnd(B, nA) * 2, rnd(B, nA) * 2, rnd(B, nA) * 2, rnd(B, nA) * 2
    action = torch.randint(0, nA, (B,), device=DEV, generator=g)
    reward = rnd(B)
    discount = torch.where(torch.rand(B, device=DEV, generator=g) < 0.5,
                           torch.tensor(0.99, device=DEV), torch.tensor(0.99 ** 3, device=DEV))
    terminal = (torch.rand(B, device=DEV, generator=g) < 0.1).float()
    weights = torch.rand(B, device=DEV, generator=g) + 0.05
    return q, action, tq, tnq, nq, reward, discount, terminal, weights


def run(mode, q, action, tq, tnq, nq, reward, discount, terminal, weights, alpha, eta, clip,
        mean):
    from pfrl_b200.ops.losses import adv_td_loss

    return adv_td_loss(q, action, tq, tnq, reward, discount, terminal, weights, mode,
                       alpha=alpha, eta=eta, next_q=nq if mode == "double_pal" else None,
                       clip_delta=clip, mean=mean)


def check_targets(mode, q, action, tq, tnq, nq, reward, discount, terminal, alpha, eta):
    """y, t, delta of the kernel against torch fp32 and fp64; returns the kernel's t."""
    _, delta, y, t = run(mode, q, action, tq, tnq, nq, reward, discount, terminal, None,
                         alpha, eta, True, True)
    args = (mode, tq, tnq, nq, action, reward, discount, terminal, alpha, eta)
    t32 = target_ref(*args, torch.float32)
    y32 = gather(q, action)
    check("%s y" % mode, y, y32)
    if mode in EXACT:
        check("%s t (alpha %r)" % (mode, alpha), t, t32)
        check("%s delta" % mode, delta, torch.abs(y32 - t32))
        t64 = target_ref(*args, torch.float64)
        finite = torch.isfinite(t64)
        check("%s t vs fp64" % mode, t[finite], t64[finite],
              (16 * U * (tq.abs().amax(1) + tnq.abs().amax(1) + reward.abs()).double())[finite])
    else:
        b = t_bound(mode, tq, tnq, reward, eta)
        check("%s t vs fp64 (eta %r)" % (mode, eta), t, target_ref(*args, torch.float64), b)
        check("%s t vs fp32 (eta %r)" % (mode, eta), t, t32, b)
        check("%s delta" % mode, delta, torch.abs(y32 - t))
    return t


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("nA", [1, 2, 18, 33, 257])
@pytest.mark.parametrize("B", [1, 31, 32, 33, 255, 256, 257, 4099])
def test_adv_td_loss(B, nA, mode):
    from pfrl_b200 import _lib
    from pfrl_b200.ops.losses import _p

    q, action, tq, tnq, nq, reward, discount, terminal, weights = inputs(B, nA, 17 * B + nA)
    for alpha, eta in zip(ALPHAS, ETAS):
        t = check_targets(mode, q, action, tq, tnq, nq, reward, discount, terminal, alpha, eta)
    y = gather(q, action)
    for clip in (True, False):
        for mean in (True, False):
            for w in (weights, None):
                qk = q.clone().requires_grad_(True)
                loss, _, yk, tk = run(mode, qk, action, tq, tnq, nq, reward, discount, terminal,
                                      w, ALPHAS[-1], ETAS[-1], clip, mean)
                check("t repeat", tk, t)
                y64, t64 = y.double(), t.double()
                d = (y64 - t64).abs()
                el = torch.where(d < 1, 0.5 * d * d, d - 0.5) if clip else 0.5 * d * d
                if w is not None:
                    el = el * w.double()
                div = B if mean else 1
                bound = (math.ceil(B / 256) + 10 + 5) * U * float(el.abs().sum()) / div
                want = float(el.sum()) / div
                assert abs(loss.item() - want) <= bound, (clip, mean, w is None, loss.item(),
                                                          want, bound)
                loss.backward()
                g_direct = torch.empty(B, nA, device=DEV)
                act = action.long().contiguous()
                gl = torch.ones(1, device=DEV)
                L = _lib.load()
                _lib.check(L.b2rl_td_loss_bwd(_p(yk), _p(tk), _p(w), _p(act), _p(gl), B, nA,
                                              int(clip), int(mean), _p(g_direct),
                                              ctypes.c_void_p(torch.cuda.current_stream()
                                                              .cuda_stream)))
                check("grad", qk.grad, g_direct)
                qa = q.clone().requires_grad_(True)
                value_loss(gather(qa, action), t, w, clip, mean).backward()
                check("grad vs fp32 autograd", qk.grad, qa.grad,
                      4 * U * qa.grad.abs().double() + 1e-30)


def planted(nA=6):
    """Rows where a tie rule, a NaN-free max or the exp range decides the target."""
    rows = []
    base = torch.tensor([0.5, -1.0, 2.0, 0.25, -0.75, 1.5])[:nA]

    def row(tq=None, tnq=None, nq=None, a=0, r=0.5, disc=0.99, term=0.0):
        rows.append((base.clone() if tq is None else torch.tensor(tq, dtype=torch.float32),
                     base.flip(0).clone() if tnq is None else torch.tensor(tnq, dtype=torch.float32),
                     base.clone() if nq is None else torch.tensor(nq, dtype=torch.float32),
                     a, r, disc, term))

    # DoublePAL: online Q(s') ties at 1 and 3 whose target values differ (first index wins)
    row(nq=[0.0, 5.0, 1.0, 5.0, 2.0, -1.0], tnq=[0.1, -0.3, 0.2, 0.7, 0.0, 0.4], a=2)
    row(nq=[5.0, 5.0, 5.0, 5.0, 5.0, 5.0], tnq=[0.9, 0.1, 0.2, 0.3, 0.4, 0.5], a=3)
    # ties in Q'(s) and Q'(s'), including the stored action
    row(tq=[1.0, 3.0, 3.0, -2.0, 3.0, 0.0], tnq=[2.0, 2.0, -1.0, 2.0, 0.5, 0.0], a=2)
    row(tq=[1.0, 3.0, 3.0, -2.0, 3.0, 0.0], tnq=[2.0, 2.0, -1.0, 2.0, 0.5, 0.0], a=1)
    # PAL: both advantages equal
    row(tq=[1.0, 2.0, 0.0, 0.0, 0.0, 0.0], tnq=[3.0, 4.0, 0.0, 0.0, 0.0, 0.0], a=0)
    # terminal = 1, discount = 0
    row(term=1.0, a=4)
    row(disc=0.0, a=5, r=-1.25)
    # |eta Q'| about 100 for eta = 2 (DPP / DPPL overflow without the max shift)
    row(tq=[50.0, -49.0, 49.5, 10.0, -50.0, 0.0], tnq=[-50.0, 49.9, 50.0, 49.0, -3.0, 1.0], a=1)
    row(tq=[-50.0, -49.0, -49.5, -50.0, -50.0, -48.0], tnq=[-50.0] * 6, a=0)
    # constant rows
    row(tq=[0.3] * 6, tnq=[-0.7] * 6, nq=[1.0] * 6, a=2)
    q = torch.stack([r[0] * 0.5 + 0.1 for r in rows])
    tq, tnq, nq = (torch.stack([r[k] for r in rows]) for k in (0, 1, 2))
    action = torch.tensor([r[3] for r in rows])
    reward, discount, terminal = (torch.tensor([r[k] for r in rows], dtype=torch.float32)
                                  for k in (4, 5, 6))
    return [x.to(DEV) for x in (q, action, tq, tnq, nq, reward, discount, terminal)]


@pytest.mark.parametrize("mode", MODES)
def test_planted_rows(mode):
    q, action, tq, tnq, nq, reward, discount, terminal = planted()
    for alpha, eta in ((0.9, 2.0), (1.0 / 3, 1.0), (0.99, 0.1)):
        check_targets(mode, q, action, tq, tnq, nq, reward, discount, terminal, alpha, eta)
    if mode == "double_pal":  # the first tied index, not the last
        _, _, _, t = run(mode, q, action, tq, tnq, nq, reward, discount, terminal, None, 0.0,
                         1.0, True, True)
        want = reward + discount * (1 - terminal) * gather(tnq, nq.argmax(1))
        check("double_pal first tie", t[:2], want[:2])
        assert t[0].item() != (reward[0] + discount[0] * tnq[0, 3]).item()


@pytest.mark.parametrize("mode", ["dpp", "dppl", "dpp_greedy"])
def test_one_action_operator_is_the_value(mode):
    """nA = 1: L(x) = x, so t = Q'(s) + T(L = Q'(s')) - Q'(s)."""
    B = 300
    q, action, tq, tnq, nq, reward, discount, terminal, _ = inputs(B, 1, 5)
    tq[:7, 0] = torch.tensor([0.0, 1e-30, -3.5, 40.0, -60.0, 1e4, 7.0], device=DEV)
    for eta in ETAS:
        _, _, _, t = run(mode, q, action, tq, tnq, nq, reward, discount, terminal, None, 0.0,
                         eta, True, True)
        want = tq[:, 0] + (reward + discount * (1 - terminal) * tnq[:, 0]) - tq[:, 0]
        bound = None if mode != "dppl" else \
            4 * U * (tq.abs()[:, 0] + tnq.abs()[:, 0] + reward.abs()).double()
        check("%s nA=1 eta %r" % (mode, eta), t, want, bound)


def test_invalid_arguments_raise():
    from pfrl_b200 import _lib
    from pfrl_b200._lib import B2rlError
    from pfrl_b200.ops.losses import _p

    L = _lib.load()
    B, nA = 4, 3
    f = lambda *s: torch.zeros(*s, device=DEV)  # noqa: E731
    q, tq, tnq, nq = f(B, nA), f(B, nA), f(B, nA), f(B, nA)
    act = torch.zeros(B, dtype=torch.long, device=DEV)
    vec = [f(B) for _ in range(3)]
    outs = [f(B) for _ in range(4)] + [f(1)]
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def call(mode=0, q_=q, nq_=None, B_=B, nA_=nA, eta=1.0, reward=vec[0], loss=outs[4]):
        return L.b2rl_adv_td_loss_fwd(mode, _p(q_), _p(act), _p(tq), _p(tnq), _p(nq_),
                                      _p(reward), _p(vec[1]), _p(vec[2]), None, B_, nA_, 0.9,
                                      eta, 1, 1, *(_p(o) for o in outs[:4]), _p(loss), s)

    assert call() == 0
    torch.cuda.synchronize()
    for kw in (dict(q_=None), dict(reward=None), dict(loss=None), dict(B_=0), dict(nA_=0),
               dict(B_=-1), dict(mode=6), dict(mode=-1), dict(mode=2), dict(mode=3, eta=0.0),
               dict(mode=4, eta=-1.0), dict(mode=3, eta=float("nan")), dict(mode=4, eta=1e-50)):
        with pytest.raises(B2rlError):
            _lib.check(call(**kw))
    assert call(mode=2, nq_=nq) == 0 and call(mode=5, eta=0.0) == 0
    torch.cuda.synchronize()
