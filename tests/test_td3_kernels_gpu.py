"""GPU: the fused TD3 / DDPG critic-update kernels (csrc/sac.cu) against the reference.

k_td3_smooth is compared bit for bit with td3.py's default_target_policy_smoothing_func on
the same noise; k_td3_critic_loss's target bit for bit with the eager target expressions of
TD3 (n-step discount) and DDPG (gamma), its gradients bit for bit with torch's mse_loss
backward, and its losses and gradients against fp64 with bounds derived from the roundings
and the depth of the fp32 reduction."""
import ctypes
import os
import sys
from unittest import mock

import numpy as np
import pytest
import torch
from torch.nn import functional as F

sys.path.insert(0, os.path.dirname(__file__))
from soft_update_ref import bits  # noqa: E402

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
INF, NAN = float("inf"), float("nan")
SIZES = [1, 31, 32, 33, 255, 256, 257, 4097, 65536]
ROWS_PER_CTA = 1024  # B2RL_CRITIC_LOSS_ROWS_PER_CTA


def _same_bits(got, want, what=""):
    np.testing.assert_array_equal(bits(got), bits(want), err_msg=str(what))


# ---- k_td3_smooth ---------------------------------------------------------------------

def _smoothing_inputs(n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    action = (torch.rand(n, 6, generator=g, device="cuda") * 4 - 2)
    noise = torch.randn(n, 6, generator=g, device="cuda") * 3
    planted_a = torch.tensor([INF, -INF, NAN, 1.0, -1.0, 0.5, -0.5, 0.0, -0.0, 1.5, -1.5, 0.75],
                             device="cuda")
    # 0.2 * 2.5 = 0.5 rounds to the clamp bound; +-inf noise saturates; NaN noise stays NaN
    planted_e = torch.tensor([2.5, -2.5, 2.5000002, -2.4999998, INF, -INF, 0.0, -0.0, 1e30,
                              -1e30, NAN, 1.0], device="cuda")
    flat_a, flat_e = action.view(-1), noise.view(-1)
    k = min(flat_a.numel(), len(planted_a) * len(planted_e))
    ia = torch.arange(k, device="cuda")
    flat_a[:k] = planted_a[ia % len(planted_a)]
    flat_e[:k] = planted_e[(ia // len(planted_a)) % len(planted_e)]
    return action, noise


@pytest.mark.parametrize("n", [1, 17, 256, 4099])
def test_smoothing_is_bit_equal_to_the_default_function(n):
    from pfrl_b200.agents.td3 import default_target_policy_smoothing_func
    from pfrl_b200.ops.sac import td3_smooth

    action, noise = _smoothing_inputs(n, n)
    with mock.patch.object(torch, "randn_like", lambda x: noise):
        want = default_target_policy_smoothing_func(action)
    got = td3_smooth(action, noise)
    assert got.shape == want.shape and got.dtype == torch.float32
    _same_bits(got, want, n)
    if n >= 17:
        assert torch.isnan(want).any() and (want == 1).any() and (want == -1).any()
    fin = ~torch.isnan(want)
    assert ((got[fin] >= -1) & (got[fin] <= 1)).all()


def test_smoothing_refusals():
    from pfrl_b200.ops.sac import td3_smooth

    a = torch.zeros(4, 2, device="cuda")
    for bad in (a.double(), a.cpu(), torch.zeros(4, 3, device="cuda")):
        with pytest.raises(ValueError):
            td3_smooth(a, bad)
    with pytest.raises(ValueError):
        td3_smooth(a.cpu(), a.cpu())
    assert td3_smooth(a[:0], a[:0]).shape == (0, 2)


# ---- k_td3_critic_loss: target ---------------------------------------------------------

# (next_q1, next_q2) planted rows: NaN and inf heads, q1 < q2, q1 > q2, ties, signed zeros
_NEXT_ROWS = [(NAN, 1.0), (1.0, NAN), (NAN, NAN), (INF, 1.0), (1.0, -INF), (INF, INF),
              (-INF, 3.0), (1.0, 2.0), (2.0, 1.0), (1.5, 1.5), (-0.0, 0.0), (0.0, -0.0),
              (-7.25, -7.25), (3e38, 3e38)]


def _critic_inputs(n, seed, planted=True, td3=True):
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = torch.randn(n, generator=g, device="cuda") * 3
    disc = torch.tensor([0.0, 0.99, 0.99 ** 2, 0.99 ** 3], device="cuda")[
        torch.randint(0, 4, (n,), generator=g, device="cuda")]
    term = (torch.rand(n, generator=g, device="cuda") < 0.3).float()
    nq1 = torch.randn(n, 1, generator=g, device="cuda") * 10
    nq2 = torch.randn(n, 1, generator=g, device="cuda") * 10
    p1 = torch.randn(n, generator=g, device="cuda") * 10
    p2 = torch.randn(n, generator=g, device="cuda") * 10
    if planted:
        rows = torch.tensor(_NEXT_ROWS, device="cuda")
        k = min(n, len(_NEXT_ROWS))
        pos = torch.randperm(n, generator=g, device="cuda")[:k]
        nq1[pos, 0], nq2[pos, 0] = rows[:k, 0], rows[:k, 1]
        term[pos[: k // 2]] = 0.0
        disc[pos] = 0.99
    return r, disc, term, nq1, nq2, p1, p2


def _eager_td3_target(r, disc, term, nq1, nq2):
    """td3.py:181-236 on q [n, 1]."""
    return r + disc * (1.0 - term) * torch.flatten(torch.min(nq1, nq2))


def _eager_ddpg_target(r, gamma, term, nq):
    """ddpg.py:150-173."""
    return r + gamma * (1.0 - term) * nq.reshape((len(r),))


@pytest.mark.parametrize("n", [1, 14, 33, 1024, 1025, 4097])
def test_target_is_bit_equal_to_the_eager_expressions(n):
    from pfrl_b200.ops.sac import critic_loss

    r, disc, term, nq1, nq2, p1, p2 = _critic_inputs(n, n)
    got, _, _ = critic_loss(r, disc, term, nq1, nq2, p1, p2)
    want = _eager_td3_target(r, disc, term, nq1, nq2)
    _same_bits(got, want, ("td3", n))
    if n >= len(_NEXT_ROWS):
        assert torch.isnan(want).sum() >= 3 and torch.isinf(want).any()
    for gamma in (0.99, 1 / 3, 0.0, 1.0):
        got, _, _ = critic_loss(r, gamma, term, nq1, None, p1, None)
        _same_bits(got, _eager_ddpg_target(r, gamma, term, nq1), ("ddpg", n, gamma))


# ---- losses and gradients ----------------------------------------------------------------

def _reduction_depth(n):
    """Longest chain of fp32 additions behind one loss: 4 rows per thread, 5 warp shuffles,
    8 warp sums, then over the CTA sums (ceil(ctas / 256) per thread, 5 + 7 again)."""
    ctas = -(-n // ROWS_PER_CTA)
    depth = 4 + 5 + 7
    if ctas > 1:
        depth += -(-ctas // 256) + 5 + 7
    return depth


@pytest.mark.parametrize("n", SIZES)
def test_losses_and_gradients_against_fp64(n):
    from pfrl_b200.ops.sac import critic_loss

    r, disc, term, nq1, nq2, p1, p2 = _critic_inputs(n, n + 1, planted=False)
    for twin in (True, False):
        q1 = p1.clone().requires_grad_()
        q2 = p2.clone().requires_grad_() if twin else None
        y, l1, l2 = critic_loss(r, disc, term, nq1, nq2 if twin else None, q1, q2)
        (l1 + (l2 if twin else 0)).backward()
        # against torch's mse_loss backward on the kernel's (bit-exact) target
        for q, p in ((q1, p1), (q2, p2))[: 2 if twin else 1]:
            ref = p.clone().requires_grad_()
            F.mse_loss(y, ref).backward()
            _same_bits(q.grad, ref.grad, (n, twin))
        # against fp64: the loss is a sum of n squares, each off by at most 3U relative
        # (difference, square), summed over `depth` fp32 additions, then divided once
        depth = _reduction_depth(n)
        for q, p, loss in ((q1, p1, l1), (q2, p2, l2))[: 2 if twin else 1]:
            d64 = p.double() - y.double()
            sq = d64 * d64
            exact = float(sq.sum()) / n
            bound = ((1 + U) ** (3 + depth + 1) - 1) * float(sq.sum()) / n * 1.0001
            got = float(loss.detach())
            assert abs(got - exact) <= bound, (n, twin, got, exact, bound)
            g_exact = 2.0 / n * d64
            g_err = (q.grad.double() - g_exact).abs()
            assert (g_err <= 3.0001 * U * g_exact.abs() + 2.0 ** -149).all(), (n, twin)


def test_two_launches_give_the_same_bits():
    from pfrl_b200.ops.sac import critic_loss

    r, disc, term, nq1, nq2, p1, p2 = _critic_inputs(65536, 5, planted=False)
    outs = []
    for _ in range(2):
        q1, q2 = p1.clone().requires_grad_(), p2.clone().requires_grad_()
        y, l1, l2 = critic_loss(r, disc, term, nq1, nq2, q1, q2)
        (l1 + l2).backward()
        outs.append([y, l1.detach(), l2.detach(), q1.grad, q2.grad])
    for a, b in zip(*outs):
        _same_bits(a, b)


def test_critic_loss_refusals():
    from pfrl_b200.ops.sac import critic_loss

    r, disc, term, nq1, nq2, p1, p2 = _critic_inputs(64, 0)
    good = (r, disc, term, nq1, nq2, p1, p2)
    for i in range(len(good)):
        for bad in (good[i].double(), good[i].cpu(), good[i][:-1]):
            args = list(good)
            args[i] = bad
            with pytest.raises(ValueError):
                critic_loss(*args)
    e = r[:0]
    with pytest.raises(ValueError):
        critic_loss(e, disc[:0], e, nq1[:0], nq2[:0], e, e)
    with pytest.raises(ValueError):
        critic_loss(e, 0.99, e, nq1[:0], None, e, None)


def test_critic_loss_abi_refusals():
    """Bad arguments are refused on the host before a launch: nothing is written."""
    from pfrl_b200 import _lib

    L = _lib.load()
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    n = 2 * ROWS_PER_CTA
    buf = torch.zeros(16, n, device="cuda")
    buf[:8] = 1.0  # inputs; rows 8.. are outputs and scratch
    p = [ctypes.c_void_p(buf[i].data_ptr()) for i in range(16)]

    def call(nn=n, pred2=p[7], grad2=p[10], loss2=p[12], partial=p[13], reward=p[0]):
        return L.b2rl_td3_critic_loss(reward, p[1], 0.99, p[2], p[3], p[4], p[5], pred2, nn,
                                      p[8], p[9], grad2, p[11], loss2, partial, stream)

    invalid, out_of_range = -1, -4  # B2RL_ERR_INVALID, B2RL_ERR_RANGE
    assert call(reward=None) == invalid
    assert call(grad2=None) == invalid
    assert call(loss2=None) == invalid
    assert call(partial=None) == invalid
    assert call(nn=0) == out_of_range
    assert call(nn=-5) == out_of_range
    with pytest.raises(_lib.B2rlError):
        _lib.check(call(nn=0))
    assert L.b2rl_td3_smooth(p[8], p[9], 0, p[10], stream) == out_of_range
    assert L.b2rl_td3_smooth(None, p[9], 4, p[10], stream) == invalid
    torch.cuda.synchronize()
    assert not buf[8:].any()
    assert call() == 0  # terminal rows: target = reward = 1
    torch.cuda.synchronize()
    assert torch.equal(buf[8], torch.ones(n, device="cuda"))
