"""b2rl_acer_loss (csrc/acer.cu) against the fp64 closed form (oracle/acer_closed_form.py),
per element.

Both sides read the same fp32 inputs and compute in fp64; the kernel stores fp32.  So
each element may differ by the fp32 rounding of the result (2^-24 relative, bounded here
by 2^-23) plus fp64 reassociation of sums whose terms are larger than the result
(bounded by 1e-12 of the largest element of the row's terms).  The Q gradient's target is
the fp32 rounding of Q_ret, which fp64 reassociation can move by one fp32 ulp of Q_ret."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.acer_closed_form import acer_loss_grads  # noqa: E402

pytestmark = pytest.mark.gpu
EPS32 = 2.0 ** -23


def _inputs(T, K, seed, degenerate=False, tied_q=False):
    rng = np.random.RandomState(seed)
    z = (rng.randn(T, K) * 2).astype(np.float32)
    if degenerate:
        z[0, :2] = [1e10, 1e-10]
        if T > 1:
            z[-1, :2] = [1e-10, 1e10]
    z = torch.distributions.Categorical(logits=torch.tensor(z)).logits.numpy()
    q = (np.full((T, K), 0.5) if tied_q else rng.randn(T, K)).astype(np.float32)
    avg = (z + 0.3 * rng.randn(T, K)).astype(np.float32)
    mu = (z + 0.5 * rng.randn(T, K)).astype(np.float32)
    a = rng.randint(K, size=T)
    if degenerate:
        a[0] = 0
    r = rng.randn(T)
    return z, q, avg, mu, a, r


def _check(T, K, cfg, seed=0, on_policy=False, bootstrap=0.7, **kind):
    from pfrl_b200.ops import acer as fused

    z, q, avg, mu, a, r = _inputs(T, K, seed, **kind)
    dev = torch.device("cuda:0")
    kl0 = 0.125
    avg_kl = torch.tensor([kl0], dtype=torch.float64, device=dev)
    g_z, g_q = fused.loss_grads(
        torch.tensor(z, device=dev), torch.tensor(q, device=dev), torch.tensor(a, device=dev),
        torch.tensor(r, device=dev), avg_z=torch.tensor(avg, device=dev),
        mu_z=None if on_policy else torch.tensor(mu, device=dev),
        bootstrap=None if bootstrap is None else torch.tensor(bootstrap, device=dev),
        average_kl=avg_kl, **cfg)
    # the kernel reads the bootstrap value as the fp32 device scalar it is
    boot32 = None if bootstrap is None else float(np.float32(bootstrap))
    want_z, want_q, want_kl = acer_loss_grads(
        z, q, a, r, avg_z=avg, mu_z=None if on_policy else mu, bootstrap=boot32,
        average_kl=kl0, **cfg)
    got_z, got_q = g_z.double().cpu().numpy(), g_q.double().cpu().numpy()
    for got, want in ((got_z, want_z), (got_q, want_q)):
        assert np.array_equal(np.isnan(got), np.isnan(want))
    ok = ~np.isnan(want_z)
    scale = np.nanmax(np.abs(want_z), axis=1, keepdims=True) + 1.0
    bound = EPS32 * np.abs(want_z) + 1e-12 * scale * (1 + abs(cfg["delta"]))
    err = np.abs(got_z - want_z)
    assert (err[ok] <= bound[ok]).all(), float(np.max((err - bound)[ok]))
    # one fp32 ulp of the target: cq |Q_ret| <= cq |Q| + |g_q|
    cq = cfg["Q_loss_coef"] / (T if cfg["normalize_loss_by_steps"] else 1)
    q_bound = EPS32 * (2 * np.abs(want_q) + cq * np.abs(q))
    assert (np.abs(got_q - want_q) <= q_bound).all()
    if cfg["use_trust_region"]:
        got_kl = float(avg_kl.item())
        if np.isnan(want_kl):
            assert np.isnan(got_kl)
        else:
            assert got_kl == pytest.approx(want_kl, rel=1e-12, abs=1e-300)
    else:
        assert float(avg_kl.item()) == kl0


def _cfg(c=10, tr=True, delta=1.0, **over):
    cfg = dict(gamma=0.99, truncation_threshold=c, use_trust_region=tr, delta=delta, beta=0.01,
               pi_loss_coef=1.0, Q_loss_coef=0.5, normalize_loss_by_steps=True,
               use_Q_opc=False, average_kl_decay=0.99)
    cfg.update(over)
    return cfg


@pytest.mark.parametrize("K", [2, 4, 18, 33, 1024])
@pytest.mark.parametrize("T", [1, 2, 5, 33, 257, 2049])
def test_shapes(T, K):
    _check(T, K, _cfg(), seed=T * 7 + K)
    _check(T, K, _cfg(c=None, tr=False), seed=T + K, on_policy=True, bootstrap=None)


@pytest.mark.parametrize("on_policy", [False, True])
@pytest.mark.parametrize("c", [None, 0, 1, 10, np.inf])
@pytest.mark.parametrize("delta", [0.0, 1.0])
@pytest.mark.parametrize("tr", [False, True])
def test_modes(on_policy, c, delta, tr):
    _check(5, 18, _cfg(c=c, tr=tr, delta=delta), seed=3, on_policy=on_policy)
    _check(33, 4, _cfg(c=c, tr=tr, delta=delta), seed=4, on_policy=on_policy, bootstrap=None)


@pytest.mark.parametrize("c", [None, 0, 1, 10, np.inf])
@pytest.mark.parametrize("tr", [False, True])
def test_degenerate_logits_and_tied_q(c, tr):
    _check(4, 2, _cfg(c=c, tr=tr), seed=5, degenerate=True)
    _check(6, 18, _cfg(c=c, tr=tr), seed=6, degenerate=True, tied_q=True)


@pytest.mark.parametrize("over", [dict(use_Q_opc=True), dict(normalize_loss_by_steps=False),
                                  dict(pi_loss_coef=0.3, Q_loss_coef=2.0, beta=0.0)])
def test_options(over):
    _check(33, 18, _cfg(**over), seed=8)
    _check(5, 4, _cfg(tr=False, **over), seed=9, bootstrap=None)


def test_invalid_arguments_are_refused():
    from pfrl_b200 import _lib

    L = _lib.load()
    assert L.b2rl_acer_loss(0, 4, *([None] * 7), 0.9, 0, 0.0, 0, 0.0, 0.0, 1.0, 1.0, 1, 0,
                            None, 0.0, None, None, None, None) != 0
