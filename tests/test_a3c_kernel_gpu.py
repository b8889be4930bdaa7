"""GPU: b2rl_a3c_loss (csrc/a3c.cu) against an fp64 restatement per element, with a bound
derived per element, and against torch's autograd of the reference's expression on the same
GPU.  Returns are bit for bit the Python fp64 scan rounded to fp32."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from test_a3c_cpu import fused_call, make_rows, reference_loss  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
EPS32 = float(np.finfo(np.float32).eps)


def fp64_grads(dist, v, actions, R32, beta, pf, vf):
    """The kernel's contract in fp64 from its fp32 coefficients: (policy grads, g_v)."""
    from pfrl_b200.ops.a3c import coefficients
    from pfrl_b200.ops.reinforce import row_grads_torch

    c_lp, c_h, g_v = coefficients(R32, v.detach(), beta, pf, vf)
    if type(dist) is torch.distributions.Categorical:
        kw = dict(z=dist._param, actions=actions)
    else:
        kw = dict(loc=dist.base_dist.loc, scale=dist.base_dist.scale, action_values=actions)
    kw = {k: x.detach().cpu() for k, x in kw.items()}
    # row_grads_torch's arithmetic without the final fp32 rounding
    fmin = torch.finfo(torch.float32).min
    c_lp = c_lp.double().cpu()
    if "z" in kw:
        z = kw["z"].double()
        p = torch.softmax(z, 1)
        c = z.clamp(min=fmin)
        h = -(p * c).sum(1)
        g = c_h * (-p * ((z >= fmin).double() + c + h[:, None]))
        g.scatter_add_(1, kw["actions"].reshape(-1, 1).long(), c_lp[:, None])
        return [g], g_v.cpu()
    loc = kw["loc"].double()
    s = kw["scale"].double().expand_as(loc)
    d = kw["action_values"].double() - loc
    inv = 1.0 / s
    return [c_lp[:, None] * d * inv * inv,
            c_lp[:, None] * (d * d * inv ** 3 - inv) + c_h * inv], g_v.cpu()


SIZES_N = [1, 2, 5, 31, 32, 33, 257, 4096]
SIZES_D = [1, 2, 18, 31, 33, 1024]


@pytest.mark.parametrize("N", SIZES_N)
@pytest.mark.parametrize("D", SIZES_D)
@pytest.mark.parametrize("discrete", [True, False])
def test_kernel_against_fp64_and_the_reference(N, D, discrete):
    if N * D > 300000:
        D = max(1, 300000 // N)
    rng = np.random.RandomState(N * 7 + D)
    gamma = [0.0, 0.99, 1.0][(N + D) % 3]
    bootstrap = None if (N + D) % 2 else float(np.float32(rng.randn()))
    beta, pf, vf = 0.013, 5 / 3, 0.5 * 5 / 3
    rewards = list(rng.randn(N) * 3)
    dist, leaves, v, actions = make_rows(rng, N, D, discrete, device=DEV)
    grads, g_v, R, _, _ = fused_call(dist, v, actions, rewards, bootstrap, gamma, beta, pf,
                                     vf)
    torch.cuda.synchronize()
    # returns: bit for bit the Python scan
    from pfrl_b200.ops.a3c import returns_scan

    want_R = returns_scan(rewards, bootstrap, gamma)
    assert np.array_equal(R.cpu().numpy().view(np.uint32), want_R.view(np.uint32))
    # against fp64: fp64 below the fp32 coefficients, one fp32 rounding at the store
    want, want_gv = fp64_grads(dist, v, actions, want_R, beta, pf, vf)
    assert torch.equal(g_v.cpu(), want_gv)
    for g, w in zip(grads, want):
        bound = 4 * EPS32 * w.abs() + 1e-12 * (1 + w.abs().max())
        assert ((g.cpu().double() - w).abs() <= bound).all()
    # against torch's autograd of the reference's expression on the GPU
    _, loss = reference_loss(dist, v, actions, rewards, bootstrap, gamma, beta, pf, vf)
    loss.backward()
    assert torch.equal(g_v, v.grad.reshape(-1))
    for leaf, g in zip(leaves, grads):
        ref = leaf.grad
        tol = 1e-5 * (1 + ref.abs().max())
        assert (g - ref).abs().max() <= tol


def test_logits_at_finfo_min_and_absent_scale():
    rng = np.random.RandomState(0)
    N, K = 9, 6
    dist, _, v, actions = make_rows(rng, N, K, True, device=DEV)
    z = dist._param.detach().clone()
    z[:, 0] = torch.finfo(torch.float32).min
    actions = torch.full((N,), 1, device=DEV)
    d2 = torch.distributions.Categorical(logits=z)
    (g_z,), g_v, R, _, _ = fused_call(d2, v, actions, list(rng.randn(N)), None, 0.9, 0.5,
                                      1.0, 0.5)
    want, _ = fp64_grads(d2, v, actions, R.cpu().numpy(), 0.5, 1.0, 0.5)
    assert torch.isfinite(g_z).all()
    np.testing.assert_allclose(g_z.cpu().numpy(), want[0].numpy(), rtol=1e-6, atol=1e-7)
    # an Independent(Normal) with scale 1 given as None
    dist, leaves, v, act = make_rows(rng, N, 3, False, device=DEV, scale=False)
    from pfrl_b200.ops import a3c as fused

    r = torch.as_tensor(rng.randn(N), device=DEV)
    (g_loc, g_scale), _, _, _, _ = fused.loss_grads(v, r, None, 0.9, 0.1, 1.0, 0.5,
                                                    loc=dist.base_dist.loc, scale=None,
                                                    action_values=act, scale_grad=False)
    assert g_scale is None
    (g_loc2, _), _, _, _, _ = fused.loss_grads(
        v, r, None, 0.9, 0.1, 1.0, 0.5, loc=dist.base_dist.loc,
        scale=torch.ones(N, 3, device=DEV), action_values=act)
    assert torch.equal(g_loc, g_loc2)


def test_loss_terms_against_the_reference():
    rng = np.random.RandomState(3)
    for discrete in (True, False):
        dist, _, v, actions = make_rows(rng, 5, 4, discrete, device=DEV)
        rewards = list(rng.randn(5))
        _, _, _, pi_loss, v_loss = fused_call(dist, v, actions, rewards, 0.25, 0.99, 0.01,
                                              1.0, 0.5, want_loss=True)
        _, loss = reference_loss(dist, v, actions, rewards, 0.25, 0.99, 0.01, 1.0, 0.5)
        np.testing.assert_allclose(float(pi_loss + v_loss), float(loss), rtol=1e-5, atol=1e-6)
