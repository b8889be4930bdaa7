"""A3C's loss gradient (csrc/a3c.cu) behind torch.

``loss_grads`` launches the kernel for CUDA tensors.  For CPU tensors it runs the same
arithmetic as torch operations (``loss_grads_torch``), so that it can be checked on a
machine without a GPU; the agent itself only takes the fused path on CUDA.
"""
import numpy as np
import torch

from pfrl_b200 import _lib
from pfrl_b200.ops.ppo import _f32, _p, _stream
from pfrl_b200.ops.reinforce import row_grads_torch


def returns_scan(rewards, bootstrap, gamma):
    """The reference's returns: ``R = bootstrap`` (0 when None), then ``R = R * gamma + r``
    from the last step back, in fp64 with each operation rounded (Python floats), rounded to
    fp32 at the end."""
    R = 0.0 if bootstrap is None else float(bootstrap)
    out = []
    for r in reversed(np.asarray(rewards, dtype=np.float64).tolist()):
        R = R * float(gamma) + r
        out.append(R)
    return np.asarray(out[::-1], dtype=np.float32)


def coefficients(R32, v, beta, pi_factor, v_factor):
    """The fp32 gradients the reference's backward hands log pi(a), H and v of each row:
    ``(c_lp [N], c_h, g_v [N])`` with c_lp = fl32(pf * -adv), c_h = -fl32(pf * fl32(beta)) and
    g_v = fl32(fl32(2 * fl32(v - R)) * fl32(vf / 2)), adv = fl32(R - v)."""
    pf, vf = np.float32(pi_factor), np.float32(v_factor)
    R32 = torch.as_tensor(R32, dtype=torch.float32, device=v.device)
    v = _f32(v).reshape(-1)
    c_lp = (R32 - v).neg() * pf
    c_h = -(pf * np.float32(beta))
    g_v = (v - R32) * np.float32(2) * (vf / np.float32(2))
    return c_lp, float(c_h), g_v


def loss_grads_torch(v, rewards, bootstrap, gamma, beta, pi_factor, v_factor, *, z=None,
                     actions=None, loc=None, scale=None, action_values=None):
    """The kernel's arithmetic, stored in fp32: the fp64 scan on the host, the fp32
    coefficients, then fp64 torch operations."""
    boot = None if bootstrap is None else float(bootstrap.reshape(()))
    R32 = returns_scan(torch.as_tensor(rewards).cpu().numpy(), boot, gamma)
    c_lp, c_h, g_v = coefficients(R32, v, beta, pi_factor, v_factor)
    grads, lp, h = row_grads_torch(c_lp.double(), c_h, z=z, actions=actions, loc=loc,
                                   scale=scale, action_values=action_values)
    R = torch.as_tensor(R32, device=v.device)
    adv = (R - _f32(v).reshape(-1)).double()
    pf = float(np.float32(pi_factor))
    pi_loss = ((-adv * lp - float(np.float32(beta)) * h) * pf).float().sum()
    d = (_f32(v).reshape(-1) - R).double()
    v_loss = (d * d * 0.5 * float(np.float32(v_factor))).float().sum()
    return grads, g_v, R, pi_loss, v_loss


def loss_grads(v, rewards, bootstrap, gamma, beta, pi_factor, v_factor, *, z=None,
               actions=None, loc=None, scale=None, action_values=None, scale_grad=True,
               want_loss=False):
    """d loss / d(distribution parameters) and d loss / d v for A3C's loss over N rows,
    ``pi_factor * sum(-adv log pi(a) - beta H) + v_factor * sum((v - R)^2) / 2``.

    A Categorical: ``z`` [N, K] (``Categorical._param``) and int64 ``actions`` [N]; the
    grads are ``(g_z,)``.  An ``Independent(Normal, 1)``: ``loc`` [N, A], ``scale`` [N, A]
    or None (= 1) and the sampled ``action_values`` [N, A]; the grads are
    ``(g_loc, g_scale)``, g_scale None when ``scale_grad`` is false.  ``v`` [N] or [N, 1]
    fp32, ``rewards`` fp64 [N], ``bootstrap`` a one-element fp32 device tensor or None
    (terminal).  Returns ``(grads, g_v [N], returns [N] fp32, pi_loss, v_loss)``, the last
    two fp32 device scalars with ``want_loss`` and None otherwise."""
    if not v.is_cuda:
        grads, g_v, R, pi_loss, v_loss = loss_grads_torch(
            v, rewards, bootstrap, gamma, beta, pi_factor, v_factor, z=z, actions=actions,
            loc=loc, scale=scale, action_values=action_values)
        if z is None and not scale_grad:
            grads = (grads[0], None)
        if not want_loss:
            pi_loss = v_loss = None
        return grads, g_v, R, pi_loss, v_loss
    L = _lib.load()
    v = _f32(v).reshape(-1)
    N = v.shape[0]
    dev = v.device
    rewards = rewards.detach().to(torch.float64).reshape(N).contiguous()
    if bootstrap is not None:
        bootstrap = _f32(bootstrap).reshape(1)
    if z is not None:
        z = _f32(z)
        D = z.shape[1]
        assert z.shape == (N, D), "z must be [%d, K], got %s" % (N, tuple(z.shape))
        actions = actions.detach().to(torch.int64).reshape(N).contiguous()
        g_z = torch.empty((N, D), dtype=torch.float32, device=dev)
        grads = (g_z,)
        ptrs = (_p(z), None, None, _p(actions), None, _p(g_z), None, None)
    else:
        loc = _f32(loc)
        D = loc.shape[1]
        assert loc.shape == (N, D), "loc must be [%d, A], got %s" % (N, tuple(loc.shape))
        if scale is not None:
            scale = _f32(scale.expand(N, D))
        action_values = _f32(action_values).reshape(N, D)
        g_loc = torch.empty((N, D), dtype=torch.float32, device=dev)
        g_scale = torch.empty((N, D), dtype=torch.float32, device=dev) if scale_grad else None
        grads = (g_loc, g_scale)
        ptrs = (None, _p(loc), _p(scale), None, _p(action_values), None, _p(g_loc), _p(g_scale))
    # g_v, R, and each row's pi_loss and v_loss terms
    out = torch.empty((4 if want_loss else 2, N), dtype=torch.float32, device=dev)
    terms = (_p(out[2]), _p(out[3])) if want_loss else (None, None)
    z_p, loc_p, scale_p, act_p, val_p, gz_p, gloc_p, gscale_p = ptrs
    with torch.cuda.device(dev):  # the stream of the tensors' device, not the current one
        _lib.check(L.b2rl_a3c_loss(
            N, D, z_p, loc_p, scale_p, act_p, val_p, _p(v), _p(rewards), _p(bootstrap),
            float(gamma), float(beta), float(pi_factor), float(v_factor), gz_p, gloc_p,
            gscale_p, _p(out[0]), _p(out[1]), *terms, _stream()))
    if want_loss:
        return grads, out[0], out[1], out[2].sum(), out[3].sum()
    return grads, out[0], out[1], None, None
