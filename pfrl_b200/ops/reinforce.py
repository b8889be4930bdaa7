"""REINFORCE's loss gradient (csrc/reinforce.cu) behind torch.

``loss_grads`` launches the kernel for CUDA tensors.  For CPU tensors it runs the same
arithmetic as torch operations (``loss_grads_torch``), so that the agent's recompute
path can be exercised on a machine without a GPU; the agent itself only takes that path
on CUDA.
"""
import numpy as np
import torch

from pfrl_b200 import _lib
from pfrl_b200.ops.ppo import _f32, _p, _stream


def _coefs(R, batchsize, beta):
    """The fp32 gradients the reference's backward hands log pi(a) and H of each row:
    fl32(fl32(1 / bs) * fl32(-R)) and -fl32(fl32(1 / bs) * fl32(beta))."""
    inv_bs = torch.tensor(np.float32(1) / np.float32(batchsize), dtype=torch.float32)
    c_lp = inv_bs.to(R.device) * -R
    c_h = -(inv_bs * torch.tensor(np.float32(beta), dtype=torch.float32))
    return c_lp.double(), float(c_h)


def row_grads_torch(c_lp, c_h, *, z=None, actions=None, loc=None, scale=None,
                    action_values=None):
    """Given the gradients ``c_lp`` [N] (fp64) and ``c_h`` (a float) that a loss hands
    log pi(a) and H of each row, the rows' d loss / d(distribution parameters) in fp64 torch
    operations, stored in fp32: ``(grads, lp, h)`` with ``grads`` ``(g_z,)`` or
    ``(g_loc, g_scale)`` and the rows' fp64 log pi(a) and H."""
    fmin = torch.finfo(torch.float32).min
    if z is not None:
        z = z.detach().double()
        p = torch.softmax(z, dim=1)
        c = z.clamp(min=fmin)
        h = -(p * c).sum(1)
        dh = -p * ((z >= fmin).double() + c + h[:, None])
        g = c_h * dh
        a = actions.reshape(-1, 1).long()
        g.scatter_add_(1, a, c_lp[:, None])
        out = (g.float(),)
        lp = z.gather(1, a)[:, 0]
    else:
        loc = loc.detach().double()
        s = torch.ones_like(loc) if scale is None else scale.detach().double().expand_as(loc)
        d = action_values.detach().double() - loc
        inv_s = 1.0 / s
        g_loc = c_lp[:, None] * d * inv_s * inv_s
        g_scale = c_lp[:, None] * (d * d * inv_s ** 3 - inv_s) + c_h * inv_s
        out = (g_loc.float(), g_scale.float())
        half_log_2pi = 0.5 * np.log(2 * np.pi)
        lp = (-(d * d) * 0.5 * inv_s * inv_s - s.log() - half_log_2pi).sum(1)
        h = (0.5 + half_log_2pi + s.log()).sum(1)
    return out, lp, h


def loss_grads_torch(R, batchsize, beta, *, z=None, actions=None, loc=None, scale=None,
                     action_values=None, want_loss=False):
    """The kernel's arithmetic in fp64 torch operations, stored in fp32."""
    c_lp, c_h = _coefs(_f32(R).reshape(-1), batchsize, beta)
    out, lp, h = row_grads_torch(c_lp, c_h, z=z, actions=actions, loc=loc, scale=scale,
                                 action_values=action_values)
    if want_loss:
        Rd = _f32(R).reshape(-1).double()
        inv_bs = float(np.float32(1) / np.float32(batchsize))
        row_loss = ((-Rd * lp - float(np.float32(beta)) * h) * inv_bs).float()
        return out + (row_loss.sum(), h.float().sum())
    return out


def loss_grads(R, batchsize, beta, *, z=None, actions=None, loc=None, scale=None,
               action_values=None, scale_grad=True, want_loss=False):
    """d loss / d(distribution parameters) for loss = sum_rows(-R log pi(a) - beta H) /
    batchsize over N rows.

    A Categorical: ``z`` [N, K] (``Categorical._param``) and int64 ``actions`` [N]; returns
    ``(g_z,)``.  An ``Independent(Normal, 1)``: ``loc`` [N, A], ``scale`` [N, A] or None
    (= 1) and the sampled ``action_values`` [N, A]; returns ``(g_loc, g_scale)``, g_scale
    None when ``scale_grad`` is false.  ``R`` [N] fp32.  With ``want_loss``, the fp32 loss
    and the sum of the rows' entropies follow (device scalars)."""
    if not R.is_cuda:
        out = loss_grads_torch(R, batchsize, beta, z=z, actions=actions, loc=loc, scale=scale,
                               action_values=action_values, want_loss=want_loss)
        if z is None and not scale_grad:
            out = (out[0], None) + out[2:]
        return out
    L = _lib.load()
    R = _f32(R).reshape(-1)
    N = R.shape[0]
    dev = R.device
    if z is not None:
        z = _f32(z)
        D = z.shape[1]
        assert z.shape == (N, D), "z must be [%d, K], got %s" % (N, tuple(z.shape))
        actions = actions.detach().to(torch.int64).reshape(N).contiguous()
        g_z = torch.empty((N, D), dtype=torch.float32, device=dev)
        outs = (g_z,)
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
        outs = (g_loc, g_scale)
        ptrs = (None, _p(loc), _p(scale), None, _p(action_values), None, _p(g_loc), _p(g_scale))
    rows = torch.empty((2, N), dtype=torch.float32, device=dev) if want_loss else None
    z_p, loc_p, scale_p, act_p, val_p, gz_p, gloc_p, gscale_p = ptrs
    with torch.cuda.device(dev):  # the stream of the tensors' device, not the current one
        _lib.check(L.b2rl_reinforce_loss(
            N, D, z_p, loc_p, scale_p, act_p, val_p, _p(R), int(batchsize), float(beta), gz_p,
            gloc_p, gscale_p, _p(rows[0]) if want_loss else None,
            _p(rows[1]) if want_loss else None, _stream()))
    if want_loss:
        return outs + (rows[0].sum(), rows[1].sum())
    return outs
