"""NAF ops (csrc/naf.cu) as torch.autograd Functions: the head that turns the raw linear
outputs into P = L L^T, and the TD loss of the DQN family with a ``QuadraticActionValue``.
Inputs are fp32 CUDA tensors; there is no CPU path here -- the Q-function and the agents use
the reference's torch formulation on CPU."""
import torch

from pfrl_b200 import _lib
from pfrl_b200.ops.losses import _f32, _p, _stream

# target of each agent (include/b2rl.h): the advantage-learning values where they are shared
NAF_MODES = {"al": 0, "pal": 1, "double_pal": 2, "dpp_greedy": 5, "dqn": 6, "double_dqn": 7}


class _NafHead(torch.autograd.Function):
    @staticmethod
    def forward(ctx, diag_pre, non_diag):
        L = _lib.load()
        B, n = diag_pre.shape
        dp = _f32(diag_pre)
        nd = None if non_diag is None else _f32(non_diag)
        mat = torch.empty((B, n, n), dtype=torch.float32, device=dp.device)
        _lib.check(L.b2rl_naf_head_fwd(_p(dp), _p(nd), B, n, _p(mat), _stream()))
        ctx.save_for_backward(dp, nd if nd is not None else torch.empty(0, device=dp.device))
        ctx.has_nd = nd is not None
        return mat

    @staticmethod
    def backward(ctx, grad_mat):
        L = _lib.load()
        dp, nd = ctx.saved_tensors
        B, n = dp.shape
        g_dp = torch.empty_like(dp)
        g_nd = torch.empty_like(nd) if ctx.has_nd else None
        _lib.check(L.b2rl_naf_head_bwd(_p(dp), _p(nd) if ctx.has_nd else None,
                                       _p(_f32(grad_mat)), B, n, _p(g_dp), _p(g_nd), _stream()))
        return g_dp, g_nd


def head(diag_pre, non_diag=None):
    """P = L L^T [B, n, n] with L's diagonal exp(diag_pre) [B, n] and the entries below it
    ``non_diag`` [B, n(n-1)/2] in np.tril_indices(n, -1) order (None when n = 1)."""
    return _NafHead.apply(diag_pre, non_diag)


def _bound(b, n):
    """A bound of QuadraticActionValue ([n] or [1] tensor, or None) as [n] fp32 contiguous."""
    return None if b is None else _f32(b).reshape(-1).expand(n).contiguous()


class _NafTdLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, mu, mat, v, action, tq, tnq, nq, reward, discount, terminal, weights,
                mode, alpha, clip_delta, mean):
        L = _lib.load()
        B, n = mu.shape
        dev = mu.device
        muc, matc, vc = _f32(mu), _f32(mat), _f32(v)
        act = _f32(action).reshape(B, n)
        w = None if weights is None else _f32(weights)
        t_mu = t_mat = t_v = n_mu = None
        if tq is not None:
            t_mu, t_mat, t_v = _f32(tq.mu), _f32(tq.mat), _f32(tq.v)
        if nq is not None:
            n_mu = _f32(nq.mu)
        tn_mu, tn_mat, tn_v = _f32(tnq.mu), _f32(tnq.mat), _f32(tnq.v)
        lo, hi = _bound(tnq.min_action, n), _bound(tnq.max_action, n)
        nlo = _bound(nq.min_action, n) if nq is not None else None
        nhi = _bound(nq.max_action, n) if nq is not None else None
        y = torch.empty(B, dtype=torch.float32, device=dev)
        t = torch.empty(B, dtype=torch.float32, device=dev)
        delta = torch.empty(B, dtype=torch.float32, device=dev)
        scratch = torch.empty(B, dtype=torch.float32, device=dev)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        _lib.check(L.b2rl_naf_td_loss_fwd(
            NAF_MODES[mode], _p(muc), _p(matc), _p(vc), _p(act), _p(t_mu), _p(t_mat), _p(t_v),
            _p(tn_mu), _p(tn_mat), _p(tn_v), _p(n_mu), _p(lo), _p(hi), _p(nlo), _p(nhi),
            _p(_f32(reward)), _p(_f32(discount)), _p(_f32(terminal)), _p(w), B, n, float(alpha),
            int(clip_delta), int(mean), _p(y), _p(t), _p(delta), _p(scratch), _p(loss),
            _stream()))
        ctx.save_for_backward(muc, matc, act, y, t,
                              w if w is not None else torch.empty(0, device=dev))
        ctx.has_w = w is not None
        ctx.cfg = (B, n, int(clip_delta), int(mean))
        ctx.mark_non_differentiable(delta, y, t)
        return loss, delta, y, t

    @staticmethod
    def backward(ctx, g_loss, *unused):
        L = _lib.load()
        mu, mat, act, y, t, w = ctx.saved_tensors
        B, n, clip_delta, mean = ctx.cfg
        g_mu, g_mat = torch.empty_like(mu), torch.empty_like(mat)
        g_v = torch.empty(B, dtype=torch.float32, device=mu.device)
        _lib.check(L.b2rl_naf_td_loss_bwd(
            _p(mu), _p(mat), _p(act), _p(y), _p(t), _p(w) if ctx.has_w else None,
            _p(_f32(g_loss).reshape(1)), B, n, clip_delta, mean, _p(g_mu), _p(g_mat), _p(g_v),
            _stream()))
        return (g_mu, g_mat, g_v) + (None,) * 12


def td_loss(qout, action, target_next, reward, discount, terminal, weights, mode, target=None,
            next_online=None, alpha=0.0, clip_delta=True, mean=True):
    """TD loss of a DQN-family agent whose Q-function returns ``QuadraticActionValue``.

    ``qout``: the online net at s (the only one that gets a gradient); ``target`` and
    ``target_next``: the target net at s and s'; ``next_online``: the online net at s'.
    ``mode`` is one of ``NAF_MODES``: "dqn", "double_dqn" (needs ``next_online``), "al",
    "pal", "double_pal" (needs ``next_online``) and "dpp_greedy"; all but the DQN modes need
    ``target``.  Returns (loss, |y - t|, y, t)."""
    B = qout.mu.shape[0]
    return _NafTdLoss.apply(qout.mu, qout.mat, qout.v.reshape(B), action, target, target_next,
                            next_online, reward, discount, terminal, weights, mode, alpha,
                            clip_delta, mean)
