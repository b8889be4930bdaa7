"""TRPO kernels (csrc/trpo.cu) behind torch: the surrogate objective as an autograd
Function, the Fisher metric product, the conjugate-gradient steps and the line-search
decision.  Distribution kinds: GAUSSIAN = Independent(Normal(loc, scale), 1) with params
(loc, scale) [N, A]; CATEGORICAL = Categorical with params (logits,) [N, K]."""
import torch

from pfrl_b200 import _lib
from pfrl_b200.ops.ppo import _f32, _p, _stream

GAUSSIAN, CATEGORICAL = 0, 1


def _cuda(t):
    """``t`` as an fp32 contiguous CUDA tensor (a copy if it is not one already)."""
    assert t.is_cuda, "the TRPO kernels take CUDA tensors"
    return _f32(t)


def _buffer(t, name):
    """A tensor a kernel writes in place: it must already be fp32, contiguous and on CUDA,
    since a converted copy would take the write."""
    assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous(), \
        "%s must be a contiguous fp32 CUDA tensor, got %s %s" % (name, t.dtype, t.device)
    return t


def _rows(t, N):
    return _cuda(t).reshape(N, -1)


def _actions(kind, actions, N):
    if kind == GAUSSIAN:
        return _rows(actions, N)
    return actions.detach().to(torch.int64).reshape(N).contiguous()


def _objective(kind, params, old, actions, log_prob_old, adv, adv_stats, entropy_coef, grad):
    L = _lib.load()
    N = params[0].shape[0]
    dev = params[0].device
    p = [_rows(x, N) for x in params]
    o = [_rows(x, N) for x in old]
    A = p[0].shape[1]
    g = [torch.empty_like(x) for x in p] if grad else [None, None]
    out = torch.empty(3, dtype=torch.float32, device=dev)
    scratch = torch.empty(((N + 255) // 256) * 3, dtype=torch.float64, device=dev)
    p1 = p[1] if kind == GAUSSIAN else None
    o1 = o[1] if kind == GAUSSIAN else None
    g1 = g[1] if kind == GAUSSIAN else None
    _lib.check(L.b2rl_trpo_objective(
        kind, N, A, _p(p[0]), _p(p1), _p(o[0]), _p(o1), _p(_actions(kind, actions, N)),
        _p(_cuda(log_prob_old).view(-1)), _p(_cuda(adv).view(-1)),
        _p(None if adv_stats is None else _cuda(adv_stats)), float(entropy_coef), _p(g[0]),
        _p(g1), _p(scratch), _p(out), _stream()))
    return out, g


def objective(kind, params, old, actions, log_prob_old, adv, adv_stats, entropy_coef):
    """out[3] = gain, mean KL(old || new), mean entropy (no gradient)."""
    return _objective(kind, params, old, actions, log_prob_old, adv, adv_stats, entropy_coef,
                      False)[0]


class _TrpoGain(torch.autograd.Function):
    @staticmethod
    def forward(ctx, kind, old, actions, log_prob_old, adv, adv_stats, entropy_coef, *params):
        out, g = _objective(kind, params, old, actions, log_prob_old, adv, adv_stats,
                            entropy_coef, True)
        ctx.save_for_backward(*[x for x in g if x is not None])
        ctx.shapes = [x.shape for x in params]
        ctx.mark_non_differentiable(out)
        return out[0].clone(), out

    @staticmethod
    def backward(ctx, g_gain, g_out):
        grads = [(gr * g_gain).view(s) for gr, s in zip(ctx.saved_tensors, ctx.shapes)]
        return (None,) * 7 + tuple(grads)


def gain(kind, params, old, actions, log_prob_old, adv, adv_stats, entropy_coef):
    """Returns (gain (differentiable in params), out[3] = gain, kl, mean entropy)."""
    return _TrpoGain.apply(kind, old, actions, log_prob_old, adv, adv_stats, entropy_coef,
                           *params)


def fisher(kind, params, tangents):
    """M u / N for tangents u of the distribution parameters (same shapes as params).
    Returns one tensor per tangent; None where a tangent is None (a constant scale)."""
    L = _lib.load()
    N = params[0].shape[0]
    p = [_rows(x, N) for x in params]
    u = [None if t is None else _rows(t, N) for t in tangents]
    m = [None if t is None else torch.empty_like(t) for t in u]
    if kind == GAUSSIAN:
        p1, u1, m1 = p[1], (u[1] if len(u) > 1 else None), (m[1] if len(m) > 1 else None)
    else:
        p1 = u1 = m1 = None
    _lib.check(L.b2rl_trpo_fisher(kind, N, p[0].shape[1], _p(p[0]), _p(p1), _p(u[0]), _p(u1),
                                  _p(m[0]), _p(m1), _stream()))
    return [None if mi is None else mi.view(t.shape) for mi, t in zip(m, tangents)]


def cg_init(b):
    """x = 0, r = p = b; returns (x, r, p, state) for cg_iter."""
    L = _lib.load()
    b = _cuda(b).view(-1)
    x, r, p = torch.empty_like(b), torch.empty_like(b), torch.empty_like(b)
    state = torch.empty(2, dtype=torch.float64, device=b.device)
    _lib.check(L.b2rl_trpo_cg_init(b.numel(), _p(b), _p(x), _p(r), _p(p), _p(state), _stream()))
    return x, r, p, state


def cg_iter(Ap, x, r, p, state, tol):
    L = _lib.load()
    for t, name in ((x, "x"), (r, "r"), (p, "p")):
        _buffer(t, name)
    assert state.is_cuda and state.dtype == torch.float64 and state.numel() == 2
    Ap = _cuda(Ap).view(-1)
    assert Ap.numel() == x.numel() == r.numel() == p.numel()
    _lib.check(L.b2rl_trpo_cg_iter(x.numel(), _p(Ap), _p(x), _p(r), _p(p), _p(state),
                                   float(tol), _stream()))


def cg_step(x, Ax, max_kl):
    """Returns (full_step = sqrt(2 max_kl / (dId + 1e-8)) * x, dId [1])."""
    L = _lib.load()
    x = _cuda(x).view(-1)
    Ax = _cuda(Ax).view(-1)
    assert Ax.numel() == x.numel()
    full = torch.empty_like(x)
    dId = torch.empty(1, dtype=torch.float32, device=x.device)
    _lib.check(L.b2rl_trpo_cg_step(x.numel(), _p(x), _p(Ax), float(max_kl), _p(full), _p(dId),
                                   _stream()))
    return full, dId


def line_search(cand, gain0, max_kl, theta_old, full_step, theta=None):
    """cand [C, 3], gain0 [3]: objective outputs.  Writes theta (new or given) and returns
    (theta, record[3] = accepted KL, step size (0 if none), 1 if accepted)."""
    L = _lib.load()
    cand, gain0 = _cuda(cand), _cuda(gain0)
    theta_old, full_step = _cuda(theta_old).view(-1), _cuda(full_step).view(-1)
    assert cand.dim() == 2 and cand.shape[1] == 3 and gain0.numel() >= 1
    assert full_step.numel() == theta_old.numel()
    if theta is None:
        theta = torch.empty_like(theta_old)
    assert _buffer(theta, "theta").numel() == theta_old.numel()
    record = torch.empty(3, dtype=torch.float32, device=theta.device)
    _lib.check(L.b2rl_trpo_line_search(cand.shape[0], _p(cand), _p(gain0), float(max_kl),
                                       theta_old.numel(), _p(theta_old), _p(full_step),
                                       _p(theta), _p(record), _stream()))
    return theta, record
