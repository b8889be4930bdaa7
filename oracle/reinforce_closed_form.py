"""Closed-form fp64 restatement of REINFORCE's loss gradient
(pfrl/agents/reinforce.py:176-195), the arithmetic of csrc/reinforce.cu.

TEST INFRASTRUCTURE ONLY.  loss = sum_rows(-R log pi(a) - beta H) / batchsize.  The
gradients are taken with respect to a ``Categorical``'s ``_param`` (normalised logits) or
an ``Independent(Normal, 1)``'s loc and scale, as the reference's backward reaches them.
The two per-row coefficients the backward hands log pi(a) and H,
fl(fl(1 / batchsize) * fl(-R)) and -fl(fl(1 / batchsize) * fl(beta)), are rounded in
``coef_dtype``: float32 for an fp32 policy (what the kernel does), float64 for an fp64
one.  tests/test_reinforce_cpu.py checks this against the reference formulation's
autograd; tests/test_reinforce_kernel_gpu.py checks the kernel against this.
"""
import numpy as np

FP32_MIN = float(np.finfo(np.float32).min)


def coefficients(R, batchsize, beta, coef_dtype=np.float32):
    """(c_lp [N], c_H) as fp64 values of the coef_dtype products."""
    f = np.dtype(coef_dtype).type
    inv_bs = f(1) / f(batchsize)
    R = np.asarray(R)
    c_lp = (inv_bs * (-R.astype(coef_dtype))).astype(coef_dtype)
    c_h = -(inv_bs * f(beta))
    return c_lp.astype(np.float64), float(c_h)


def categorical_grads(z, actions, R, beta, batchsize, coef_dtype=np.float32):
    """Returns (g_z [N, K], loss, entropy sum), fp64."""
    z = np.asarray(z, np.float64)
    N, K = z.shape
    a = np.asarray(actions, np.int64).reshape(N)
    c_lp, c_h = coefficients(R, batchsize, beta, coef_dtype)
    m = np.max(z, axis=1, keepdims=True)
    with np.errstate(invalid="ignore", over="ignore", under="ignore"):
        lse = m + np.log(np.sum(np.exp(z - m), axis=1, keepdims=True))
        p = np.exp(z - lse)
        c = np.maximum(z, FP32_MIN)
        h = -np.sum(p * c, axis=1)
        dh = -p * ((z >= FP32_MIN) + c + h[:, None])
    g = c_h * dh
    g[np.arange(N), a] += c_lp
    lp = z[np.arange(N), a]
    loss = np.sum(-np.asarray(R, np.float64) * lp - float(beta) * h) / batchsize
    return g, float(loss), float(np.sum(h))


def gaussian_grads(loc, scale, action_values, R, beta, batchsize, coef_dtype=np.float32):
    """Returns (g_loc [N, A], g_scale [N, A], loss, entropy sum), fp64.  scale None = 1."""
    loc = np.asarray(loc, np.float64)
    s = np.ones_like(loc) if scale is None else np.broadcast_to(
        np.asarray(scale, np.float64), loc.shape)
    d = np.asarray(action_values, np.float64).reshape(loc.shape) - loc
    c_lp, c_h = coefficients(R, batchsize, beta, coef_dtype)
    c_lp = c_lp[:, None]
    with np.errstate(over="ignore", divide="ignore", invalid="ignore"):
        inv_s = 1.0 / s
        g_loc = c_lp * d * inv_s * inv_s
        g_scale = c_lp * (d * d * inv_s ** 3 - inv_s) + c_h * inv_s
        half_log_2pi = 0.5 * np.log(2 * np.pi)
        lp = np.sum(-(d * d) * 0.5 * inv_s * inv_s - np.log(s) - half_log_2pi, axis=1)
        h = np.sum(0.5 + half_log_2pi + np.log(s), axis=1)
    loss = np.sum(-np.asarray(R, np.float64) * lp - float(beta) * h) / batchsize
    return g_loc, g_scale, float(loss), float(np.sum(h))


def reference_returns(r_seq):
    """The reference's returns of one episode's reward record (whose last reward
    _observe_train appended twice)."""
    return np.cumsum(list(reversed(r_seq[1:])))[::-1]
