"""Closed-form fp64 restatement of ACER's discrete-action loss gradient
(pfrl/agents/acer.py:16-115, 207-248, 423-552), the arithmetic of csrc/acer.cu.

TEST INFRASTRUCTURE ONLY.  ``z`` is the policy's ``Categorical._param`` (normalised
logits), and the gradients are taken with respect to it, as the reference's
``torch.autograd.grad`` takes them.  tests/test_acer_cpu.py checks this against the
reference formulation's autograd; tests/test_acer_kernel_gpu.py checks the kernel
against this.
"""
import numpy as np


def _log_softmax(x):
    x = np.asarray(x, dtype=np.float64)
    m = np.max(x, axis=-1, keepdims=True)
    with np.errstate(invalid="ignore", over="ignore"):
        lse = m + np.log(np.sum(np.exp(x - m), axis=-1, keepdims=True))
    return x - lse


def _nonzero(p):
    """torch decides p == 0 on the fp32 probabilities."""
    return np.asarray(p, dtype=np.float32) != 0


def acer_loss_grads(z, q, actions, rewards, *, avg_z=None, mu_z=None, bootstrap=None, gamma,
                    truncation_threshold, use_trust_region, delta, beta, pi_loss_coef,
                    Q_loss_coef, normalize_loss_by_steps, use_Q_opc, average_kl=0.0,
                    average_kl_decay=0.0):
    """Returns (g_z [T, K], g_q [T, K], average_kl after the update), all fp64."""
    z = np.asarray(z, np.float64)
    q = np.asarray(q, np.float64)
    T, K = z.shape
    a = np.asarray(actions, np.int64).reshape(T)
    r = np.asarray(rewards, np.float64).reshape(T)
    lp = _log_softmax(z)
    p = np.exp(lp)
    nz = _nonzero(p)
    v = np.sum(p * q, axis=1)
    Q = q[np.arange(T), a]
    h = -np.sum(np.where(nz, p * lp, 0.0), axis=1)
    with np.errstate(over="ignore", invalid="ignore"):
        if mu_z is not None:
            lmu = _log_softmax(mu_z)
            rho = np.exp(lp[np.arange(T), a] - lmu[np.arange(T), a])
        else:
            rho = np.ones(T)
        if use_trust_region:
            la = _log_softmax(avg_z)
            pa = np.exp(la)
            nza = _nonzero(pa)
            kl_terms = np.where(nza, np.where(nz, pa * (la - lp), np.inf), 0.0)
            kl = np.sum(kl_terms, axis=1)
            k = np.where(nza & nz, pa, 0.0)
    # the scan, in Python floats as the reference's
    adv = np.zeros(T)
    q_ret_t = np.zeros(T)
    q_ret = 0.0 if bootstrap is None else float(bootstrap)
    q_opc = q_ret
    avg_kl = float(average_kl)
    for t in reversed(range(T)):
        q_ret = float(r[t]) + gamma * q_ret
        q_opc = float(r[t]) + gamma * q_opc
        adv[t] = (q_opc if use_Q_opc else q_ret) - v[t]
        q_ret_t[t] = q_ret
        if use_trust_region:
            avg_kl += (1 - average_kl_decay) * (kl[t] - avg_kl)
        q_ret = min(1.0, rho[t]) * (q_ret - Q[t]) + v[t]
        q_opc = q_opc - Q[t] + v[t]
    g = np.zeros((T, K))
    corr = mu_z is not None and truncation_threshold is not None
    for t in range(T):
        w = min(truncation_threshold, rho[t]) if corr else rho[t]
        g[t, a[t]] = -w * adv[t]
        if corr:
            c = float(truncation_threshold)
            with np.errstate(over="ignore", invalid="ignore"):
                x = 1.0 - c * np.exp(lmu[t] - lp[t])
                cw = np.where(np.isnan(x), x, np.maximum(x, 0.0)) * p[t]
            g[t] -= cw * (q[t] - v[t])
        if use_trust_region:
            kk = float(np.dot(k[t], k[t]))
            kf = 0.0
            if kk > 0:
                f = (float(np.dot(k[t], g[t])) - delta) / kk
                kf = f if f > 0 else 0.0
            if kf != 0.0:
                g[t] -= kf * k[t]
        g[t] += np.where(nz[t], beta * p[t] * (1.0 + lp[t] + h[t]), 0.0)
    scale = 1.0 / T if normalize_loss_by_steps else 1.0
    g_z = pi_loss_coef * scale * g
    g_q = np.zeros((T, K))
    g_q[np.arange(T), a] = Q_loss_coef * scale * (Q - q_ret_t.astype(np.float32))
    return g_z, g_q, avg_kl
