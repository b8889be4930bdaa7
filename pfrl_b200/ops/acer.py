"""ACER's discrete-action loss gradient (csrc/acer.cu) behind torch."""
import torch

from pfrl_b200 import _lib
from pfrl_b200.ops.ppo import _f32, _p, _stream

SCRATCH_PER_STEP = 10


def _rows(t, name, T, K):
    assert t.is_cuda, "%s must be a CUDA tensor" % name
    t = _f32(t)
    assert t.shape == (T, K), "%s must be [%d, %d], got %s" % (name, T, K, tuple(t.shape))
    return t


def loss_grads(z, q, actions, rewards, *, avg_z=None, mu_z=None, bootstrap=None, gamma,
               truncation_threshold, use_trust_region, delta, beta, pi_loss_coef, Q_loss_coef,
               normalize_loss_by_steps, use_Q_opc, average_kl=None, average_kl_decay=0.0):
    """(g_z, g_q) = d total / d z and d total / d q of ACER's loss on one sequence of T steps.

    z, q [T, K]: the policy's ``Categorical._param`` and the Q values; avg_z: the average
    model's logits (needed with the trust region); mu_z: the behaviour policy's logits, None
    for the online (on-policy) update; actions [T] int64; rewards [T] fp64 on the device;
    bootstrap: a device scalar, or None when the last step is terminal.  average_kl: an fp64
    device tensor of one element that takes the steps' KL when use_trust_region is set."""
    L = _lib.load()
    T, K = z.shape
    dev = z.device
    z = _rows(z, "z", T, K)
    q = _rows(q, "q", T, K)
    avg_z = None if avg_z is None else _rows(avg_z, "avg_z", T, K)
    mu_z = None if mu_z is None else _rows(mu_z, "mu_z", T, K)
    actions = actions.detach().to(torch.int64).reshape(T).contiguous()
    assert rewards.is_cuda and rewards.dtype == torch.float64 and rewards.numel() == T
    rewards = rewards.reshape(T).contiguous()
    if bootstrap is not None:
        bootstrap = _f32(bootstrap).reshape(1)
    if use_trust_region:
        assert avg_z is not None, "the trust region needs the average model's logits"
        assert average_kl is not None and average_kl.dtype == torch.float64 \
            and average_kl.is_cuda and average_kl.numel() == 1 and average_kl.is_contiguous()
    out = torch.empty((2, T, K), dtype=torch.float32, device=dev)
    scratch = torch.empty(T * SCRATCH_PER_STEP, dtype=torch.float64, device=dev)
    truncate = truncation_threshold is not None
    _lib.check(L.b2rl_acer_loss(
        T, K, _p(z), _p(q), _p(avg_z), _p(mu_z), _p(actions), _p(rewards), _p(bootstrap),
        float(gamma), int(truncate), float(truncation_threshold) if truncate else 0.0,
        int(bool(use_trust_region)), float(delta), float(beta), float(pi_loss_coef),
        float(Q_loss_coef), int(bool(normalize_loss_by_steps)), int(bool(use_Q_opc)),
        _p(average_kl if use_trust_region else None), float(average_kl_decay), _p(scratch),
        _p(out[0]), _p(out[1]), _stream()))
    return out[0], out[1]
