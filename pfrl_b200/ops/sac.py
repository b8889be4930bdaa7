"""SAC / TD3 / DDPG update tail (csrc/sac.cu) behind torch: multi-tensor Polyak
averaging in one launch, the entropy-regularised TD target, TD3's target-policy smoothing
and the TD3 / DDPG critic target and losses, rounded like the reference's sequence of
separate fp32 operations (the losses are sums in a fixed order of their own)."""
import ctypes

import torch

from pfrl_b200 import _lib


def _stream(device):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def polyak_(targets, sources, tau):
    """targets[i] = targets[i] * float(1 - tau) + float(tau) * sources[i], in place, one
    launch per 96 tensors (pfrl/utils/copy_param.py:9-22).  fp32 contiguous tensors on
    one CUDA device; zero-size pairs are skipped.  The targets must not share memory with
    each other or with any source: the kernel updates all pairs concurrently."""
    assert len(targets) == len(sources)
    if not targets:
        return
    device = targets[0].device
    pairs = []
    for t, s in zip(targets, sources):
        assert t.is_cuda and t.device == device and s.device == device
        assert t.dtype == torch.float32 and s.dtype == torch.float32
        assert t.is_contiguous() and s.is_contiguous() and t.shape == s.shape
        if t.numel():  # an empty CUDA tensor has no storage (data_ptr() == 0)
            pairs.append((t, s))
    if not pairs:
        return
    L = _lib.load()
    arr = (_lib.TensorPair * len(pairs))()
    for i, (t, s) in enumerate(pairs):
        arr[i].dst, arr[i].src, arr[i].numel = t.data_ptr(), s.data_ptr(), t.numel()
    _lib.check(L.b2rl_polyak(arr, len(pairs), float(tau), _stream(device)))


def sac_target(reward, discount, terminal, q1, q2, log_prob, temperature):
    """reward + discount * (1 - terminal) * (min(q1, q2) - temperature * log_prob), fp32 [n]
    (pfrl/agents/soft_actor_critic.py:225-240).  Every input, and temperature when it is a
    tensor, must be a CUDA tensor on reward's device; temperature may also be a float."""
    device = reward.device
    inputs = (reward, discount, terminal, q1, q2, log_prob)
    if isinstance(temperature, torch.Tensor):
        inputs += (temperature,)
    if device.type != "cuda" or any(t.device != device for t in inputs):
        raise ValueError("sac_target: every tensor must be on one CUDA device, got %s"
                         % ", ".join(str(t.device) for t in inputs))
    n = reward.numel()
    args = [t.detach().reshape(-1).float().contiguous()
            for t in (reward, discount, terminal, q1, q2, log_prob)]
    assert all(t.numel() == n for t in args)
    out = torch.empty(n, dtype=torch.float32, device=device)
    if n == 0:
        return out
    if isinstance(temperature, torch.Tensor):
        assert temperature.numel() == 1
        tdev = temperature.detach().reshape(-1).float().contiguous()
        tptr, tval = ctypes.c_void_p(tdev.data_ptr()), 0.0
    else:
        tptr, tval = None, float(temperature)
    L = _lib.load()
    _lib.check(L.b2rl_sac_target(*[ctypes.c_void_p(t.data_ptr()) for t in args], tptr, tval, n,
                                 ctypes.c_void_p(out.data_ptr()), _stream(device)))
    return out


def _require_f32_cuda(name, tensors):
    device = tensors[0].device
    if device.type != "cuda" or any(t.device != device for t in tensors):
        raise ValueError("%s: every tensor must be on one CUDA device, got %s"
                         % (name, ", ".join(str(t.device) for t in tensors)))
    if any(t.dtype != torch.float32 for t in tensors):
        raise ValueError("%s: every tensor must be float32, got %s"
                         % (name, ", ".join(str(t.dtype) for t in tensors)))
    return device


def td3_smooth(action, noise):
    """clamp(action + clamp(0.2 * noise, -0.5, 0.5), -1, 1): TD3's default target-policy
    smoothing (pfrl/agents/td3.py:20-24) for a given ``noise`` (the caller's
    ``torch.randn_like(action)``), bit for bit.  fp32 CUDA tensors of one shape."""
    device = _require_f32_cuda("td3_smooth", (action, noise))
    if action.shape != noise.shape:
        raise ValueError("td3_smooth: action %s and noise %s differ in shape"
                         % (tuple(action.shape), tuple(noise.shape)))
    a, e = action.detach().contiguous(), noise.detach().contiguous()
    out = torch.empty_like(a)
    if a.numel():
        _lib.check(_lib.load().b2rl_td3_smooth(ctypes.c_void_p(a.data_ptr()),
                                               ctypes.c_void_p(e.data_ptr()), a.numel(),
                                               ctypes.c_void_p(out.data_ptr()), _stream(device)))
    return out


class _KernelMseLoss(torch.autograd.Function):
    """mse_loss(target, pred) whose value and d loss / d pred were formed by
    b2rl_td3_critic_loss; the backward scales that gradient by the upstream one, as torch's
    mse_loss backward does."""

    @staticmethod
    def forward(ctx, pred, loss, grad):
        ctx.save_for_backward(grad)
        return loss

    @staticmethod
    def backward(ctx, grad_loss):
        grad, = ctx.saved_tensors
        return grad * grad_loss, None, None


def critic_loss(reward, discount, terminal, next_q1, next_q2, pred_q1, pred_q2):
    """The critic update of TD3 / DDPG after its forwards, in one launch.

    target = reward + discount * (1 - terminal) * min(next_q1, next_q2), as td3.py's eager
    expression bit for bit; ``discount`` is a tensor (TD3's n-step discount) or a float
    (DDPG's gamma), and ``next_q2`` / ``pred_q2`` may be None (DDPG: next_q1 is the next
    value, one critic).  Returns (target, loss1, loss2): loss_c = mse_loss(target, pred_c),
    differentiable with respect to pred_c, and loss2 None without a second critic.  Every
    tensor is fp32 on one CUDA device with n elements (the Q tensors [n] or [n, 1])."""
    with_discount = isinstance(discount, torch.Tensor)
    tensors = [t for t in (reward, discount if with_discount else None, terminal, next_q1,
                           next_q2, pred_q1, pred_q2) if t is not None]
    device = _require_f32_cuda("critic_loss", tensors)
    n = reward.numel()
    if n == 0 or any(t.numel() != n for t in tensors):
        raise ValueError("critic_loss: need n > 0 elements in every tensor, got %s"
                         % ", ".join(str(tuple(t.shape)) for t in tensors))
    flat = [None if t is None else t.detach().reshape(-1).contiguous()
            for t in (reward, discount if with_discount else None, terminal, next_q1, next_q2,
                      pred_q1, pred_q2)]
    two = pred_q2 is not None
    target = torch.empty(n, dtype=torch.float32, device=device)
    grads = torch.empty((2 if two else 1, n), dtype=torch.float32, device=device)
    losses = torch.empty(2 if two else 1, dtype=torch.float32, device=device)
    ctas = -(-n // 1024)  # B2RL_CRITIC_LOSS_ROWS_PER_CTA
    partial = torch.empty(2 * ctas, dtype=torch.float32, device=device) if ctas > 1 else None
    p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())  # noqa: E731
    _lib.check(_lib.load().b2rl_td3_critic_loss(
        *[p(t) for t in flat[:2]], 0.0 if with_discount else float(discount),
        *[p(t) for t in flat[2:]], n, p(target), p(grads[0]), p(grads[1]) if two else None,
        p(losses[0]), p(losses[1]) if two else None, p(partial), _stream(device)))
    loss1 = _KernelMseLoss.apply(pred_q1.reshape(-1), losses[0], grads[0])
    loss2 = _KernelMseLoss.apply(pred_q2.reshape(-1), losses[1], grads[1]) if two else None
    return target, loss1, loss2
