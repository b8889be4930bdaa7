"""SAC / TD3 / DDPG update tail (csrc/sac.cu) behind torch: multi-tensor Polyak
averaging in one launch and the entropy-regularised TD target, both rounded like the
reference's sequence of separate fp32 operations."""
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
