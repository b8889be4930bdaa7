"""Parameter copies between networks (pfrl/utils/copy_param.py)."""
import bisect

import torch


def copy_param(target_link, source_link):
    """Hard copy of every state_dict entry (copy_param.py:4-6)."""
    target_link.load_state_dict(source_link.state_dict())


_AVERAGED = (torch.float32, torch.float64, torch.float16)


def _span(t):
    return t.data_ptr(), t.data_ptr() + t.numel() * t.element_size()


def _one_launch_ok(targets, sources):
    """True when the pairs can go to b2rl_polyak together: all fp32, contiguous,
    on one CUDA device, and no target shares memory with another target or with
    a source (the kernel updates every pair at once, so a shared word would be
    read and written by two CTAs)."""
    device = targets[0].device
    if device.type != "cuda":
        return False
    for t in targets + sources:
        if t.device != device or t.dtype != torch.float32 or not t.is_contiguous():
            return False
    spans = sorted(_span(t) for t in targets)
    for (_, end), (begin, _) in zip(spans, spans[1:]):
        if begin < end:
            return False
    begins = [b for b, _ in spans]
    for s in sources:
        s_begin, s_end = _span(s)
        # the last target that starts before the source ends is the only one that
        # can overlap it (targets are disjoint and sorted)
        i = bisect.bisect_left(begins, s_end) - 1
        if i >= 0 and spans[i][1] > s_begin:
            return False
    return True


@torch.no_grad()
def soft_copy_param(target_link, source_link, tau):
    """Polyak averaging ``target = (1 - tau) * target + tau * source`` over the
    fp32, fp64 and fp16 state_dict entries, in state_dict order
    (copy_param.py:9-22).  Every other entry (integer buffers such as
    BatchNorm's ``num_batches_tracked``, bf16 tensors) is left as it is: the
    reference rebinds them in a copy of the target's state_dict, which does not
    touch the target module.

    When every averaged pair is fp32, contiguous, on one CUDA device and no
    target shares memory with another target or a source, all pairs go in one
    launch (b2rl_polyak), rounded like the reference.  Otherwise the
    reference's own per-entry loop runs, so other dtypes round as it does and a
    tied parameter (one tensor under two names) is averaged twice."""
    tgt = target_link.state_dict()
    src = source_link.state_dict()
    f_t, f_s = [], []
    for k, tv in tgt.items():
        sv = src[k]
        if sv.dtype in _AVERAGED:
            assert tv.shape == sv.shape
            if tv.numel():
                f_t.append(tv)
                f_s.append(sv)
    if not f_t:
        return
    if _one_launch_ok(f_t, f_s):
        # one launch for the whole network (csrc/sac.cu, K9)
        from pfrl_b200.ops.sac import polyak_

        polyak_(f_t, f_s, tau)
    else:
        for tv, sv in zip(f_t, f_s):
            tv.mul_(1 - tau)
            tv.add_(tau * sv)


def copy_grad(target_link, source_link):
    """Give ``target_link``'s parameters clones of ``source_link``'s gradients
    (``None`` where the source has none)."""
    pairs = zip(target_link.parameters(), source_link.parameters())
    for dst, src in pairs:
        assert dst.shape == src.shape
        dst.grad = None if src.grad is None else src.grad.clone()


def copy_grad_into(target_link, source_link):
    """``copy_grad``'s result, with the gradients that ``target_link`` already holds
    overwritten in one multi-tensor copy instead of replaced by clones; a missing target
    gradient is cloned once."""
    dst, src = [], []
    for t, s in zip(target_link.parameters(), source_link.parameters()):
        assert t.shape == s.shape
        if s.grad is None:
            t.grad = None
        elif t.grad is None or t.grad.dtype != s.grad.dtype or t.grad.device != s.grad.device:
            t.grad = s.grad.clone()
        else:
            dst.append(t.grad)
            src.append(s.grad)
    if dst:
        torch._foreach_copy_(dst, src)


def synchronize_parameters(src, dst, method, tau=None):
    """copy_param.py:37-41"""
    if method == "hard":
        copy_param(dst, src)
    elif method == "soft":
        soft_copy_param(dst, src, tau)
    else:
        raise ValueError("unknown target update method: %r" % (method,))
