"""The reference's soft target update (pfrl/utils/copy_param.py:9-22) restated line
for line, and the small networks tests/golden/soft_update.npz is made from.

TEST INFRASTRUCTURE ONLY.  oracle/gen_golden_soft_update.py builds these networks
and runs the reference's own soft_copy_param on them; tests/test_soft_update_cpu.py
pins the restatement to that fixture, and the GPU tests then use the restatement
as the reference on the device."""
import numpy as np
import torch
from torch import nn

# the sequence of updates the fixture records, in order
TAUS = (5e-3, 1 / 3, 0.37, 1.0, 0.0)
NETS = ("mlp_bn_fp32", "mlp_bn_fp64", "mlp_bn_fp16", "mlp_bn_bf16", "tied", "noncontig_buffer",
        "zero_size", "special_values")
_DTYPES = dict(fp32=torch.float32, fp64=torch.float64, fp16=torch.float16, bf16=torch.bfloat16)


def reference_soft_copy(target_link, source_link, tau):
    """copy_param.py:9-22: average the fp32 / fp64 / fp16 entries in place; every other
    entry is rebound in the dict copy, which leaves the target module as it is."""
    target_dict = target_link.state_dict()
    source_dict = source_link.state_dict()
    for k, target_value in target_dict.items():
        source_value = source_dict[k]
        if source_value.dtype in [torch.float32, torch.float64, torch.float16]:
            assert target_value.shape == source_value.shape
            target_value.mul_(1 - tau)
            target_value.add_(tau * source_value)
        else:
            # Scalar type
            # Some modules such as BN has scalar value `num_batches_tracked`
            target_dict[k] = source_value


def special_values(dtype, n, gen):
    """n values of `dtype`: randn with NaN, +-inf, +-0.0, the smallest subnormals of the
    dtype and of fp32, and the largest finite value planted at the front."""
    info = torch.finfo(dtype)
    planted = [float("nan"), float("inf"), -float("inf"), -0.0, 0.0, info.smallest_normal / 4,
               -info.smallest_normal / 2, info.smallest_normal * 2 ** -9, 2.0 ** -149, -2.0 ** -149,
               info.max, -info.max, 1.0, -1.0]
    x = torch.randn(n, generator=gen, dtype=torch.float64)
    x[:len(planted)] = torch.tensor(planted, dtype=torch.float64)
    return x[torch.randperm(n, generator=gen)].to(dtype)


class _Tied(nn.Module):
    """One Linear registered under two names (state_dict lists it twice, same storage)."""

    def __init__(self):
        super().__init__()
        self.first = nn.Linear(6, 5)
        self.second = self.first
        self.head = nn.Linear(5, 3)


class _Buffers(nn.Module):
    def __init__(self):
        super().__init__()
        self.body = nn.Linear(7, 4)


def make_net(name, seed):
    """A freshly initialised network of kind `name`, deterministic in `seed` (CPU); the
    global generator the layers initialise from is restored afterwards."""
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(seed)
        return _make_net(name, seed, torch.Generator().manual_seed(seed))


def _make_net(name, seed, gen):
    if name.startswith("mlp_bn_"):
        net = nn.Sequential(nn.Linear(9, 16), nn.BatchNorm1d(16), nn.ReLU(), nn.Linear(16, 3))
        net = net.to(_DTYPES[name[len("mlp_bn_"):]])
        bn = net[1]
        with torch.no_grad():
            bn.running_mean.copy_(torch.randn(16, generator=gen))
            bn.running_var.copy_(torch.rand(16, generator=gen) + 0.5)
            bn.weight.copy_(torch.rand(16, generator=gen) + 0.5)
        bn.num_batches_tracked.fill_(3 + 8 * seed)
        return net
    if name == "tied":
        return _Tied()
    net = _Buffers()
    if name == "noncontig_buffer":
        # a registered buffer that is a transposed view of its storage
        net.register_buffer("stat_t", torch.randn(5, 3, generator=gen).t())
        net.register_buffer("stride2", torch.randn(12, generator=gen)[::2])
    elif name == "zero_size":
        net.register_buffer("empty", torch.zeros(0))
        net.register_buffer("empty_2d", torch.zeros(3, 0))
        net.empty_param = nn.Parameter(torch.zeros(0, 4))
        net.register_buffer("steps", torch.tensor(seed, dtype=torch.int64))
    elif name == "special_values":
        net.s32 = nn.Parameter(special_values(torch.float32, 64, gen))
        net.s64 = nn.Parameter(special_values(torch.float64, 32, gen))
        net.register_buffer("s16", special_values(torch.float16, 64, gen))
    else:
        raise ValueError(name)
    return net


def make_pair(name):
    """(target, source) as the fixture starts them: two differently seeded nets."""
    return make_net(name, 0), make_net(name, 1)


def to_numpy(t):
    """A state_dict entry as numpy, bf16 as its uint16 bit pattern (numpy has no bf16)."""
    t = t.detach().cpu()
    if t.dtype == torch.bfloat16:
        t = t.contiguous().view(torch.uint16)
    return t.numpy().copy()


def bits(t):
    """A tensor's bit pattern as an integer numpy array (NaN payloads and signed zeros
    compare exactly)."""
    t = t.detach().cpu().contiguous()
    if t.is_floating_point():
        t = t.view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])
    return t.numpy()


def array_bits(a, like):
    """Bit pattern of a fixture array holding an entry shaped and typed like `like`."""
    return bits(from_numpy(a, like.dtype))


def from_numpy(a, dtype):
    t = torch.from_numpy(np.asarray(a).copy(order="C"))
    if dtype == torch.bfloat16:
        t = t.view(torch.bfloat16)
    assert t.dtype == dtype
    return t
