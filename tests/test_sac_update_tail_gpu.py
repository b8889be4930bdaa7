"""GPU: the SAC / TD3 / DDPG update tail (csrc/sac.cu, K9) against the reference.

k_polyak (through ops.sac.polyak_ and the raw C ABI) and k_sac_target are compared
bit for bit with the reference's expressions run eagerly on the same device, and
against fp64 per element with a bound derived from their roundings.
utils.copy_param.soft_copy_param is compared on every dispatch route with the
restatement of pfrl/utils/copy_param.py:9-22 in tests/soft_update_ref.py, which
tests/test_soft_update_cpu.py pins to the reference itself.  The agents' target
syncs and SAC's Q update are compared with the same restatements."""
import copy
import ctypes
import os
import sys

import numpy as np
import pytest
import torch
from torch import nn

sys.path.insert(0, os.path.dirname(__file__))
from soft_update_ref import bits, make_pair, reference_soft_copy  # noqa: E402

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
TINY = 2.0 ** -149  # smallest fp32 subnormal
TAUS = (0.0, 1.0, 5e-3, 1 / 3, 1 - 2.0 ** -24, 1e-300)


def _same_bits(got, want, what=""):
    np.testing.assert_array_equal(bits(got), bits(want), err_msg=str(what))


def _planted(n, gen, salt):
    """fp32 [n] on CUDA: randn at mixed scales, with NaN, +-inf, +-0.0, subnormals and
    large values planted at seeded positions."""
    x = torch.randn(n, generator=gen, device="cuda") * \
        torch.exp2(torch.randint(-8, 9, (n,), generator=gen, device="cuda").float())
    planted = torch.tensor([float("nan"), float("inf"), -float("inf"), -0.0, 0.0, TINY, -TINY,
                            2.0 ** -130, -3 * 2.0 ** -140, 2.0 ** -126, 1e38, -1e38],
                           device="cuda")
    k = min(n, len(planted))
    pos = torch.randperm(n, generator=gen, device="cuda")[:k]
    x[pos] = planted[(torch.arange(k, device="cuda") + salt) % len(planted)]
    return x


def _eager_polyak(t, s, tau):
    """The reference's two operations on one fp32 tensor (copy_param.py:17-18)."""
    t.mul_(1 - tau)
    t.add_(tau * s)


def _check_polyak_fp64(got, d, s, tau):
    """|k - ((1-tau)d + tau s)| <= 4U((1-tau)|d| + tau|s|) + 3 * 2^-149 where the inputs
    are finite: float(1 - tau), float(tau), the two products and the sum each round once
    (relative U each, at most 2^-150 absolute in the subnormal range)."""
    d64, s64 = d.double(), s.double()
    fin = torch.isfinite(d64) & torch.isfinite(s64)
    exact = (1 - tau) * d64 + tau * s64
    bound = 4 * U * ((1 - tau) * d64.abs() + tau * s64.abs()) + 3 * TINY
    err = (got.double() - exact).abs()
    bad = fin & ~(err <= bound)
    assert not bad.any(), (tau, got[bad][:5], exact[bad][:5], bound[bad][:5])


# ---- k_polyak through ops.sac.polyak_ ---------------------------------------------

@pytest.mark.parametrize("numel", [1, 255, 256, 2047, 2048, 2049, 3 * 2048 - 1, 3 * 2048 + 1,
                                   2 ** 20 + 3])
def test_polyak_numel_edges(numel):
    from pfrl_b200.ops.sac import polyak_

    g = torch.Generator(device="cuda").manual_seed(numel)
    d0, s = _planted(numel, g, 0), _planted(numel, g, 5)
    for tau in TAUS:
        got, want = d0.clone(), d0.clone()
        polyak_([got], [s], tau)
        _eager_polyak(want, s, tau)
        _same_bits(got, want, (numel, tau))
        _check_polyak_fp64(got, d0, s, tau)


def _pair_sizes(n_pairs):
    # small, chunk-edge and zero sizes interleaved; the last pair is empty
    cycle = [1, 0, 255, 2049, 0, 7, 2048, 300, 0, 4097]
    sizes = [cycle[i % len(cycle)] for i in range(n_pairs)]
    sizes[-1] = 0
    if n_pairs == 1:
        sizes = [2049]
    return sizes


@pytest.mark.parametrize("n_pairs", [1, 95, 96, 97, 191, 192, 193])
def test_polyak_pair_counts(n_pairs):
    """Pair counts around the 96-pair launch split, empty tensors among them."""
    from pfrl_b200 import _lib
    from pfrl_b200.ops.sac import polyak_

    g = torch.Generator(device="cuda").manual_seed(n_pairs)
    sizes = _pair_sizes(n_pairs)
    d0 = [_planted(n, g, i) if n else torch.empty(0, device="cuda") for i, n in enumerate(sizes)]
    s = [_planted(n, g, i + 3) if n else torch.empty(0, device="cuda")
         for i, n in enumerate(sizes)]
    for tau in (5e-3, 1 / 3):
        want = [t.clone() for t in d0]
        for t, src in zip(want, s):
            _eager_polyak(t, src, tau)
        # ops.sac.polyak_ (skips the empty pairs: an empty CUDA tensor has no storage)
        got = [t.clone() for t in d0]
        polyak_(got, s, tau)
        for i, (a, b) in enumerate(zip(got, want)):
            _same_bits(a, b, (n_pairs, tau, i))
        # the raw ABI with the empty pairs passed through, pointing into real storage
        # (an empty tensor's own data_ptr() is 0, which the ABI refuses)
        pool = torch.zeros(2, device="cuda")
        got = [t.clone() for t in d0]
        arr = (_lib.TensorPair * n_pairs)()
        for i, (a, b) in enumerate(zip(got, s)):
            if a.numel():
                arr[i].dst, arr[i].src, arr[i].numel = a.data_ptr(), b.data_ptr(), a.numel()
            else:
                arr[i].dst, arr[i].src, arr[i].numel = pool.data_ptr(), pool.data_ptr() + 4, 0
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        _lib.check(_lib.load().b2rl_polyak(arr, n_pairs, float(tau), stream))
        for i, (a, b) in enumerate(zip(got, want)):
            _same_bits(a, b, (n_pairs, tau, i, "abi"))
        assert torch.equal(pool, torch.zeros(2, device="cuda"))


def test_many_small_tensors_and_large_one():
    from pfrl_b200.ops.sac import polyak_

    g = torch.Generator(device="cuda").manual_seed(1)
    shapes = [(1,), (3,), (2049,), (4096,), (7, 13)] * 45 + [(1 << 20,)]   # > 96 pairs
    t = [torch.randn(s, device="cuda", generator=g) for s in shapes]
    s_ = [torch.randn(s, device="cuda", generator=g) for s in shapes]
    want = [a.clone().mul_(1 - 0.005).add_(0.005 * b) for a, b in zip(t, s_)]
    polyak_(t, s_, 0.005)
    for a, b in zip(t, want):
        assert torch.equal(a, b)


def test_polyak_abi_refusals():
    """Refused before any launch: no target changes."""
    from pfrl_b200 import _lib

    L = _lib.load()
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    d = torch.ones(300, device="cuda")
    s = torch.zeros(300, device="cuda")

    def pairs(*specs):
        arr = (_lib.TensorPair * len(specs))()
        for i, (dp, sp, n) in enumerate(specs):
            arr[i].dst, arr[i].src, arr[i].numel = dp, sp, n
        return arr

    good = (d.data_ptr(), s.data_ptr(), d.numel())
    for tau in (-1e-300, -0.5, 1 + 2.0 ** -52, 2.0, float("nan"), float("inf")):
        assert L.b2rl_polyak(pairs(good), 1, tau, stream) == -4, tau
    assert L.b2rl_polyak(pairs(good), -1, 0.5, stream) != 0
    assert L.b2rl_polyak(None, 1, 0.5, stream) != 0
    assert L.b2rl_polyak(None, 0, 0.5, stream) == 0
    # a bad pair anywhere, even after a full launch's worth of good ones
    for bad in ((0, s.data_ptr(), 4), (d.data_ptr(), 0, 4), (d.data_ptr(), s.data_ptr(), -1)):
        assert L.b2rl_polyak(pairs(*([good] * 100 + [bad])), 101, 0.5, stream) == -1, bad
    torch.cuda.synchronize()
    assert torch.equal(d, torch.ones(300, device="cuda"))


def test_polyak_refuses_mixed_devices_and_dtypes():
    from pfrl_b200.ops.sac import polyak_

    d = torch.ones(8, device="cuda")
    for src in (torch.ones(8), torch.ones(8, device="cuda", dtype=torch.float64),
                torch.ones(16, device="cuda")[::2]):
        with pytest.raises(AssertionError):
            polyak_([d], [src], 0.5)
    assert torch.equal(d, torch.ones(8, device="cuda"))


# ---- soft_copy_param on CUDA, one case per dispatch route ---------------------------

def _mixed_pair():
    t, s = make_pair("mlp_bn_fp32")
    t[3].half()
    s[3].half()
    return t, s


_ROUTES = {
    # name: (build, whether the single polyak_ launch is used)
    "fp32": (lambda: make_pair("mlp_bn_fp32"), True),
    "fp16": (lambda: make_pair("mlp_bn_fp16"), False),
    "fp64": (lambda: make_pair("mlp_bn_fp64"), False),
    "bf16": (lambda: make_pair("mlp_bn_bf16"), False),
    "mixed": (_mixed_pair, False),
    "noncontig_buffer": (lambda: make_pair("noncontig_buffer"), False),
    "tied": (lambda: make_pair("tied"), False),
    "zero_size": (lambda: make_pair("zero_size"), True),
    "special_values": (lambda: make_pair("special_values"), False),
}


@pytest.mark.parametrize("route", list(_ROUTES))
def test_soft_copy_param_routes(route, monkeypatch):
    from pfrl_b200.ops import sac as sac_ops
    from pfrl_b200.utils.copy_param import soft_copy_param

    build, kernel = _ROUTES[route]
    target, source = (m.cuda() for m in build())
    if route == "noncontig_buffer":
        assert any(not v.is_contiguous() for v in target.state_dict().values())
    ref_t, ref_s = copy.deepcopy(target), copy.deepcopy(source)
    if route == "tied":
        assert ref_t.first.weight is ref_t.second.weight
    calls = []
    real = sac_ops.polyak_
    monkeypatch.setattr(sac_ops, "polyak_", lambda *a: calls.append(1) or real(*a))
    before = {k: v.clone() for k, v in target.state_dict().items()}
    for i, tau in enumerate((5e-3, 1 / 3, 0.37, 1.0, 0.0, 1 - 2.0 ** -24)):
        soft_copy_param(target, source, tau)
        reference_soft_copy(ref_t, ref_s, tau)
        for (k, a), b in zip(target.state_dict().items(), ref_t.state_dict().values()):
            _same_bits(a, b, (route, tau, k))
    assert len(calls) == (6 if kernel else 0)
    for k, v in target.state_dict().items():
        if not v.is_floating_point() or v.dtype == torch.bfloat16:
            assert torch.equal(v, before[k]), k  # integer and bf16 entries stay
    for (k, a), b in zip(source.state_dict().items(), ref_s.state_dict().values()):
        _same_bits(a, b, (route, "source", k))


def test_polyak_matches_reference_sequence():
    """A BatchNorm MLP on the kernel path through several updates; the target's
    num_batches_tracked keeps its own value."""
    from pfrl_b200.utils.copy_param import soft_copy_param

    torch.manual_seed(0)
    mk = lambda: torch.nn.Sequential(  # noqa: E731
        torch.nn.Linear(23, 256), torch.nn.ReLU(), torch.nn.BatchNorm1d(256),
        torch.nn.Linear(256, 256), torch.nn.ReLU(), torch.nn.Linear(256, 1)).cuda()
    src, dst = mk(), mk()
    src[2].num_batches_tracked.fill_(17)
    src(torch.randn(64, 23, device="cuda"))  # moves src's running statistics
    ref = copy.deepcopy(dst)
    for tau in (5e-3, 0.01, 0.37, 1.0, 0.0):
        reference_soft_copy(ref, src, tau)
        soft_copy_param(dst, src, tau)
        for (k, a), b in zip(dst.state_dict().items(), ref.state_dict().values()):
            _same_bits(a, b, (tau, k))
    assert int(dst[2].num_batches_tracked) == 0


# ---- k_sac_target ---------------------------------------------------------------

def _eager_sac_target(reward, discount, terminal, q1, q2, log_prob, temperature):
    """soft_actor_critic.py:236-240 on q [B, 1], log_prob [B]."""
    next_q = torch.min(q1, q2)
    entropy_term = temperature * log_prob[..., None]
    assert next_q.shape == entropy_term.shape
    return reward + discount * (1.0 - terminal) * torch.flatten(next_q - entropy_term)


_INF, _NAN = float("inf"), float("nan")
# (q1, q2, log_prob) planted rows
_ROWS = [(_NAN, 1.0, 0.5), (1.0, _NAN, 0.5), (_NAN, _NAN, 0.5), (-2.0, _NAN, 0.5),
         (_INF, 1.0, 0.5), (1.0, -_INF, 0.5), (_INF, _INF, 0.5), (-_INF, 3.0, 0.5),
         (1.0, 2.0, _INF), (1.0, 2.0, -_INF), (_INF, 2.0, _INF), (_INF, 2.0, -_INF),
         (-0.0, 0.0, 0.0), (0.0, -0.0, 0.0), (-0.0, 0.0, -0.0), (0.0, -0.0, -0.0),
         (-0.0, -0.0, 0.0), (TINY, -TINY, TINY), (3 * TINY, 2.0 ** -127, -2.0 ** -130),
         (2.0 ** -126, 2.0 ** -126 - TINY, 2.0 ** -140), (0.0, 0.0, 1.0)]


def _sac_inputs(B, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = torch.randn(B, generator=g, device="cuda") * 3
    q1 = torch.randn(B, 1, generator=g, device="cuda") * 10
    q2 = torch.randn(B, 1, generator=g, device="cuda") * 10
    lp = torch.randn(B, generator=g, device="cuda") * 4
    disc = torch.tensor([0.0, 0.99, 0.99 ** 2, 0.99 ** 3], device="cuda")[
        torch.randint(0, 4, (B,), generator=g, device="cuda")]
    term = torch.tensor([0.0, 1.0, 0.5], device="cuda")[
        torch.randint(0, 3, (B,), generator=g, device="cuda")]
    rows = torch.tensor(_ROWS, dtype=torch.float32, device="cuda")
    k = min(B, len(_ROWS))
    pos = torch.randperm(B, generator=g, device="cuda")[:k]
    q1[pos, 0], q2[pos, 0], lp[pos] = rows[:k, 0], rows[:k, 1], rows[:k, 2]
    # signed zeros and subnormals reach the output where the reward is -0.0 (the sum
    # keeps the other operand's sign) and the weight is one
    r[pos[12:k]] = -0.0
    disc[pos[12:k]], term[pos[12:k]] = 1.0, 0.0
    return r, disc, term, q1, q2, lp


def _temperature(kind):
    if kind == "0.1":
        return 0.1
    if kind == "1/3":
        return 1 / 3
    if kind == "tensor0d":
        return torch.exp(torch.tensor(-1.4391, device="cuda"))
    return torch.tensor([0.2371], device="cuda")


@pytest.mark.parametrize("temp_kind", ["0.1", "1/3", "tensor0d", "tensor1"])
@pytest.mark.parametrize("B", [1, 255, 256, 257, 4099, 2 ** 20])
def test_sac_target_matches_eager_expression(B, temp_kind):
    from pfrl_b200.ops.sac import sac_target

    r, disc, term, q1, q2, lp = _sac_inputs(B, B)
    temp = _temperature(temp_kind)
    want = _eager_sac_target(r, disc, term, q1, q2, lp, temp)
    got = sac_target(r, disc, term, q1, q2, lp, temp)
    assert got.shape == want.shape == (B,)
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(got), nan)
    _same_bits(got[~nan], want[~nan], (B, temp_kind))
    if B >= len(_ROWS):
        assert nan.sum() >= 4  # the NaN rows really reach the output
    # against fp64 where the exact value is finite: five roundings of at most U relative
    # each, and at most 2^-150 absolute each in the subnormal range
    alpha = float(temp) if isinstance(temp, torch.Tensor) else temp
    q64 = torch.minimum(q1.double(), q2.double()).flatten()
    alp = alpha * lp.double()
    w = disc.double() * (1 - term.double())
    exact = r.double() + w * (q64 - alp)
    bound = 6 * U * (r.double().abs() + w.abs() * (q64.abs() + alp.abs())) + 4 * TINY
    fin = torch.isfinite(exact)
    err = (got.double() - exact).abs()
    bad = fin & ~(err <= bound)
    assert not bad.any(), (got[bad][:5], exact[bad][:5])


def test_sac_target_nan_rows():
    """One NaN Q head makes the target NaN, as torch.min does; the other head is not
    taken instead."""
    from pfrl_b200.ops.sac import sac_target

    q1 = torch.tensor([[_NAN], [1.0], [_NAN], [-_INF]], device="cuda")
    q2 = torch.tensor([[1.0], [_NAN], [_NAN], [_NAN]], device="cuda")
    ones = torch.ones(4, device="cuda")
    got = sac_target(ones * 0, ones * 0.99, ones * 0, q1, q2, ones * 0, 0.2)
    assert torch.isnan(got).all()


def test_sac_target_refusals(monkeypatch):
    """A CPU temperature or input is refused by the device checks before anything is
    launched; an empty batch returns an empty target without a launch."""
    from pfrl_b200.ops import sac as sac_ops

    def no_launch():
        raise AssertionError("sac_target reached the library")

    monkeypatch.setattr(sac_ops._lib, "load", no_launch)
    r, disc, term, q1, q2, lp = _sac_inputs(64, 0)
    with pytest.raises(ValueError):
        sac_ops.sac_target(r, disc, term, q1, q2, lp, torch.tensor(0.2))
    with pytest.raises(ValueError):
        sac_ops.sac_target(r, disc, term, q1.cpu(), q2, lp, 0.2)
    with pytest.raises(ValueError):
        sac_ops.sac_target(r.cpu(), disc.cpu(), term.cpu(), q1.cpu(), q2.cpu(), lp.cpu(), 0.2)
    e = torch.empty(0, device="cuda")
    out = sac_ops.sac_target(e, e, e, e[:, None], e[:, None], e, torch.tensor(0.2, device="cuda"))
    assert out.shape == (0,) and out.is_cuda and out.dtype == torch.float32
    assert _eager_sac_target(e, e, e, e[:, None], e[:, None], e, 0.2).shape == (0,)


# ---- agent level ----------------------------------------------------------------

OBS, ACT = 11, 3


def _squashed(x):
    from torch import distributions

    mean, log_scale = torch.chunk(x, 2, dim=1)
    base = distributions.Independent(
        distributions.Normal(mean, torch.exp(torch.clamp(log_scale, -20, 2))), 1)
    return distributions.transformed_distribution.TransformedDistribution(
        base, [distributions.transforms.TanhTransform(cache_size=1)])


def _qf(batchnorm=False):
    from pfrl_b200 import nn as pnn

    layers = [pnn.ConcatObsAndAction(), nn.Linear(OBS + ACT, 32)]
    if batchnorm:
        layers.append(nn.BatchNorm1d(32))
    return nn.Sequential(*layers, nn.ReLU(), nn.Linear(32, 1))


def _det_policy():
    from pfrl_b200 import policies

    return nn.Sequential(nn.Linear(OBS, 32), nn.ReLU(), nn.Linear(32, ACT), nn.Tanh(),
                         policies.DeterministicHead())


def _make_agent(kind, seed=0, **kw):
    from pfrl_b200 import agents, explorers, nn as pnn
    from pfrl_b200.replay_buffers import ReplayBuffer
    from pfrl_b200.utils import set_random_seed
    from pfrl_b200.utils.phi import Identity

    set_random_seed(seed)
    adam = lambda m: torch.optim.Adam(m.parameters(), lr=3e-3)  # noqa: E731
    common = dict(replay_start_size=64, minibatch_size=32, phi=Identity(), gpu=0)
    if kind == "sac":
        policy = nn.Sequential(nn.Linear(OBS, 32), nn.ReLU(), nn.Linear(32, 2 * ACT),
                               pnn.Lambda(_squashed))
        q1, q2 = _qf(batchnorm=True), _qf()
        kw.setdefault("entropy_target", -ACT)
        return agents.SoftActorCritic(policy, q1, q2, adam(policy), adam(q1), adam(q2),
                                      ReplayBuffer(4096), gamma=0.99, soft_update_tau=0.37,
                                      temperature_optimizer_lr=3e-3, **common, **kw)
    ex = explorers.AdditiveGaussian(0.3, -1, 1)
    if kind == "td3":
        p, q1, q2 = _det_policy(), _qf(), _qf(batchnorm=True)
        return agents.TD3(p, q1, q2, adam(p), adam(q1), adam(q2), ReplayBuffer(4096), 0.99, ex,
                          soft_update_tau=1 / 3, **common)
    p, q = _det_policy(), _qf(batchnorm=True)
    return agents.DDPG(p, q, adam(p), adam(q), ReplayBuffer(4096), 0.99, ex,
                       target_update_method="soft", target_update_interval=1,
                       soft_update_tau=0.05, **common)


def _train(agent, steps, seed=1):
    from pfrl_b200.envs import SyntheticContinuousVectorEnv

    env = SyntheticContinuousVectorEnv(4, OBS, ACT, device="cuda", seed=seed, mean_episode_len=20)
    obs = env.reset()
    for _ in range(steps):
        a = agent.batch_act(obs)
        obs, r, d, info = env.step(a)
        agent.batch_observe(obs, r, d, np.zeros(4, dtype=bool))
        obs = env.reset(np.logical_not(d))


def _sync_pairs(agent, kind):
    if kind == "sac":
        return [(agent.q_func1, agent.target_q_func1), (agent.q_func2, agent.target_q_func2)]
    if kind == "td3":
        return [(agent.policy, agent.target_policy), (agent.q_func1, agent.target_q_func1),
                (agent.q_func2, agent.target_q_func2)]
    return [(agent.model, agent.target_model)]


@pytest.mark.parametrize("kind", ["sac", "td3", "ddpg"])
def test_agent_target_sync_matches_reference(kind):
    agent = _make_agent(kind)
    pairs = _sync_pairs(agent, kind)
    start = [[v.clone() for v in dst.state_dict().values()] for _, dst in pairs]
    _train(agent, 40)  # 64 transitions to start, then one update per env step
    for (_, dst), before in zip(pairs, start):  # the updates really moved the targets
        assert any(not torch.equal(a, b) for a, b in zip(dst.state_dict().values(), before))
    clones = [(copy.deepcopy(src), copy.deepcopy(dst)) for src, dst in pairs]
    agent.sync_target_network()
    for src_c, dst_c in clones:
        reference_soft_copy(dst_c, src_c, agent.soft_update_tau)
    for (_, dst), (_, dst_c) in zip(pairs, clones):
        for (k, a), b in zip(dst.state_dict().items(), dst_c.state_dict().values()):
            _same_bits(a, b, (kind, k))
        for k, v in dst.state_dict().items():
            if k.endswith("num_batches_tracked"):
                assert int(v) == 0, k  # the target's own count, never the source's


def _batch(B, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return dict(
        state=torch.randn(B, OBS, generator=g, device="cuda"),
        next_state=torch.randn(B, OBS, generator=g, device="cuda"),
        action=torch.rand(B, ACT, generator=g, device="cuda") * 2 - 1,
        reward=torch.randn(B, generator=g, device="cuda"),
        discount=torch.full((B,), 0.99, device="cuda") ** torch.randint(
            1, 4, (B,), generator=g, device="cuda"),
        is_state_terminal=(torch.rand(B, generator=g, device="cuda") < 0.2).float())


@pytest.mark.parametrize("temperature", ["fixed", "learned"])
def test_sac_update_q_func_kernel_target_matches_eager(temperature, monkeypatch):
    """update_q_func with k_sac_target gives bit-equal Q parameters to the same update
    with the reference's eager target expression."""
    from pfrl_b200.ops import sac as sac_ops

    kw = dict(entropy_target=None, initial_temperature=0.1) if temperature == "fixed" else {}
    results = []
    for eager in (False, True):
        if eager:
            monkeypatch.setattr(sac_ops, "sac_target", _eager_sac_target)
        agent = _make_agent("sac", seed=5, **kw)
        torch.manual_seed(11)
        for step in range(3):
            agent.update_q_func(_batch(96, step))
            if agent.temperature_holder is not None:
                agent.update_temperature(torch.randn(96, device="cuda"))
        torch.cuda.synchronize()
        results.append([p.detach().clone() for q in (agent.q_func1, agent.q_func2)
                        for p in q.state_dict().values()])
    for a, b in zip(*results):
        _same_bits(a, b, temperature)
