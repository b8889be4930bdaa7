"""Every gathered sequence, recurrent state, reward and behaviour-policy row of the
device EpisodicReplayBuffer against what was appended, across observation layouts and
dtypes, actions, state structures and dtypes, eviction and ring wrap.

The oracle is a plain model of the reference's buffer (pfrl/replay_buffers/episodic.py)
kept in this file: it records every transition as given (observations materialised,
states cloned to the host in their own dtype, mu as appended), commits an episode when it
stops, drops whole oldest episodes while more than ``capacity`` transitions are live, and
samples from numpy's global stream as the reference does (sample_n_k over the live
episodes, then one randint per episode longer than max_len, in sample order).  The
expected batch is built with plain torch: a stable longest-first sort, pack_sequence,
fp32 rewards and terminals, actions in their appended dtype, and recurrent states
stacked on a new axis 1 with zeros for a None (None when every state on a side is None).

Each sample is checked bit for bit, with equal dtype and shape, through four paths:
  1. the packed batch (k_seq_gather, DeviceEpisodes.batch), every field;
  2. the materialised list-of-dicts view (exact Python-float rewards, the stored mu);
  3. sample(n) transitions (k_gather) against the model's live records in order;
  4. _rewards_f64_device and mu_rows of single (sub)episodes, including runs that
     straddle the end of the ring.
The same model checks run without a GPU over the numpy store in
tests/test_episodic_data_path_cpu.py.
"""
import collections
import dataclasses

import numpy as np
import pytest
import torch
from torch.nn.utils.rnn import pack_sequence

from pfrl_b200 import _lib
from pfrl_b200.replay_buffers import EpisodicReplayBuffer
from pfrl_b200.replay_buffers.episodic import DeviceEpisodes
from pfrl_b200.utils.lazy_frames import LazyFrames
from pfrl_b200.utils.phi import Identity, RawU8, ScaleU8
from pfrl_b200.utils.random import sample_n_k

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GAMMA = 0.97
REWARDS = (0.1, 1.0 / 3.0, -2.0 / 3.0, 1e-40, 0.0)  # none of them an fp32 value but 0.0


# ------------------------------------------------------------------ the model
class Model:
    """The reference's episodic buffer, transitions kept as appended."""

    def __init__(self, capacity):
        self.capacity = capacity
        self.current = collections.defaultdict(list)
        self.episodes = collections.deque()
        self.n_live = 0
        self.overlong = 0  # episodes longer than the whole buffer

    def append(self, env, rec):
        self.current[env].append(rec)
        if rec["is_state_terminal"]:
            self.stop(env)

    def stop(self, env):
        ep = self.current.pop(env, None)
        if not ep:
            return
        self.episodes.append(ep)
        self.n_live += len(ep)
        self.overlong += self.capacity is not None and len(ep) > self.capacity
        while self.capacity is not None and self.n_live > self.capacity:
            self.n_live -= len(self.episodes.popleft())

    def sample_episodes(self, n, max_len):
        eps = [self.episodes[i] for i in sample_n_k(len(self.episodes), n)]
        out = []
        for ep in eps:
            if max_len is not None and len(ep) > max_len:
                s = np.random.randint(0, len(ep) - max_len + 1)
                ep = ep[s:s + max_len]
            out.append(ep)
        return out

    def live(self):
        return [r for ep in self.episodes for r in ep]


def _host_state(s):
    if s is None:
        return None
    if isinstance(s, tuple):
        return tuple(_host_state(x) for x in s)
    if isinstance(s, np.ndarray):
        return torch.from_numpy(s.copy())
    return s.detach().cpu().clone()


def _concat(states):
    like = next((s for s in states if s is not None), None)
    if like is None:
        return None
    if isinstance(like, tuple):
        return tuple(_concat([None if s is None else s[i] for s in states])
                     for i in range(len(like)))
    return torch.stack([torch.zeros_like(like) if s is None else s for s in states], dim=1)


# ------------------------------------------------------------------ scenarios
@dataclasses.dataclass
class Scenario:
    obs: tuple          # ("vec", dtype, shape) | ("lazy", stack)
    action: str         # "int" | "np_int64" | "f32x6" | "f64x2"
    state: str          # "none" | "gru" | "lstm" | "nested8" | "np_lstm" | "np_f64" | "gru_f16"
    mu: str             # "none" | "cat" | "cat_f64" | "gauss"
    capacity: object
    n_trans: int
    n_envs: int
    lengths: tuple      # episode lengths to draw from
    phis: tuple
    unbounded: int = 0
    part_capacity: object = None


def _host_phi(x):
    return np.asarray(x, dtype=np.float64) * 0.5 - 3.0


PHIS = {"id": Identity(), "scale": ScaleU8(), "raw": RawU8(), "host": _host_phi}

SCENARIOS = {
    # padded 20 B parts, GRU, wraps a 6 000-record store more than twice, > 1024 episodes
    "f32x5-gru-big": Scenario(("vec", np.float32, (5,)), "int", "gru", "cat", 6000, 15500, 4,
                              (1, 1, 1, 2, 2, 3, 5) * 30 + (300,), ("id",)),
    "f32x376-nested8": Scenario(("vec", np.float32, (376,)), "f32x6", "nested8", "gauss", 777,
                                2200, 2, (1, 2, 7, 30, 90), ("id",)),
    "f32x3x64x64": Scenario(("vec", np.float32, (3, 64, 64)), "f64x2", "none", "none", None,
                            420, 3, (1, 5, 40, 120), ("id",), unbounded=512, part_capacity=1024),
    "f16x7-np-f64": Scenario(("vec", np.float16, (7,)), "np_int64", "np_f64", "cat_f64", 500,
                             1300, 3, (1, 3, 8, 20, 60), ("id",)),
    "f64x3-gru-f16": Scenario(("vec", np.float64, (3,)), "int", "gru_f16", "gauss", 301, 950, 1,
                              (1, 4, 17), ("id",)),
    "i32x6-np-lstm": Scenario(("vec", np.int32, (6,)), "f32x6", "np_lstm", "none", 250, 800, 4,
                              (1, 2, 6, 33), ("id",)),
    "u8x13-host-phi": Scenario(("vec", np.uint8, (13,)), "int", "lstm", "cat", 400, 1000, 2,
                               (1, 9, 40), ("host", "id")),
    "lazy4": Scenario(("lazy", 4), "int", "lstm", "cat", 300, 760, 2, (1, 3, 12, 50),
                      ("scale", "raw")),
    "lazy8": Scenario(("lazy", 8), "np_int64", "gru", "none", 200, 520, 3, (1, 5, 20),
                      ("raw", "scale")),
    # a 7-record ring rewritten hundreds of times between two flushes: only the last write
    # of a state or mu row may reach the device (torch's scatters leave duplicates unordered)
    "tiny-ring": Scenario(("vec", np.float32, (5,)), "int", "lstm", "cat", 7, 3000, 2, (1, 2, 3),
                          ("id",)),
    # an episode longer than the whole buffer empties it
    "overlong": Scenario(("vec", np.float32, (5,)), "int", "lstm", "cat", 100, 800, 1,
                         (150,) + (3, 7, 12, 20) * 3, ("id",)),
}


def _state(kind, rng, dev):
    """One recurrent state of the scenario's kind (None about 20 % of the time)."""
    if kind == "none" or rng.rand() < 0.2:
        return None
    g = lambda *shape: torch.from_numpy(rng.randn(*shape).astype(np.float32)).to(dev)  # noqa: E731
    if kind == "gru":
        return g(1, 1, 8)
    if kind == "gru_f16":
        return g(1, 1, 6).half()
    if kind == "lstm":
        return (g(2, 1, 8), g(2, 1, 8))
    if kind == "nested8":  # 8 leaves, some with inner > 1
        return ((g(2, 1, 3, 4), g(2, 1, 3, 4)), g(1, 1, 5), (g(3, 2), (g(1, 1, 1), g(4,))),
                (g(2, 1, 3, 4), g(1, 7, 2)))
    if kind == "np_lstm":
        return (rng.randn(2, 4).astype(np.float32), rng.randn(2, 4).astype(np.float32))
    if kind == "np_f64":  # doubles that fp32 cannot hold; the low words are arbitrary bits
        return (rng.randn(2, 1, 5), rng.randn(2, 1, 5) * 1e-310)
    raise ValueError(kind)


def _mu(kind, rng, dev):
    if kind == "none":
        return None
    D = torch.distributions
    if kind == "cat":
        return D.Categorical(logits=torch.from_numpy(rng.randn(1, 5).astype(np.float32)).to(dev))
    if kind == "cat_f64":
        return D.Categorical(logits=torch.from_numpy(rng.randn(1, 4)).to(dev))
    loc = torch.from_numpy(rng.randn(1, 3).astype(np.float32)).to(dev)
    scale = torch.from_numpy(rng.rand(1, 3).astype(np.float32) + 0.1).to(dev)
    return D.Independent(D.Normal(loc, scale), 1)


def _action(kind, rng):
    if kind == "int":
        return int(rng.randint(18))
    if kind == "np_int64":
        return np.int64(rng.randint(-5, 1 << 40))
    if kind == "f32x6":
        return rng.randn(6).astype(np.float32)
    return rng.randn(2)  # f64x2


def build(sc, seed, dev, buffer_cls=EpisodicReplayBuffer):
    """The scenario's transitions appended to a device buffer and to the model."""
    rng = np.random.RandomState(seed)
    kw = dict(device=dev)
    if sc.part_capacity is not None:
        kw["part_capacity"] = sc.part_capacity
    if sc.capacity is None:
        kw["unbounded_capacity"] = sc.unbounded
    buf = buffer_cls(sc.capacity, **kw)
    model = Model(sc.capacity)
    left = [0] * sc.n_envs
    cut = [False] * sc.n_envs     # the episode ends by stop_current_episode
    last = [None] * sc.n_envs     # the env's latest observation (shared with the next step)
    frames = [None] * sc.n_envs
    lengths = list(sc.lengths)
    for i in range(sc.n_trans):
        env = int(rng.randint(sc.n_envs))
        if left[env] == 0:
            left[env] = int(rng.choice(lengths))
            cut[env] = rng.rand() < 0.4
            last[env] = None
            if sc.obs[0] == "lazy":
                frames[env] = [rng.randint(0, 256, (1, 84, 84), dtype=np.uint8)
                               for _ in range(sc.obs[1])]
        left[env] -= 1
        if sc.obs[0] == "lazy":
            f = frames[env]
            s = LazyFrames(list(f), stack_axis=0)
            f.append(rng.randint(0, 256, (1, 84, 84), dtype=np.uint8))
            del f[0]
            ns = LazyFrames(list(f), stack_axis=0)
        else:
            _, dtype, shape = sc.obs
            new = lambda: (rng.randn(*shape) * 1000).astype(dtype)  # noqa: E731
            s = last[env] if last[env] is not None else new()
            ns = new()
            last[env] = ns
        a = _action(sc.action, rng)
        r = float(REWARDS[int(rng.randint(len(REWARDS)))] + (rng.randn() if rng.rand() < .5 else 0))
        end = left[env] == 0
        term = end and not cut[env]
        rs, nrs = _state(sc.state, rng, dev), _state(sc.state, rng, dev)
        mu = _mu(sc.mu, rng, dev)
        extra = dict(recurrent_state=rs, next_recurrent_state=nrs)
        if mu is not None:
            extra["mu"] = mu
        buf.append(s, a, r, ns, is_state_terminal=term, env_id=env, **extra)
        model.append(env, dict(state=np.array(s), action=a, reward=r, next_state=np.array(ns),
                               is_state_terminal=term, recurrent_state=_host_state(rs),
                               next_recurrent_state=_host_state(nrs), mu=mu))
        if end and not term:
            buf.stop_current_episode(env_id=env)
            model.stop(env)
    assert len(buf) == model.n_live and buf.n_episodes == len(model.episodes)
    assert [L for _, L, _ in buf._episodes] == [len(ep) for ep in model.episodes]
    return buf, model


# ------------------------------------------------------------------ comparisons
def _leaves(s):
    if s is None:
        return []
    if isinstance(s, tuple):
        return [y for x in s for y in _leaves(x)]
    return [s]


def _structure(s):
    if isinstance(s, tuple):
        return tuple(_structure(x) for x in s)
    return None if s is None else "leaf"


def same_bits(got, exp, what=""):
    got = torch.as_tensor(got).detach().cpu()
    exp = torch.as_tensor(exp).detach().cpu()
    assert got.dtype == exp.dtype, (what, got.dtype, exp.dtype)
    assert got.shape == exp.shape, (what, got.shape, exp.shape)
    assert torch.equal(got.contiguous().view(torch.uint8), exp.contiguous().view(torch.uint8)), what


def same_state(got, exp, what=""):
    assert _structure(got) == _structure(exp), what
    for x, y in zip(_leaves(got), _leaves(exp)):
        same_bits(x if isinstance(x, torch.Tensor) else torch.from_numpy(np.asarray(x)), y, what)


def same_mu(got, exp, what=""):
    """``got`` is the stored ``exp`` rebuilt from its parameters (a Categorical normalises
    its logits again, on the device that holds them)."""
    D = torch.distributions
    assert type(got) is type(exp), what
    if isinstance(exp, D.Categorical):
        same_bits(got.logits, D.Categorical(logits=exp.logits).logits, what)
    else:
        assert got.reinterpreted_batch_ndims == exp.reinterpreted_batch_ndims
        same_bits(got.base_dist.loc, exp.base_dist.loc, what)
        same_bits(got.base_dist.scale, exp.base_dist.scale, what)


def mu_row(mu):
    if isinstance(mu, torch.distributions.Categorical):
        return mu.logits.reshape(-1)
    return torch.cat([mu.base_dist.loc.reshape(-1), mu.base_dist.scale.reshape(-1)])


def _obs(recs, key, phi):
    return torch.from_numpy(np.stack([np.asarray(phi(r[key])) for r in recs]))


def _actions(recs):
    return torch.from_numpy(np.array([r["action"] for r in recs]))


def _rewards32(recs):
    return torch.from_numpy(np.array([r["reward"] for r in recs]).astype(np.float32))


def expected_batch(eps, phi):
    eps = sorted(eps, key=len, reverse=True)
    out = {}
    for k in ("state", "next_state"):
        out[k] = pack_sequence([_obs(ep, k, phi) for ep in eps])
    bs = out["state"].batch_sizes
    out["action"] = pack_sequence([_actions(ep) for ep in eps]).data
    out["reward"] = pack_sequence([_rewards32(ep) for ep in eps]).data
    out["is_state_terminal"] = pack_sequence([torch.tensor(
        [float(r["is_state_terminal"]) for r in ep], dtype=torch.float32) for ep in eps]).data
    out["discount"] = torch.full((int(bs.sum()),), GAMMA, dtype=torch.float32)
    out["recurrent_state"] = _concat([ep[0]["recurrent_state"] for ep in eps])
    out["next_recurrent_state"] = _concat([ep[0]["next_recurrent_state"] for ep in eps])
    return out


def check_packed(got, exp):
    for k in ("state", "next_state"):
        same_bits(got[k].batch_sizes, exp[k].batch_sizes, k + " batch_sizes")
        same_bits(got[k].data, exp[k].data, k)
    for k in ("action", "reward", "is_state_terminal", "discount"):
        same_bits(got[k], exp[k], k)
    for k in ("recurrent_state", "next_recurrent_state"):
        same_state(got[k], exp[k], k)


def check_transition(got, exp, what=""):
    same_bits(torch.from_numpy(np.asarray(got["state"])), torch.from_numpy(exp["state"]), what)
    same_bits(torch.from_numpy(np.asarray(got["next_state"])),
              torch.from_numpy(exp["next_state"]), what)
    a = exp["action"]
    if isinstance(a, int):
        assert type(got["action"]) is int and got["action"] == a, what
    elif np.ndim(a) == 0:
        assert got["action"] == a, what
    else:
        same_bits(torch.from_numpy(np.asarray(got["action"])), torch.from_numpy(a), what)
    assert type(got["reward"]) is float and got["reward"] == exp["reward"], what
    assert got["is_state_terminal"] == exp["is_state_terminal"], what
    assert got["next_action"] is None
    same_state(got["recurrent_state"], exp["recurrent_state"], what)
    same_state(got["next_recurrent_state"], exp["next_recurrent_state"], what)
    if exp["mu"] is None:
        assert "mu" not in got, what
    else:
        same_mu(got["mu"], exp["mu"], what)


def check_materialised(got_eps, exp_eps):
    assert len(got_eps) == len(exp_eps)
    for j, (g, e) in enumerate(zip(got_eps, exp_eps)):
        assert len(g) == len(e), j
        for t, (gt, et) in enumerate(zip(g, e)):
            check_transition(gt, et, (j, t))


def check_single(buf, de, sub, mu=True):
    """_rewards_f64_device and mu_rows of the one (sub)episode in ``de``."""
    rew = buf._rewards_f64_device(de)
    same_bits(rew, torch.tensor([r["reward"] for r in sub], dtype=torch.float64), "f64 rewards")
    if mu and buf._mu_layout is not None and all(r["mu"] is not None for r in sub):
        same_bits(buf.mu_rows(de), torch.stack([mu_row(r["mu"]) for r in sub]), "mu rows")


def check_sample_episodes(buf, model, B, max_len, phi, seed, materialise=True, mu=True):
    np.random.seed(seed)
    exp = model.sample_episodes(B, max_len)
    np.random.seed(seed)
    de = buf.sample_episodes(B, max_len)
    assert list(de.length) == [len(e) for e in exp]
    assert list(de.last_terminal) == [e[-1]["is_state_terminal"] for e in exp]
    srt = de.sorted_by_length()
    exp_sorted = sorted(exp, key=len, reverse=True)
    assert list(srt.last_terminal) == [e[-1]["is_state_terminal"] for e in exp_sorted]
    check_packed(srt.batch(GAMMA, phi), expected_batch(exp, phi))
    if materialise:
        check_materialised(list(de), exp)
    if B == 1:
        check_single(buf, de, exp[0], mu=mu)
    return de


def check_sample(buf, model, n, phi, seed):
    np.random.seed(seed)
    live = model.live()
    exp = [live[i] for i in sample_n_k(len(live), n)]
    np.random.seed(seed)
    exps = buf.sample(n)
    b = exps.batch(GAMMA, phi)
    for k in ("state", "next_state"):
        same_bits(b[k], _obs(exp, k, phi), k)
    same_bits(b["action"], _actions(exp), "action")
    same_bits(b["reward"], _rewards32(exp), "reward")
    same_bits(b["is_state_terminal"], torch.tensor(
        [float(r["is_state_terminal"]) for r in exp], dtype=torch.float32), "terminal")
    same_bits(b["discount"], torch.full((n,), GAMMA, dtype=torch.float32), "discount")
    for got, e in zip(exps, exp):
        assert len(got) == 1
        g = got[0]
        same_bits(torch.from_numpy(np.asarray(g["state"])), torch.from_numpy(e["state"]))
        same_bits(torch.from_numpy(np.asarray(g["next_state"])), torch.from_numpy(e["next_state"]))
        assert type(g["reward"]) is float and g["reward"] == e["reward"]
        assert g["is_state_terminal"] == e["is_state_terminal"]


def check_ring_wrap(buf, model, stride=1):
    """mu_rows and the fp64 rewards of every live episode (and a cut of it) that runs
    across the end of the ring; returns how many there were."""
    cap = buf._alloc_capacity
    n = 0
    for i, ((f, L, _), ep) in enumerate(zip(buf._episodes, model.episodes)):
        if f % cap + L <= cap or L < 2:
            continue
        n += 1
        for lo, hi in ((0, L), (1, L), (0, L - 1), (cap - f % cap - 1, cap - f % cap + 1)):
            if not 0 <= lo < hi <= L:
                continue
            de = DeviceEpisodes(buf, [f + lo], [hi - lo], [f + L])
            check_single(buf, de, ep[lo:hi])
    return n


def check_scenario(buf, model, sc, batch_sizes, seed=0):
    """Every (B, max_len, phi) of the scenario with B <= the live episodes, each sampled
    twice (the second launch reuses what the first allocated), then sample(n)."""
    n_eps = len(model.episodes)
    for phi in sc.phis:
        for B in batch_sizes:
            for max_len in MAX_LENS:
                if B > n_eps:
                    continue
                for rep in range(2):
                    seed += 1
                    check_sample_episodes(buf, model, B, max_len, PHIS[phi], seed,
                                          materialise=phi == sc.phis[0] and rep == 0)
        for n in (1, 33, 257):
            if n <= model.n_live:
                seed += 1
                check_sample(buf, model, n, PHIS[phi], seed)
    check_ring_wrap(buf, model)


def ring_wrap_case(dev, mu_kind, buffer_cls=EpisodicReplayBuffer):
    """Episodes of 4 in a 10-record buffer: the third one (records 8..11) and later ones
    run across the end of the ring, so mu_rows takes its two-slice branch."""
    rng = np.random.RandomState(3)
    buf, model = buffer_cls(10, device=dev), Model(10)
    straddled = 0
    for i in range(4 * 7):
        rec = dict(state=np.full(3, i, np.float32), action=i,
                   reward=REWARDS[i % len(REWARDS)] + i,
                   next_state=np.full(3, i + 1, np.float32), is_state_terminal=i % 4 == 3,
                   mu=_mu(mu_kind, rng, dev))
        buf.append(**rec)
        model.append(0, dict(rec, recurrent_state=None, next_recurrent_state=None))
        if i % 4 == 3:
            straddled += check_ring_wrap(buf, model)
    assert straddled >= 2
    return buf, model


def refusal_case(dev, buffer_cls=EpisodicReplayBuffer):
    """A refused mu or state leaves nothing behind: the episode keeps only the accepted
    transitions."""
    D = torch.distributions
    buf, model = buffer_cls(50, device=dev), Model(50)

    def rec(t, **kw):
        return dict(dict(state=np.full(5, t, np.float32), action=t, reward=0.1 * t,
                         next_state=np.full(5, t + 1, np.float32), is_state_terminal=False,
                         recurrent_state=torch.full((1, 1, 8), float(t), device=dev),
                         next_recurrent_state=None,
                         mu=D.Categorical(logits=torch.full((1, 5), float(t), device=dev))),
                    **kw)

    r = rec(0)
    buf.append(**r)
    model.append(0, r)
    with pytest.raises(NotImplementedError, match="Categorical"):
        buf.append(**rec(1, mu=D.Normal(torch.zeros(1, 5, device=dev),
                                        torch.ones(1, 5, device=dev))))
    with pytest.raises(AssertionError, match="layout"):
        buf.append(**rec(2, mu=D.Categorical(logits=torch.zeros(1, 4, device=dev))))
    with pytest.raises(AssertionError, match="layout"):
        buf.append(**rec(3, mu=D.Categorical(
            logits=torch.zeros(1, 5, device=dev, dtype=torch.float64))))
    with pytest.raises(TypeError, match="dtypes changed"):
        buf.append(**rec(4, recurrent_state=torch.zeros(1, 1, 8, dtype=torch.float64, device=dev)))
    with pytest.raises(AssertionError, match="layout changed"):
        buf.append(**rec(5, recurrent_state=torch.zeros(1, 1, 9, device=dev)))
    r = rec(6, is_state_terminal=True)
    buf.append(**r)
    model.append(0, r)
    assert len(buf) == model.n_live == 2
    check_sample_episodes(buf, model, 1, None, Identity(), seed=0)
    with pytest.raises(TypeError, match="dtypes"):
        buffer_cls(50, device=dev).append(**rec(0, recurrent_state=torch.zeros(
            2, 3, dtype=torch.int16, device=dev)))


# ------------------------------------------------------------------ GPU tests
_BUILT = {}


def scenario(name):
    if name not in _BUILT:
        _BUILT[name] = build(SCENARIOS[name], seed=sorted(SCENARIOS).index(name) + 1, dev=DEV)
    return _BUILT[name]


B_ALL = (1, 2, 31, 32, 33, 257, 1024)
MAX_LENS = (None, 1, 7, 80)


@pytest.mark.parametrize("max_len", MAX_LENS)
@pytest.mark.parametrize("B", B_ALL)
def test_big_store_every_batch_size(B, max_len):
    buf, model = scenario("f32x5-gru-big")
    assert buf.store.napp > 2 * buf._alloc_capacity and buf.n_episodes >= 1025
    assert max(len(ep) for ep in model.episodes) > 256
    for rep in range(2):  # the second launch reuses what the first allocated
        check_sample_episodes(buf, model, B, max_len, Identity(), seed=1000 * B + rep,
                              materialise=B <= 257 or rep == 0)


def test_big_store_samples_and_ring_wrap():
    buf, model = scenario("f32x5-gru-big")
    for n, seed in ((1, 1), (257, 2), (4000, 3)):
        check_sample(buf, model, n, Identity(), seed)
    check_ring_wrap(buf, model)
    for seed in range(40):
        check_sample_episodes(buf, model, 1, [None, 7, 80][seed % 3], Identity(), seed)


@pytest.mark.parametrize("name", [n for n in SCENARIOS if n != "f32x5-gru-big"])
def test_scenario(name):
    buf, model = scenario(name)
    check_scenario(buf, model, SCENARIOS[name], B_ALL)
    if name == "overlong":
        assert model.overlong > 0


@pytest.mark.parametrize("mu_kind", ["cat", "cat_f64", "gauss"])
def test_mu_rows_and_rewards_across_the_ring_end(mu_kind):
    ring_wrap_case(DEV, mu_kind)


@pytest.mark.parametrize("name", ["f16x7-np-f64", "f32x376-nested8", "lazy4"])
def test_save_load_gives_the_same_batches(name, tmp_path):
    buf, model = scenario(name)
    sc = SCENARIOS[name]
    buf.save(str(tmp_path / "buf.pkl"))
    back = EpisodicReplayBuffer(sc.capacity, device=DEV)
    back.load(str(tmp_path / "buf.pkl"))
    assert len(back) == len(buf) and back.n_episodes == buf.n_episodes
    phi = PHIS[sc.phis[0]]
    for seed, (B, max_len) in enumerate(((1, None), (7, 7), (min(257, buf.n_episodes), None))):
        a = check_sample_episodes(buf, model, B, max_len, phi, seed, materialise=False)
        # a saved Categorical is the rebuilt one, whose logits were normalised again
        b = check_sample_episodes(back, model, B, max_len, phi, seed, materialise=False,
                                  mu=sc.mu == "gauss")
        assert list(a.length) == list(b.length)
    for ea, eb in zip(buf._all_episodes(), back._all_episodes()):
        for ta, tb in zip(ea, eb):
            assert ("mu" in ta) == ("mu" in tb)
            if "mu" in ta:
                same_mu(tb["mu"], ta["mu"])
            same_state(tb["recurrent_state"], ta["recurrent_state"])
            same_state(tb["next_recurrent_state"], ta["next_recurrent_state"])


def test_fp64_states_and_mu_keep_their_dtype():
    # numpy states are fp64 unless asked otherwise; the ring used to round them to fp32
    buf, model = scenario("f16x7-np-f64")
    np.random.seed(5)
    de = buf.sample_episodes(3, None).sorted_by_length()
    b = de.batch(GAMMA, Identity())
    for leaf in _leaves(b["recurrent_state"]) + _leaves(b["next_recurrent_state"]):
        assert leaf.dtype == torch.float64
    assert buf.mu_rows(DeviceEpisodes(buf, de.first[:1], de.length[:1], de.end[:1])).dtype \
        == torch.float64
    check_sample_episodes(buf, model, 3, None, Identity(), seed=5)


def test_refused_appends_leave_nothing_behind():
    refusal_case(DEV)


def test_batch_size_limits_raise():
    buf, _ = scenario("f32x5-gru-big")
    with pytest.raises(_lib.B2rlError):
        buf.sample_episodes(0).batch(GAMMA, Identity())
    with pytest.raises(_lib.B2rlError):
        buf.sample_episodes(_lib.SEQ_MAX_B + 1).sorted_by_length().batch(GAMMA, Identity())
