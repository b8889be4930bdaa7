"""Recurrent DQN / DoubleDQN (DRQN) and the episodic replay buffers, without a GPU.

The device EpisodicReplayBuffer runs its real host logic (episode table, whole-episode
eviction, part liveness, recurrent-state ring, packing) over
tests/fake_episodic_store.EpisodicOracleStore; HostEpisodicReplayBuffer follows the
reference's EpisodicReplayBuffer (pfrl/replay_buffers/episodic.py).  The two must sample
the same episodes and starts from the same numpy stream and give the same batches.
"""
import pickle
from unittest import mock

import numpy as np
import pytest
import torch
from torch import nn
from torch.nn.utils.rnn import pack_sequence

import pfrl_b200
from fake_episodic_store import EpisodicOracleStore
from pfrl_b200 import replay_buffers
from pfrl_b200.nn import RecurrentBranched, RecurrentSequential
from pfrl_b200.q_functions import DiscreteActionValueHead
from pfrl_b200.replay_buffer import batch_recurrent_experiences, random_subseq
from pfrl_b200.utils import recurrent as R


@pytest.fixture
def fake_store():
    with mock.patch("pfrl_b200.replay_buffers.device_buffer.DeviceReplayStore",
                    EpisodicOracleStore), \
            mock.patch("torch.cuda.current_device", return_value=0):
        yield


# ---------------------------------------------------------------- helpers
def test_mask_get_concatenate():
    h = torch.arange(2 * 3 * 4, dtype=torch.float32).view(2, 3, 4)
    c = -h
    m = R.mask_recurrent_state_at((h, c), [0, 2])
    assert torch.equal(m[0][:, 1], h[:, 1]) and (m[0][:, [0, 2]] == 0).all()
    assert torch.equal(m[1][:, 1], c[:, 1])
    one = R.get_recurrent_state_at((h, c), 1, detach=True)
    assert one[0].shape == (2, 4)
    cat = R.concatenate_recurrent_states([one, None, one])
    assert cat[0].shape == (2, 3, 4)
    assert torch.equal(cat[0][:, 0], h[:, 1]) and (cat[0][:, 1] == 0).all()
    npcat = R.concatenate_recurrent_states([None, R.recurrent_state_as_numpy(one)])
    assert isinstance(npcat[1], np.ndarray) and npcat[1].shape == (2, 2, 4)
    assert R.concatenate_recurrent_states([None, None]) is None
    back = R.recurrent_state_from_numpy(npcat, torch.device("cpu"))
    assert torch.equal(back[0][:, 1], h[:, 1])
    assert R.mask_recurrent_state_at(None, [0]) is None
    with pytest.raises(ValueError):
        R.get_recurrent_state_at([h], 0, detach=False)
    assert R.detach_recurrent_state(None) is None


def test_flatten_and_pack_order():
    seqs = [[1, 2, 3], [4, 5], [6, 7], [8]]
    assert R.flatten_sequences_time_first(seqs) == [1, 4, 6, 8, 2, 5, 7, 3]
    ts = [torch.tensor(s, dtype=torch.float32) for s in seqs]
    assert pack_sequence(ts).data.tolist() == R.flatten_sequences_time_first(seqs)
    packed = R.pack_sequences_recursive([(t, t * 2) for t in ts])
    assert isinstance(packed, tuple) and torch.equal(packed[1].data, packed[0].data * 2)
    assert R.get_packed_sequence_info(packed)[0].tolist() == [4, 3, 1]
    assert R.pack_sequences_recursive(packed[0]) is packed[0]  # already packed


def _model(rnn="rnn", n_obs=5, n_act=3, hidden=6):
    torch.manual_seed(0)
    cell = nn.RNN(hidden, hidden) if rnn == "rnn" else nn.LSTM(hidden, hidden, num_layers=2)
    return RecurrentSequential(nn.Linear(n_obs, hidden), nn.ELU(), cell, nn.Linear(hidden, n_act),
                               DiscreteActionValueHead())


@pytest.mark.parametrize("rnn", ["rnn", "lstm"])
def test_recurrent_sequential_matches_step_by_step(rnn):
    model = _model(rnn)
    xs = [torch.randn(L, 5) for L in (4, 3, 3, 1)]
    av, rs = R.pack_and_forward(model, xs, None)
    # the same sequences one step at a time through one_step_forward
    for b, x in enumerate(xs):
        state = None
        for t in range(len(x)):
            y, state = R.one_step_forward(model, x[t:t + 1], state)
            row = sum(min(len(s), t) for s in xs) + b
            torch.testing.assert_close(y.q_values[0], av.q_values[row], rtol=1e-5, atol=1e-6)
    assert len(rs) == 1


def test_recurrent_branched():
    a, b = nn.LSTM(3, 4), nn.GRU(3, 2)
    br = RecurrentBranched(a, b)
    x = pack_sequence([torch.randn(2, 3), torch.randn(1, 3)])
    ys, rs = br(x, None)
    assert torch.equal(ys[0].data, a(x)[0].data) and torch.equal(ys[1].data, b(x)[0].data)
    assert isinstance(rs[0], tuple) and rs[1].shape == (1, 2, 2)
    assert R.is_recurrent(br) and not R.is_recurrent(nn.Linear(1, 1))


def test_random_subseq_draws_once_per_long_sequence():
    np.random.seed(3)
    assert random_subseq([1, 2], 3) == [1, 2]
    s = random_subseq(list(range(10)), 4)
    np.random.seed(3)
    i = np.random.randint(0, 7)
    assert s == list(range(i, i + 4))


def test_batch_recurrent_experiences_host_fixture():
    eps = [[dict(state=np.full(2, 10 * e + t, np.float32), action=t, reward=0.5 * t,
                 next_state=np.full(2, 10 * e + t + 1, np.float32), next_action=None,
                 is_state_terminal=t == L - 1,
                 recurrent_state=None if e == 1 else np.full((1, 3), e, np.float32),
                 next_recurrent_state=np.full((1, 3), -e, np.float32))
            for t in range(L)] for e, L in enumerate((3, 2, 2))]
    b = batch_recurrent_experiences(eps, torch.device("cpu"), lambda x: x, 0.9)
    assert b["action"].tolist() == [0, 0, 0, 1, 1, 1, 2]
    assert b["reward"].tolist() == [0.0, 0.0, 0.0, 0.5, 0.5, 0.5, 1.0]
    assert b["is_state_terminal"].tolist() == [0, 0, 0, 0, 1, 1, 1]
    assert torch.equal(b["discount"], torch.full((7,), 0.9))
    assert b["recurrent_state"].shape == (1, 3, 3)
    assert b["recurrent_state"][0, :, 0].tolist() == [0, 0, 2]
    assert len(b["state"]) == 3 and b["state"][0].shape == (3, 2)
    with pytest.raises(AssertionError):
        batch_recurrent_experiences(eps[::-1], torch.device("cpu"), lambda x: x, 0.9)


# ---------------------------------------------------------------- buffers
def _fill(bufs, n_steps, seed, n_envs=2, obs_dim=5, state="lstm"):
    """The same transitions into every buffer: per-env episodes of random length."""
    rng = np.random.RandomState(seed)
    left = [0] * n_envs
    for step in range(n_steps):
        for env in range(n_envs):
            if left[env] == 0:
                left[env] = int(rng.randint(1, 8))
            left[env] -= 1
            term = left[env] == 0 and rng.rand() < 0.7
            s = rng.randn(obs_dim).astype(np.float32)
            ns = rng.randn(obs_dim).astype(np.float32)
            if state == "lstm":
                rs = tuple(rng.randn(2, 4).astype(np.float32) for _ in range(2))
                nrs = tuple(rng.randn(2, 4).astype(np.float32) for _ in range(2))
                if rng.rand() < 0.2:
                    rs = None
            elif state == "rnn":
                rs, nrs = rng.randn(1, 4).astype(np.float32), rng.randn(1, 4).astype(np.float32)
            else:
                rs = nrs = None
            action, reward = int(rng.randint(3)), float(rng.randn())
            for buf in bufs:
                buf.append(state=s, action=action, reward=reward,
                           next_state=ns, is_state_terminal=term, env_id=env,
                           recurrent_state=rs, next_recurrent_state=nrs)
            if left[env] == 0:
                for buf in bufs:
                    buf.stop_current_episode(env_id=env)


def _same_batch(a, b):
    for k in ("action", "reward", "is_state_terminal", "discount"):
        assert torch.equal(a[k], b[k]), k
    for k in ("state", "next_state"):
        data = a[k].data if hasattr(a[k], "batch_sizes") else pack_sequence(a[k]).data
        ref = b[k].data if hasattr(b[k], "batch_sizes") else pack_sequence(b[k]).data
        assert torch.equal(data, ref), k
    for k in ("recurrent_state", "next_recurrent_state"):
        fa = [] if a[k] is None else [x for x in _leaf_list(a[k])]
        fb = [] if b[k] is None else [x for x in _leaf_list(b[k])]
        assert len(fa) == len(fb)
        for x, y in zip(fa, fb):
            assert torch.equal(x, y), k


def _leaf_list(s):
    if isinstance(s, tuple):
        return [y for x in s for y in _leaf_list(x)]
    return [s]


@pytest.mark.parametrize("state", ["lstm", "rnn", "none"])
@pytest.mark.parametrize("max_len", [None, 1, 3])
@pytest.mark.parametrize("capacity", [None, 40])
def test_device_buffer_equals_host_buffer(fake_store, state, max_len, capacity):
    host = replay_buffers.HostEpisodicReplayBuffer(capacity)
    dev = replay_buffers.EpisodicReplayBuffer(capacity, unbounded_capacity=4096)
    _fill([host, dev], 60, seed=1, state=state)
    assert len(host) == len(dev) and host.n_episodes == dev.n_episodes
    if capacity is not None:
        assert len(dev) <= capacity
    for rep in range(3):
        np.random.seed(rep)
        he = host.sample_episodes(5, max_len)
        np.random.seed(rep)
        de = dev.sample_episodes(5, max_len)
        assert [len(e) for e in he] == list(de.length)
        hs = sorted(he, key=len, reverse=True)
        hb = batch_recurrent_experiences(hs, torch.device("cpu"), None, 0.99,
                                         batch_states=_stack)
        db = batch_recurrent_experiences(de.sorted_by_length(), torch.device("cpu"),
                                         pfrl_b200.utils.phi.Identity(), 0.99)
        _same_batch(db, hb)
        # the materialised view is the reference's list of dicts
        for eh, ed in zip(he, de):
            assert [t["action"] for t in eh] == [t["action"] for t in ed]
            assert [t["reward"] for t in eh] == [t["reward"] for t in ed]
            assert all(np.array_equal(x["state"], y["state"]) for x, y in zip(eh, ed))
    np.random.seed(9)
    hs = host.sample(7)
    np.random.seed(9)
    ds = dev.sample(7)
    assert [t[0]["action"] for t in hs] == [t[0]["action"] for t in ds]


def _stack(xs, device, phi):
    return torch.as_tensor(np.stack([np.asarray(x) for x in xs]), device=device)


def test_whole_episode_eviction_and_env_separation(fake_store):
    for buf in (replay_buffers.HostEpisodicReplayBuffer(5),
                replay_buffers.EpisodicReplayBuffer(5)):
        obs = np.zeros(2, np.float32)
        for t in range(3):                       # env 0: episode of 3, interleaved with env 1
            buf.append(obs, 0, t, obs, env_id=0)
            buf.append(obs, 1, t, obs, env_id=1)
        assert len(buf) == 0 and buf.n_episodes == 0
        buf.stop_current_episode(env_id=1)
        assert len(buf) == 3 and buf.n_episodes == 1
        buf.append(obs, 0, 9, obs, is_state_terminal=True, env_id=0)   # commits env 0 (4)
        assert len(buf) == 4 and buf.n_episodes == 1                    # env 1's episode evicted
        ep = buf.sample_episodes(1)[0]
        assert [t["reward"] for t in ep] == [0, 1, 2, 9]
        buf.append(obs, 0, 5, obs, env_id=2)
        buf.stop_current_episode(env_id=2)
        assert len(buf) == 5 and buf.n_episodes == 2


def _frame(i):
    return np.full(2, i, np.float32)


def _short_episodes(buf, n):
    """n one-transition terminal episodes of env 1, two new parts each."""
    for _ in range(n):
        buf.append(_frame(-1), 0, 0.0, _frame(-2), is_state_terminal=True, env_id=1)


def test_part_liveness_counts_uncommitted_episodes(fake_store):
    """Only env 0's UNCOMMITTED long episode holds the old parts: the short episodes that
    were uploaded with them are evicted (capacity 3), so the oldest live record is recent.
    A check over live records alone would not raise here."""
    for pc, overrun in ((12, True), (64, False)):
        buf = replay_buffers.EpisodicReplayBuffer(3, part_capacity=pc)
        frames = [_frame(i) for i in range(3)]
        for t in range(2):                       # parts 0, 1, 2 (next_state shared)
            buf.append(frames[t], 0, 0.0, frames[t + 1], env_id=0)
        _short_episodes(buf, 10)                 # parts 3 .. 22; only the last 3 stay live
        assert buf._part_head == 23 and buf.n_episodes == 3
        live_oldest = min(seq for _, _, seq in buf._episodes)
        assert buf._part_head - live_oldest <= 12 < buf._part_head  # discriminating setup
        if overrun:
            with pytest.raises(MemoryError):
                buf.sample(1)
        else:
            buf.append(frames[2], 0, 0.0, _frame(3), is_state_terminal=True, env_id=0)
            ep = buf.sample_episodes(1)[0] if buf.n_episodes == 1 else None
            assert buf.n_episodes == 1 and [float(t["state"][0]) for t in ep] == [0, 1, 2]


def test_part_liveness_later_committed_episode_holds_the_minimum(fake_store):
    """Env 0's episode starts first and is committed after three short episodes: the
    oldest live part belongs to an episode that is not the oldest in commit order."""
    for pc, overrun in ((17, True), (64, False)):
        buf = replay_buffers.EpisodicReplayBuffer(20, part_capacity=pc)
        frames = [_frame(i) for i in range(6)]
        for t in range(4):                       # parts 0 .. 4
            buf.append(frames[t], 0, 0.0, frames[t + 1], env_id=0)
        _short_episodes(buf, 3)                  # parts 5 .. 10
        buf.append(frames[4], 0, 0.0, frames[5], is_state_terminal=True, env_id=0)  # part 11
        _short_episodes(buf, 4)                  # parts 12 .. 19
        assert buf._part_head == 20 and buf.n_episodes == 8
        first_committed = buf._episodes[0][2]
        assert buf._part_head - first_committed <= 17 < buf._part_head  # discriminating
        if overrun:
            with pytest.raises(MemoryError):
                buf.sample(1)
        else:
            ep = max(buf.sample_episodes(8), key=len)
            assert [float(t["state"][0]) for t in ep] == [0, 1, 2, 3, 4]


def _batches_equal(a, b):
    _same_batch(a, b)
    for k in ("recurrent_state", "next_recurrent_state"):
        assert (a[k] is None) == (b[k] is None), k


@pytest.mark.parametrize("state", ["lstm", "rnn"])
def test_save_load_round_trip(fake_store, tmp_path, state):
    """Every transition's states survive save / load: batches of windows that start
    mid-episode (max_len 2) are equal before and after, on both state sides."""
    host = replay_buffers.HostEpisodicReplayBuffer(50)
    dev = replay_buffers.EpisodicReplayBuffer(50)
    _fill([host, dev], 40, seed=4, state=state)
    phi = pfrl_b200.utils.phi.Identity()
    for buf, cls in ((host, replay_buffers.HostEpisodicReplayBuffer),
                     (dev, replay_buffers.EpisodicReplayBuffer)):
        buf.save(str(tmp_path / "b.pkl"))
        other = cls(50)
        other.load(str(tmp_path / "b.pkl"))
        assert len(other) == len(buf) and other.n_episodes == buf.n_episodes
        mid = 0
        for seed in range(6):
            np.random.seed(seed)
            a = buf.sample_episodes(6, 2)
            np.random.seed(seed)
            b = other.sample_episodes(6, 2)
            if cls is replay_buffers.EpisodicReplayBuffer:
                starts = {f for f, _, _ in buf._episodes}
                mid += sum(int(f) not in starts for f in a.first)
                ba = batch_recurrent_experiences(a.sorted_by_length(), torch.device("cpu"),
                                                 phi, 0.9)
                bb = batch_recurrent_experiences(b.sorted_by_length(), torch.device("cpu"),
                                                 phi, 0.9)
            else:
                ba = batch_recurrent_experiences(sorted(a, key=len, reverse=True),
                                                 torch.device("cpu"), None, 0.9,
                                                 batch_states=_stack)
                bb = batch_recurrent_experiences(sorted(b, key=len, reverse=True),
                                                 torch.device("cpu"), None, 0.9,
                                                 batch_states=_stack)
            _batches_equal(ba, bb)
            for x, y in zip(a, b):
                for s, u in zip(x, y):
                    for key in ("recurrent_state", "next_recurrent_state"):
                        p, q = _leaf_list(s[key]) if s[key] is not None else [], \
                            _leaf_list(u[key]) if u[key] is not None else []
                        assert len(p) == len(q) and all(
                            np.array_equal(np.asarray(m), np.asarray(n)) for m, n in zip(p, q))
    assert mid > 0  # some windows start mid-episode
    # the device view carries each transition's own states, as the host buffer does
    np.random.seed(1)
    he = host.sample_episodes(8)
    np.random.seed(1)
    de = dev.sample_episodes(8)
    n_states = 0
    for x, y in zip(he, de):
        for s, u in zip(x, y):
            for key in ("recurrent_state", "next_recurrent_state"):
                assert (s[key] is None) == (u[key] is None)
                if s[key] is not None:
                    n_states += 1
                    assert all(np.array_equal(m, n) for m, n in
                               zip(_leaf_list(s[key]), _leaf_list(u[key])))
    assert n_states > 2 * len(he)  # later steps carry states too
    with open(tmp_path / "b.pkl", "rb") as f:
        assert isinstance(pickle.load(f), list)


def test_save_load_keeps_frame_sharing(fake_store, tmp_path):
    """Frame-stacked observations come back as LazyFrames sharing their frames: the loaded
    buffer has the same stack layout and uploads no more frames than it holds."""
    from pfrl_b200.utils.lazy_frames import LazyFrames

    rng = np.random.RandomState(0)
    buf = replay_buffers.EpisodicReplayBuffer(30)
    frames = [rng.randint(0, 256, (1, 6, 6), dtype=np.uint8) for _ in range(4)]
    for t in range(25):
        s = LazyFrames(list(frames), stack_axis=0)
        frames = frames[1:] + [rng.randint(0, 256, (1, 6, 6), dtype=np.uint8)]
        buf.append(s, t % 3, 0.0, LazyFrames(list(frames), stack_axis=0),
                   is_state_terminal=t % 6 == 5)
    buf.stop_current_episode()
    buf.save(str(tmp_path / "f.pkl"))
    other = replay_buffers.EpisodicReplayBuffer(30)
    other.load(str(tmp_path / "f.pkl"))
    assert other.layout.lazy and other.layout.stack == 4
    assert other._part_head <= len(buf) + 4 * other.n_episodes
    np.random.seed(0)
    a = buf.sample_episodes(3)
    np.random.seed(0)
    b = other.sample_episodes(3)
    for x, y in zip(a, b):
        assert all(np.array_equal(p["state"], q["state"]) and
                   np.array_equal(p["next_state"], q["next_state"]) for p, q in zip(x, y))


# ---------------------------------------------------------------- agents
def _agent(cls, rbuf, rnn="rnn", seed=0, **kw):
    torch.manual_seed(seed)
    q = _model(rnn, n_obs=5, n_act=2)
    opt = torch.optim.Adam(q.parameters(), 1e-2, eps=1)
    return cls(q, opt, rbuf, gamma=0.9, explorer=pfrl_b200.explorers.ConstantEpsilonGreedy(
        0.2, lambda: np.random.randint(2)), replay_start_size=30, minibatch_size=4,
        target_update_interval=20, recurrent=True, **kw)


def _run(agent, steps, seed, n_envs=2):
    from pfrl_b200.envs.abc import ABC

    np.random.seed(seed)
    envs = [ABC(size=2, discrete=True, partially_observable=True) for _ in range(n_envs)]
    for i, e in enumerate(envs):
        e.seed(seed + i) if hasattr(e, "seed") else None
    obs = [e.reset() for e in envs]
    obs = [np.resize(np.asarray(o, np.float32), 5) for o in obs]
    actions = []
    for t in range(steps):
        acts = agent.batch_act(obs)
        actions.append(list(map(int, acts)))
        res = [e.step(a) for e, a in zip(envs, acts)]
        nobs = [np.resize(np.asarray(r[0], np.float32), 5) for r in res]
        rew = [r[1] for r in res]
        done = [r[2] for r in res]
        reset = [d or (t + 1) % 11 == 0 for d in done]
        agent.batch_observe(nobs, rew, done, reset)
        obs = [np.resize(np.asarray(e.reset(), np.float32), 5) if r else o
               for e, r, o in zip(envs, reset, nobs)]
    return actions


@pytest.mark.parametrize("cls_name", ["DQN", "DoubleDQN"])
@pytest.mark.parametrize("rnn,ep_len", [("rnn", None), ("lstm", 3)])
def test_agent_device_buffer_equals_host_buffer(fake_store, cls_name, rnn, ep_len):
    cls = getattr(pfrl_b200.agents, cls_name)
    a = _agent(cls, replay_buffers.HostEpisodicReplayBuffer(60), rnn, episodic_update_len=ep_len)
    b = _agent(cls, replay_buffers.EpisodicReplayBuffer(60), rnn, episodic_update_len=ep_len,
               phi=pfrl_b200.utils.phi.Identity())
    acts_a = _run(a, 80, seed=5)
    acts_b = _run(b, 80, seed=5)
    assert a.optim_t > 10 and a.optim_t == b.optim_t
    assert acts_a == acts_b
    for p, q in zip(a.model.parameters(), b.model.parameters()):
        torch.testing.assert_close(p, q, rtol=1e-5, atol=1e-6)
    assert np.isfinite(a.get_statistics()[1][1])
    a.stop_episode()
    assert a.test_recurrent_states is None


def test_recurrent_refusals():
    from pfrl_b200.agents import (
        AL, IQN, PAL, CategoricalDoubleDQN, CategoricalDQN, DoublePAL, DPP, DQN,
    )

    q = _model()
    rb = replay_buffers.HostEpisodicReplayBuffer(10)
    opt = torch.optim.Adam(q.parameters())
    for cls in (CategoricalDQN, CategoricalDoubleDQN, IQN, AL, PAL, DoublePAL, DPP,
                pfrl_b200.agents.dpp.DPPL, pfrl_b200.agents.dpp.DPPGreedy):
        with pytest.raises(NotImplementedError):
            cls(q, opt, rb, 0.9, pfrl_b200.explorers.Greedy(), replay_start_size=5,
                minibatch_size=2, recurrent=True)
    for kw in (dict(cuda_graph=True), dict(grad_sync=lambda m: None)):
        with pytest.raises(ValueError):
            DQN(q, opt, rb, 0.9, pfrl_b200.explorers.Greedy(), replay_start_size=5,
                minibatch_size=2, recurrent=True, **kw)
    agent = DQN(q, opt, rb, 0.9, pfrl_b200.explorers.Greedy(), replay_start_size=5,
                minibatch_size=2, recurrent=True)
    with pytest.raises(AssertionError):
        agent.update_from_episodes([], errors_out=[])
