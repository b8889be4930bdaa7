"""The n-step device buffers never hand out an experience whose observation part the
part ring has already overwritten: sample() raises MemoryError instead.

The real host logic of ReplayBuffer / PrioritizedReplayBuffer runs over
tests/fake_store.OracleBackedStore (a host copy of the part ring and the records), so
the data a sample returns can be compared with what was appended.  Every check below
is "either every live experience returns its own observations, or MemoryError":
the discriminating cases must raise, the realistic ones must not.
"""
import os
import sys
from unittest import mock

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))
from fake_store import OracleBackedStore  # noqa: E402

from pfrl_b200.replay_buffer import batch_experiences  # noqa: E402
from pfrl_b200.replay_buffers import HostReplayBuffer, PrioritizedReplayBuffer  # noqa: E402
from pfrl_b200.replay_buffers import ReplayBuffer  # noqa: E402
from pfrl_b200.utils.lazy_frames import LazyFrames  # noqa: E402
from pfrl_b200.utils.phi import Identity  # noqa: E402

CPU = torch.device("cpu")


@pytest.fixture(autouse=True)
def fake_store():
    with mock.patch("pfrl_b200.replay_buffers.device_buffer.DeviceReplayStore",
                    OracleBackedStore), \
            mock.patch("torch.cuda.current_device", return_value=0):
        yield


def _live_data_correct(buf, expected):
    """Sample every live experience of a uniform buffer and compare its state and
    next_state with ``expected`` (all experiences ever emitted, oldest first, as
    (state, next_state) arrays).  Raises MemoryError where the buffer does."""
    n = len(buf)
    exps = buf.sample(n)
    b = batch_experiences(exps, CPU, Identity(), 0.9)
    live = expected[len(expected) - n:]
    idx = exps.index.numpy()
    want_s = np.stack([np.asarray(live[i][0]) for i in idx])
    want_n = np.stack([np.asarray(live[i][1]) for i in idx])
    bad = [int(i) for j, i in enumerate(idx)
           if not (np.array_equal(b["state"][j].numpy(), want_s[j])
                   and np.array_equal(b["next_state"][j].numpy(), want_n[j]))]
    return bad


def _host_expected(host):
    return [(e[0]["state"], e[-1]["next_state"]) for e in host.memory]


def test_append_trajectory_overrun_raises():
    """60 trajectories of 7 frames (3 transitions, 1 experience each) into a 300-part
    ring: the oldest live experiences' frames are overwritten long before they are
    evicted.  Before this was checked, 18 of the 60 returned another trajectory's
    frames."""
    rng = np.random.RandomState(0)
    buf = ReplayBuffer(100, num_steps=3, part_capacity=300)
    expected, raised = [], None
    for i in range(60):
        frames = rng.randint(0, 256, (7, 16, 16), dtype=np.uint8)
        try:
            m = buf.append_trajectory(frames, np.zeros(3, np.int64), np.ones(3), None)
            assert m == 1
            expected.append((frames[0:4], frames[3:7]))
            bad = _live_data_correct(buf, expected)
        except MemoryError:
            raised = i
            break
        assert bad == [], "trajectory %d: experiences %s return other frames" % (i, bad[:5])
    # 7 frames per experience, 300 parts: the first one is overwritten in trajectory 42
    assert raised == 42
    with pytest.raises(MemoryError):
        buf.sample(1)


def test_trajectory_without_experience():
    """A trajectory shorter than n steps and without a terminal emits nothing (its tail
    is not emitted) and leaves the liveness window as it was."""
    buf = ReplayBuffer(10, num_steps=3, part_capacity=40)
    frames = np.zeros((6, 4, 4), dtype=np.uint8)
    assert buf.append_trajectory(frames, np.zeros(2, np.int64), np.ones(2)) == 0
    assert len(buf) == 0 and not buf._live_min_seq
    assert buf.append_trajectory(np.zeros((7, 4, 4), np.uint8), np.zeros(3, np.int64),
                                 np.ones(3)) == 1
    assert list(buf._live_min_seq) == [(0, 6)]


def test_reused_observation_overrun_raises():
    """170 fresh float32[32] observations into a 150-part ring, except that step 120
    hands out step 0's array again (an env with a cached reset observation).  The
    identity cache points experience 120 at part 0, which is overwritten at sequence
    150 while experience 120 is still live: sample() must raise, not return the new
    part."""
    rng = np.random.RandomState(1)
    buf = ReplayBuffer(100, num_steps=1, part_capacity=150)
    host = HostReplayBuffer(100, num_steps=1)
    obs = [rng.randn(32).astype(np.float32) for _ in range(171)]
    obs[120] = obs[0]
    raised = None
    for t in range(170):
        for b in (buf, host):
            b.append(obs[t], t, 1.0, obs[t + 1])
        try:
            bad = _live_data_correct(buf, _host_expected(host))
        except MemoryError:
            raised = t
            break
        assert bad == [], "step %d: experiences %s return another observation" % (t, bad[:5])
    # part 0 is overwritten by the append at step 150 (steps 119 / 120 upload nothing new);
    # the oldest live experience then is number 51, whose parts are still there
    assert raised == 150


def test_overrun_of_pending_window_raises():
    """Parts uploaded by appends that complete no experience (their n-step windows are
    still filling) also count: the check runs in sample() with nothing pending."""
    rng = np.random.RandomState(2)
    buf = ReplayBuffer(50, num_steps=8, part_capacity=40)
    obs = [rng.randn(4).astype(np.float32) for _ in range(60)]
    for t in range(8):
        buf.append(obs[t], 0, 0.0, obs[t + 1], env_id=0)   # experience 0: parts 0 .. 8
    buf.sample(1)
    for t in range(8, 39):
        buf.append(obs[t], 0, 0.0, obs[t + 1], env_id=1)   # parts 9 .. 39
        if t % 9 == 8:
            buf.stop_current_episode(env_id=1)
    buf.sample(1)
    assert buf._part_head == 40 and not buf._pend_exp
    for t in range(39, 45):
        buf.append(obs[t], 0, 0.0, obs[t + 1], env_id=2)   # no experience; part 0 is gone
    assert buf._part_head == 46 and not buf._pend_exp
    with pytest.raises(MemoryError):
        buf.sample(1)


@pytest.mark.parametrize("stack", [1, 4])
def test_part_ring_smaller_than_an_upload_batch(stack):
    """A part ring of fewer than 1024 parts (the pending-part batch): 600 appends before
    the first sample used to reach the store as one upload larger than the ring, which
    put_parts refuses.  Pending parts are uploaded before they exceed the ring, and every
    sample is exact."""
    rng = np.random.RandomState(3)
    cap = 37
    buf = ReplayBuffer(cap, num_steps=3, part_capacity=2 * cap + 8 * stack + 64)
    host = HostReplayBuffer(cap, num_steps=3)
    if stack == 1:
        obs = [rng.randn(5).astype(np.float32) for _ in range(601)]
        for t in range(600):
            for b in (buf, host):
                b.append(obs[t], t, 1.0, obs[t + 1], env_id=t % 2)
        assert _live_data_correct(buf, _host_expected(host)) == []
    else:
        _lazy_frames_run(buf, host, rng, 600, n_envs=3, check_every=600)
    assert buf._part_head > 3 * buf._part_capacity


def _lazy_frames_run(buf, host, rng, steps, n_envs, check_every, frame_shape=(1, 4, 4),
                     start=0):
    """Atari-style appends: per env a stack of 4 shared frames, one new frame per step,
    episode resets that repeat the reset frame 4 times (one object, like FrameStack)."""
    stacks = [None] * n_envs
    left = [0] * n_envs
    for t in range(start, start + steps):
        env = t % n_envs
        if left[env] == 0:
            f = rng.randint(0, 256, frame_shape, dtype=np.uint8)
            stacks[env] = [f] * 4
            left[env] = int(rng.randint(1, 60))
        s = LazyFrames(list(stacks[env]), stack_axis=0)
        stacks[env] = stacks[env][1:] + [rng.randint(0, 256, frame_shape, dtype=np.uint8)]
        ns = LazyFrames(list(stacks[env]), stack_axis=0)
        left[env] -= 1
        term = left[env] == 0 and rng.rand() < 0.5
        for b in (buf, host):
            b.append(s, int(rng.randint(6)), float(rng.randn()), ns, is_state_terminal=term,
                     env_id=env)
            if left[env] == 0 and not term:
                b.stop_current_episode(env_id=env)
        if (t + 1) % check_every == 0 and len(buf) > 0:
            bad = _live_data_correct(buf, _host_expected(host))
            assert bad == [], "step %d: experiences %s return other frames" % (t, bad[:5])


@pytest.mark.parametrize("cap,part_capacity", [(300, None), (300, 700), (1000, None)])
def test_lazyframes_appends_no_false_positive(cap, part_capacity):
    """The default part ring (2 * capacity + 4096) and a tighter one hold every live
    experience's frames through several ring wraps: no MemoryError, every sample exact."""
    rng = np.random.RandomState(cap)
    buf = ReplayBuffer(cap, num_steps=3, part_capacity=part_capacity)
    host = HostReplayBuffer(cap, num_steps=3)
    steps = 3 * (2 * cap + 4096 if part_capacity is None else part_capacity)
    _lazy_frames_run(buf, host, rng, steps, n_envs=3, check_every=997)
    assert buf._part_head > 2 * buf._part_capacity  # the ring wrapped at least twice


def test_save_load_then_append_no_false_positive(tmp_path):
    """A save / load round trip rebuilds the liveness window: appends after load() keep
    every sample exact, past several wraps of the part ring, without a MemoryError."""
    rng = np.random.RandomState(5)
    cap = 400
    buf = ReplayBuffer(cap, num_steps=3, part_capacity=900)
    host = HostReplayBuffer(cap, num_steps=3)
    _lazy_frames_run(buf, host, rng, 1500, n_envs=2, check_every=499)
    for env in range(2):  # save() keeps no unfinished n-step window
        buf.stop_current_episode(env_id=env)
        host.stop_current_episode(env_id=env)
    buf.save(str(tmp_path / "buf.npz"))
    other = ReplayBuffer(cap, num_steps=3, part_capacity=900)
    other.load(str(tmp_path / "buf.npz"))
    assert len(other) == len(host) == cap
    assert other._live_min_seq, "load() must rebuild the liveness window"
    assert _live_data_correct(other, _host_expected(host)) == []
    _lazy_frames_run(other, host, rng, 3000, n_envs=2, check_every=499, start=1500)
    assert other._part_head > 3 * 900


def test_save_load_keeps_the_minimum_of_a_reused_part(tmp_path):
    """The restored window keeps the minimum over all restored experiences: the last
    experience of the archive ends in the archive's first frame (the archive stores equal
    frames once), so it pins part 0 after load().  Appends that evict the oldest restored
    experiences and then overwrite part 0 while that last one is live must raise; the
    oldest live experience alone (parts 5 and 6) would not show it."""
    rng = np.random.RandomState(6)
    buf = ReplayBuffer(60, num_steps=1, part_capacity=200)
    f = [rng.randint(0, 256, (1, 4, 4), dtype=np.uint8) for _ in range(50)]
    for t in range(50):
        nxt = f[0] if t == 49 else f[t + 1]
        buf.append(LazyFrames([f[t]], stack_axis=0), 0, 0.0, LazyFrames([nxt], stack_axis=0))
    buf.save(str(tmp_path / "buf.npz"))
    other = ReplayBuffer(60, num_steps=1, part_capacity=61)
    other.load(str(tmp_path / "buf.npz"))
    assert other._part_head == 50 and len(other) == 50
    other.sample(1)
    g = [rng.randint(0, 256, (1, 4, 4), dtype=np.uint8) for _ in range(16)]
    for k in range(15):  # parts 50 .. 65; experiences 0 .. 4 are evicted
        other.append(LazyFrames([g[k]], stack_axis=0), 0, 0.0, LazyFrames([g[k + 1]], stack_axis=0))
    assert other._part_head == 66 and len(other) == 60
    with pytest.raises(MemoryError):
        other.sample(1)


def test_append_trajectory_bench_usage_no_false_positive():
    """append_trajectory as the benchmark fills its buffer: capacity + n - 1 transitions in
    chunks (4 stacking frames up front, a terminal at each chunk's end) into a ring of
    capacity + 4096 parts, then a wrap of more chunks; every experience exact."""
    rng = np.random.RandomState(7)
    cap, n_step, chunk = 6000, 3, 1 << 11
    buf = PrioritizedReplayBuffer(cap, num_steps=n_step, part_capacity=cap + 4096,
                                  normalize_by_max="memory", betasteps=None)
    uni = ReplayBuffer(cap, num_steps=n_step, part_capacity=cap + 4096)
    expected = []
    T = 3 * cap + n_step - 1
    done = 0
    while done < T:
        m = min(chunk, T - done)
        frames = rng.randint(0, 256, (m + 4, 4, 4), dtype=np.uint8)
        term = rng.rand(m) < 1e-3
        term[-1] = True
        acts = rng.randint(0, 18, size=m).astype(np.int64)
        rews = rng.randint(-1, 2, size=m).astype(np.float64)
        for b in (buf, uni):
            assert b.append_trajectory(frames, acts, rews, term) == m
        expected += [(frames[t:t + 4], None) for t in range(m)]
        done += m
        np.random.seed(done)
        exps = buf.sample(64)
        buf.update_errors(rng.rand(64).tolist())
        idx = exps.index.numpy()
        b = batch_experiences(exps, CPU, Identity(), 0.9)
        live = expected[len(expected) - len(buf):]
        assert np.array_equal(b["state"].numpy(), np.stack([live[i][0] for i in idx]))
        n = len(uni)
        e = uni.sample(n)
        s = batch_experiences(e, CPU, Identity(), 0.9)["state"].numpy()
        live = expected[len(expected) - n:]
        assert np.array_equal(s, np.stack([live[i][0] for i in e.index.numpy()]))
    assert buf._part_head > buf._part_capacity  # the ring wrapped
