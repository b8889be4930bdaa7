"""k_seq_gather (b2rl_replay_gather_sequences) against the host path on the same GPU.

The same transitions go into the device EpisodicReplayBuffer and into
HostEpisodicReplayBuffer; both sample from the same numpy stream, so they pick the
same episodes and starts.  The host path is batch_recurrent_experiences + pack_sequence
on cuda:0; the kernel's packed batch must be bit-equal to it.
"""
import numpy as np
import pytest
import torch
from torch.nn.utils.rnn import pack_sequence

import pfrl_b200
from pfrl_b200 import _lib, replay_buffers
from pfrl_b200.replay_buffer import batch_recurrent_experiences
from pfrl_b200.utils.lazy_frames import LazyFrames
from pfrl_b200.utils.phi import Identity, ScaleU8

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _fill(bufs, n_trans, seed, obs="vec", state="lstm", n_envs=3, max_ep=12):
    rng = np.random.RandomState(seed)
    left = [0] * n_envs
    frames = [[rng.randint(0, 256, (1, 84, 84), dtype=np.uint8) for _ in range(4)]
              for _ in range(n_envs)]
    for i in range(n_trans):
        env = i % n_envs
        if left[env] == 0:
            left[env] = int(rng.choice([1, 1, 2, 10, max_ep]))
        left[env] -= 1
        if obs == "vec":
            s, ns = (rng.randn(5).astype(np.float32) for _ in range(2))
        else:
            f = frames[env]
            s = LazyFrames(list(f), stack_axis=0)
            f.append(rng.randint(0, 256, (1, 84, 84), dtype=np.uint8))
            del f[0]
            ns = LazyFrames(list(f), stack_axis=0)
        if state == "lstm":
            rs, nrs = [tuple(torch.randn(2, 1, 8, device=DEV) for _ in range(2)) for _ in range(2)]
            if rng.rand() < 0.2:
                rs = None
        elif state == "rnn":
            rs, nrs = torch.randn(1, 1, 8, device=DEV), torch.randn(1, 1, 8, device=DEV)
        else:
            rs = nrs = None
        a, r, term = int(rng.randint(18)), float(rng.randn()) / 3, left[env] == 0
        for buf in bufs:
            buf.append(s, a, r, ns, is_state_terminal=term, env_id=env,
                       recurrent_state=rs, next_recurrent_state=nrs)
        if left[env] == 0:
            for buf in bufs:
                buf.stop_current_episode(env_id=env)


def _host_batch(episodes, phi):
    def bs(xs, device, phi_):
        return torch.as_tensor(np.stack([phi_(np.asarray(x)) for x in xs])).to(device)

    return batch_recurrent_experiences(sorted(episodes, key=len, reverse=True), DEV, phi, 0.99,
                                       batch_states=bs)


def _leaves(s):
    if s is None:
        return []
    if isinstance(s, tuple):
        return [y for x in s for y in _leaves(x)]
    return [s]


def _check(dev_b, host_b):
    for k in ("state", "next_state"):
        ref = pack_sequence(host_b[k])
        assert torch.equal(dev_b[k].batch_sizes, ref.batch_sizes), k
        assert dev_b[k].data.dtype == ref.data.dtype
        assert torch.equal(dev_b[k].data, ref.data), k
    for k in ("action", "reward", "is_state_terminal", "discount"):
        assert dev_b[k].dtype == host_b[k].dtype, k
        assert torch.equal(dev_b[k], host_b[k]), k
    for k in ("recurrent_state", "next_recurrent_state"):
        a, b = _leaves(dev_b[k]), _leaves(host_b[k])
        assert len(a) == len(b), k
        for x, y in zip(a, b):
            assert x.shape == y.shape and torch.equal(x, y), k


def _pair(capacity, n_trans, seed, **kw):
    host = replay_buffers.HostEpisodicReplayBuffer(capacity)
    dev = replay_buffers.EpisodicReplayBuffer(capacity, device=DEV,
                                              part_capacity=4 * capacity + 4096)
    _fill([host, dev], n_trans, seed, **kw)
    return host, dev


def _compare(host, dev, B, max_len, phi, reps=2):
    for rep in range(reps):
        np.random.seed(100 + rep)
        he = host.sample_episodes(B, max_len)
        np.random.seed(100 + rep)
        de = dev.sample_episodes(B, max_len)
        db = batch_recurrent_experiences(de.sorted_by_length(), DEV, phi, 0.99)
        _check(db, _host_batch(he, phi))


@pytest.fixture(scope="module")
def big_pair():
    # padded 20-byte observations, 2-layer LSTM (h, c), some None states; the store
    # wraps around and whole episodes are evicted
    host, dev = _pair(16000, 24000, seed=1, state="lstm", max_ep=90)
    assert dev.store.napp > dev._alloc_capacity and dev.n_episodes >= 512
    return host, dev


@pytest.mark.parametrize("B", [1, 2, 31, 32, 33, 512])
@pytest.mark.parametrize("max_len", [None, 1, 10, 80])
def test_vector_obs_lstm(big_pair, B, max_len):
    host, dev = big_pair
    _compare(host, dev, B, max_len, Identity())


@pytest.mark.parametrize("state", ["rnn", "none"])
@pytest.mark.parametrize("B", [2, 33])
def test_vector_obs_other_states(state, B):
    host, dev = _pair(500, 900, seed=7, state=state)
    _compare(host, dev, B, 10, Identity())


@pytest.mark.parametrize("scaled", [True, False])
@pytest.mark.parametrize("B,max_len", [(32, 10), (33, None), (1, 1)])
def test_lazyframes_atari(scaled, B, max_len):
    host, dev = _pair(400, 700, seed=11, obs="atari", state="lstm")
    phi = ScaleU8() if scaled else pfrl_b200.utils.phi.RawU8()
    _compare(host, dev, B, max_len, phi)


def test_invalid_arguments_raise():
    _, dev = _pair(200, 300, seed=3, state="none")
    dev._flush()
    live = dev.store.napp - dev.store.npop
    g = dev.store.gather_sequences
    with pytest.raises(_lib.B2rlError):
        g(np.zeros(0), np.zeros(0), np.zeros(0))                       # B = 0
    with pytest.raises(_lib.B2rlError):
        g([live], [1], [live + 1])                                      # outside the live range
    with pytest.raises(_lib.B2rlError):
        g([0], [5], [3])                                                # past the episode
    with pytest.raises(_lib.B2rlError):
        g([0, 10], [1, 2], [5, 20])                                     # unsorted
    with pytest.raises(_lib.B2rlError):
        g([-1], [1], [2])


def test_back_to_back_launches_equal_single_launches():
    host, dev = _pair(2000, 3000, seed=5, state="lstm", max_ep=40)
    rng = np.random.RandomState(0)
    calls = []
    for i in range(300):
        B = int(rng.choice([1, 3, 32, 100]))
        max_len = [None, 1, 10][i % 3]
        np.random.seed(i)
        calls.append(dev.sample_episodes(B, max_len).sorted_by_length())
    phi = Identity()
    together = [batch_recurrent_experiences(e, DEV, phi, 0.99) for e in calls]
    torch.cuda.synchronize()
    for e, b in zip(calls, together):
        alone = batch_recurrent_experiences(e, DEV, phi, 0.99)
        torch.cuda.synchronize()
        for k in ("state", "next_state"):
            assert torch.equal(alone[k].data, b[k].data)
        for k in ("action", "reward", "is_state_terminal"):
            assert torch.equal(alone[k], b[k])
        for x, y in zip(_leaves(alone["recurrent_state"]), _leaves(b["recurrent_state"])):
            assert torch.equal(x, y)
