"""The bytes of every sampled experience against what was appended, on every device
gather path, across part layouts, dtypes, stacks, actions, n-step episodes, batch
sizes and ring wrap.

The same transitions go into a device buffer and into HostReplayBuffer, which keeps
object references and follows the reference's n-step windows
(pfrl/replay_buffers/replay_buffer.py:33-76).  For each sample the expected batch is
the host algorithm, batch_experiences over ``host.memory[i]`` for the sampled logical
indices ``exps.index``; every field must be equal bit for bit, with the same dtype and
shape.  Exact equality is the right bar: observations and actions are byte copies,
U8_TO_F32 rounds one f32 multiply like ScaleU8 on the host, and the n-step reward is
the CPython float sum the kernels restate.

Paths: ReplayBuffer (k_gather with logical indices), PrioritizedReplayBuffer with
fused=False (k_gather through the pending sample's slots) and with fused=True, exact
and parallel (k_replay_step's gather workers; the first sample of a buffer is not
fused, the later ones are).  Part sizes run from 16 B to 112 896 B, so the fused
step's multi-piece path (parts cut into ceil(part_bytes / 8192) pieces) runs with
1, 2, 4 and 14 pieces (test_every_piece_count_ran).
"""
import numpy as np
import pytest
import torch

from pfrl_b200 import _lib
from pfrl_b200.replay_buffer import batch_experiences
from pfrl_b200.replay_buffers import HostReplayBuffer, PrioritizedReplayBuffer, ReplayBuffer
from pfrl_b200.utils.lazy_frames import LazyFrames
from pfrl_b200.utils.phi import Identity, RawU8, ScaleU8

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GAMMA = 0.97
PIECE_MAX = 8192  # step.cu: parts above this many bytes are cut into pieces
MAX_BATCH = 4100

PHIS = {"scale": ScaleU8, "raw": RawU8, "id": Identity}
ACTIONS = {  # name -> (dtype, shape); shape () is a Python int
    "int": (np.int64, ()),
    "f32x6": (np.float32, (6,)),
    "f32x17": (np.float32, (17,)),
    "f32x64": (np.float32, (64,)),   # 256 B, the largest action a record holds
    "f64x3": (np.float64, (3,)),
}

# name: (part dtype, part shape, stack, phi, action, n_step, n_envs, batch, capacity, cuda parts)
# stack 1 stores plain arrays, stack > 1 LazyFrames(stack_axis=0) over shared frames.
CASES = {
    "u8x16": (np.uint8, (16,), 1, "scale", "int", 1, 2, 1, 37, False),
    "f32x17-stack4": (np.float32, (17,), 4, "id", "f32x17", 3, 3, 33, 37, True),
    "u8x10x10-stack4": (np.uint8, (10, 10), 4, "scale", "f32x6", 8, 2, 257, 1000, False),
    "u8x10x10-stack8-raw": (np.uint8, (10, 10), 8, "raw", "int", 3, 3, 4097, 5000, True),
    "f64x7-stack4": (np.float64, (7,), 4, "id", "f64x3", 3, 2, 4097, 5000, False),
    "u8x16-stack8": (np.uint8, (16,), 8, "scale", "f32x64", 8, 3, 4097, 5000, False),
    "u8x84x84-stack4": (np.uint8, (1, 84, 84), 4, "scale", "int", 3, 3, 257, 1000, False),
    "u8x8192": (np.uint8, (8192,), 1, "scale", "f64x3", 1, 2, 33, 37, True),
    "f32x2048-stack8": (np.float32, (2048,), 8, "id", "f32x64", 8, 3, 33, 300, True),
    "u8x8208-stack4": (np.uint8, (8208,), 4, "scale", "f32x17", 3, 2, 257, 1000, False),
    "u8x8208-raw": (np.uint8, (8208,), 1, "raw", "f32x6", 1, 3, 33, 37, False),
    "f16x4104": (np.float16, (4104,), 1, "id", "int", 8, 2, 1, 37, False),
    "i32x2052-stack4": (np.int32, (2052,), 4, "id", "f32x6", 1, 3, 257, 300, True),
    "u8x4x84x84": (np.uint8, (4, 84, 84), 1, "scale", "int", 3, 3, 257, 300, True),
    "u8x4x84x84-raw": (np.uint8, (4, 84, 84), 1, "raw", "f32x64", 8, 2, 33, 37, False),
    "f32x4x84x84": (np.float32, (4, 84, 84), 1, "id", "f64x3", 3, 3, 33, 37, False),
}
PATHS = ["uniform", "per-separate", "per-fused-exact", "per-fused-parallel"]

FUSED_RAN = set()  # (obs_mode, pieces) of fused gathers that were checked


def _part_bytes(case):
    dtype, shape = case[0], case[1]
    nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
    return (nbytes + 15) // 16 * 16


def _pieces(part_bytes):
    return -(-part_bytes // PIECE_MAX)


def _obs_mode(phi_name):
    return _lib.OBS_U8_TO_F32 if phi_name == "scale" else _lib.OBS_RAW


def _np(x):
    """Host array of an observation: plain array, CUDA tensor or LazyFrames of either."""
    frames = getattr(x, "_frames", None)
    if frames is not None:
        return np.concatenate([_np(f) for f in frames], axis=0)
    if isinstance(x, torch.Tensor):
        return x.cpu().numpy()
    return np.asarray(x)


def _host_batch_states(xs, device, phi):
    return torch.as_tensor(np.stack([phi(_np(x)) for x in xs])).to(device)


class _Source:
    """Seeded transitions of one layout: per env, a stack of shared frames with one new
    frame per step; episodes end in a terminal or in stop_current_episode, and a new
    episode starts from one reset frame repeated `stack` times (one object)."""

    def __init__(self, case, seed):
        (self.dtype, self.shape, self.stack, _, act, self.n_step, self.n_envs, _, _,
         self.cuda) = case
        self.act_dtype, self.act_shape = ACTIONS[act]
        self.rng = np.random.RandomState(seed)
        self.frames = [None] * self.n_envs
        self.left = [0] * self.n_envs
        self.t = 0

    def _frame(self):
        r = self.rng
        if self.dtype == np.uint8:
            a = r.randint(0, 256, self.shape, dtype=np.uint8)
        elif self.dtype == np.int32:
            a = r.randint(-2 ** 31, 2 ** 31, self.shape, dtype=np.int64).astype(np.int32)
        else:
            a = (r.randn(*self.shape) * 3).astype(self.dtype)
        return torch.from_numpy(a).to(DEV) if self.cuda else a

    def _obs(self, frames):
        return LazyFrames(list(frames), stack_axis=0) if self.stack > 1 else frames[0]

    def step(self, bufs):
        env = self.t % self.n_envs
        self.t += 1
        r = self.rng
        if self.left[env] == 0:
            f = self._frame()
            self.frames[env] = [f] * self.stack
            self.left[env] = int(r.randint(1, 3 * self.n_step + 6))
        s = self._obs(self.frames[env])
        self.frames[env] = self.frames[env][1:] + [self._frame()]
        ns = self._obs(self.frames[env])
        if self.act_shape == ():
            a = int(r.randint(18))
        else:
            a = r.randn(*self.act_shape).astype(self.act_dtype)
        rew = float(r.randn()) * 10.0 ** int(r.randint(-3, 4))
        self.left[env] -= 1
        end = self.left[env] == 0
        term = end and r.rand() < 0.5
        for b in bufs:
            b.append(s, a, rew, ns, is_state_terminal=term, env_id=env)
            if end and not term:
                b.stop_current_episode(env_id=env)


def _make(path, cap, n_step, part_capacity):
    kw = dict(num_steps=n_step, part_capacity=part_capacity, max_batch=MAX_BATCH)
    if path == "uniform":
        return ReplayBuffer(cap, **kw)
    return PrioritizedReplayBuffer(
        cap, alpha=0.6, beta0=0.4, betasteps=100, normalize_by_max="memory",
        sample_mode="parallel" if path.endswith("parallel") else "exact",
        fused=path.startswith("per-fused"), **kw)


def _bits(t):
    return t.detach().contiguous().view(torch.uint8).cpu()


def _assert_batch_equal(got, want, idx, tag):
    for k in ("state", "next_state", "action", "reward", "discount", "is_state_terminal"):
        g, w = got[k], want[k]
        assert g.dtype == w.dtype, (tag, k, g.dtype, w.dtype)
        assert tuple(g.shape) == tuple(w.shape), (tag, k, tuple(g.shape), tuple(w.shape))
        gb, wb = _bits(g).reshape(g.shape[0], -1), _bits(w).reshape(w.shape[0], -1)
        bad = torch.nonzero((gb != wb).any(dim=1)).flatten().tolist()
        assert not bad, "%s: %s differs in %d rows, first rows %s (logical indices %s)" % (
            tag, k, len(bad), bad[:4], [int(idx[i]) for i in bad[:4]])


def _assert_materialised_equal(exps, host, idx, tag):
    """Indexing a sample materialises the reference's list-of-dicts through the gather with
    want_steps (per-step rewards and len): every transition's reward, the n-step length,
    the terminal flag, the first state / action and the last next_state."""
    got = list(exps)
    for k, i in enumerate(idx):
        e = host.memory[int(i)]
        g = got[k]
        assert len(g) == len(e), (tag, k)
        assert [t["reward"] for t in g] == [float(t["reward"]) for t in e], (tag, k)
        assert [t["is_state_terminal"] for t in g] == [bool(t["is_state_terminal"]) for t in e]
        assert np.array_equal(g[0]["state"], _np(e[0]["state"])), (tag, k)
        assert np.array_equal(g[-1]["next_state"], _np(e[-1]["next_state"])), (tag, k)
        assert np.array_equal(np.asarray(g[0]["action"]), np.asarray(e[0]["action"])), (tag, k)


def run_case(name, path):
    case = CASES[name]
    dtype, shape, stack, phi_name, act, n_step, n_envs, batch, cap, cuda = case
    part_bytes = _part_bytes(case)
    pieces = _pieces(part_bytes)
    phi = PHIS[phi_name]()
    print("layout: path=%s part_bytes=%d pieces=%d stack=%d obs=%s%s phi=%s action=%s "
          "n_step=%d envs=%d batch=%d capacity=%d parts=%s" % (
              path, part_bytes, pieces, stack, np.dtype(dtype).name, shape, phi_name, act,
              n_step, n_envs, batch, cap, "cuda" if cuda else "numpy"))
    # a part ring about twice the live window: it wraps several times over the run while
    # every live experience's parts stay in it (else sample() raises MemoryError)
    part_capacity = 2 * cap + 8 * stack + 64
    buf = _make(path, cap, n_step, part_capacity)
    host = HostReplayBuffer(cap, num_steps=n_step)
    src = _Source(case, seed=len(name) * 1000 + PATHS.index(path))
    nslots = 2
    while nslots < 2 * cap:
        nslots *= 2
    # the record ring (2P slots) and the part ring both wrap
    while len(host.memory) < cap or src.t < max(nslots + cap, 3 * part_capacity):
        src.step((buf, host))
    fused = path.startswith("per-fused")
    rounds = 4 if fused else 2
    g = torch.Generator(device=DEV).manual_seed(7)
    for r in range(rounds):
        np.random.seed(100 + r)
        exps = buf.sample(batch)
        if fused:
            assert (exps._prefetched is not None) == (r > 0), "fused step ran iff r > 0"
        idx = exps.index.cpu().numpy()
        assert idx.shape == (batch,) and 0 <= idx.min() and idx.max() < len(host.memory)
        got = batch_experiences(exps, DEV, phi, GAMMA)
        want = batch_experiences([host.memory[int(i)] for i in idx], DEV, phi, GAMMA,
                                 batch_states=_host_batch_states)
        tag = "%s/%s round %d" % (name, path, r)
        _assert_batch_equal(got, want, idx, tag)
        if r == 0:
            _assert_materialised_equal(exps, host, idx, tag)
        if fused and r > 0:
            FUSED_RAN.add((_obs_mode(phi_name), pieces))
        if path != "uniform":
            buf.update_errors(torch.rand(batch, device=DEV, generator=g) * 2 + 0.01)
        for _ in range(int(src.rng.randint(1, 3 * n_envs * n_step + 20))):
            src.step((buf, host))  # appends between the rounds
    torch.cuda.synchronize()


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("name", list(CASES))
def test_sampled_data_equals_appended(name, path):
    run_case(name, path)


def test_every_piece_count_ran():
    """The fused cases gathered parts of 1, 2 and 4 pieces in both obs modes (U8_TO_F32
    with uint8 parts) and of 14 pieces in RAW.  Cases this session did not run (a
    selection of the module) run here."""
    want = {(m, p) for m in (_lib.OBS_U8_TO_F32, _lib.OBS_RAW) for p in (1, 2, 4)}
    want.add((_lib.OBS_RAW, 14))
    table = {(_obs_mode(c[3]), _pieces(_part_bytes(c))): n for n, c in CASES.items()}
    assert want <= set(table), sorted(want - set(table))
    for key in sorted(want - FUSED_RAN):
        run_case(table[key], "per-fused-exact")
    assert want <= FUSED_RAN, sorted(want - FUSED_RAN)
    print("fused gathers checked (obs_mode, pieces):", sorted(FUSED_RAN))


@pytest.mark.parametrize("act,n_step,batch", [("int", 3, 33), ("f32x17", 8, 4097),
                                              ("f64x3", 1, 257), ("f32x64", 3, 1)])
@pytest.mark.parametrize("mode", ["exact", "parallel"])
def test_fused_step_scalars_only(act, n_step, batch, mode):
    """DeviceReplayStore.step with want_obs=False (the scalar-only gather of the fused
    step, one thread per experience): action, reward, discount and terminal of every
    drawn index equal the host algorithm's."""
    cap = 5000
    case = (np.float32, (3,), 1, "id", act, n_step, 3, batch, cap, False)
    buf = _make("per-fused-" + mode, cap, n_step, 2 * cap + 64)
    host = HostReplayBuffer(cap, num_steps=n_step)
    src = _Source(case, seed=batch + n_step)
    while src.t < 3 * cap:
        src.step((buf, host))
    buf._flush()
    store = buf.store
    lay = buf.layout
    rng = np.random.RandomState(batch)
    for r in range(3):
        res = store.step(rng.random_sample(batch), buf._gamma_pow(GAMMA), 0.4, _lib.NORM_MEMORY,
                         mode=_lib.SAMPLE_EXACT if mode == "exact" else _lib.SAMPLE_PARALLEL,
                         action_dtype=lay.torch_action_dtype(), action_shape=lay.action_shape,
                         want_obs=False)
        assert "state" not in res and "next_state" not in res
        idx = res["index"].cpu().numpy()
        want = batch_experiences([host.memory[int(i)] for i in idx], DEV, Identity(), GAMMA,
                                 batch_states=_host_batch_states)
        for k in ("action", "reward", "discount", "is_state_terminal"):
            g, w = res[k], want[k]
            assert g.dtype == w.dtype and tuple(g.shape) == tuple(w.shape), k
            assert torch.equal(_bits(g), _bits(w)), (k, r)
        store.update_priorities(rng.rand(batch) + 0.01)
        for _ in range(50):
            src.step((buf, host))
        buf._flush()


@pytest.mark.parametrize("path", ["uniform", "per-separate"])
def test_gather_want_steps(path):
    """DeviceReplayStore.gather(want_steps=True): per-step rewards (fp64, zero past the
    experience's length) and len, which materialised samples and save() read."""
    n_step, cap, batch = 8, 1000, 513
    case = (np.uint8, (10, 10), 4, "raw", "f32x6", n_step, 3, batch, cap, False)
    buf = _make(path, cap, n_step, 2 * cap + 128)
    host = HostReplayBuffer(cap, num_steps=n_step)
    src = _Source(case, seed=11)
    while src.t < 3 * cap:
        src.step((buf, host))
    np.random.seed(5)
    exps = buf.sample(batch)
    idx = exps.index.cpu().numpy()
    out = buf._gather(exps, GAMMA, RawU8(), raw=True, want_steps=True)
    sr, ln = out["step_rewards"].cpu().numpy(), out["len"].cpu().numpy()
    assert out["step_rewards"].dtype == torch.float64 and sr.shape == (batch, n_step)
    assert out["len"].dtype == torch.uint8 and ln.shape == (batch,)
    for k, i in enumerate(idx):
        e = host.memory[int(i)]
        want = np.zeros(n_step)
        want[:len(e)] = [t["reward"] for t in e]
        assert ln[k] == len(e), k
        assert sr[k].tobytes() == want.tobytes(), k
    assert set(ln.tolist()) > {n_step}, "windows shorter than n_step at episode ends"
