"""GPU: the fused single-launch replay step (b2rl_replay_step: deferred priority
write-back -> sample -> importance weights -> gather) gives bit for bit the
results of the separate launches (b2rl_per_sample, b2rl_per_weights,
b2rl_replay_gather, b2rl_per_update_errors), which the other GPU tests pin to the
oracle / the reference's golden traces.  Two buffers are driven with identical
appends, seeds and device-side TD errors; one has fused=True."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _fill_frames(buf, rng, n, hw=(12, 12)):
    frames = rng.randint(0, 256, size=(n + 4,) + hw, dtype=np.uint8)
    acts = rng.randint(0, 6, size=n).astype(np.int64)
    rews = rng.randint(-2, 3, size=n).astype(np.float64)
    term = rng.rand(n) < 0.02
    term[-1] = True
    buf.append_trajectory(frames, acts, rews, term)


def _fill_vectors(buf, rng, n, dim=17):
    obs = rng.randn(n + 1, dim).astype(np.float32)
    for t in range(n):
        buf.append(obs[t], rng.randn(6).astype(np.float32), float(rng.randn()), obs[t + 1], None,
                   bool(rng.rand() < 0.03))


CASES = [
    # capacity, kind, n_step, batch, mode, normalize_by_max, prefill
    (300, "frames", 3, 64, "exact", "memory", 500),       # tree in shared memory
    (20000, "vectors", 1, 256, "exact", True, 3000),      # deep tree (D = 3), padded parts
    (300000, "frames84", 3, 512, "exact", "memory", 9000),  # v6, D = 8, headline frame size
    (600, "frames", 2, 512, "parallel", False, 900),      # with replacement: duplicates
    (5000, "frames", 1, 700, "exact", "batch", 6000),     # batch > 512: write-back alone
    (5000, "frames", 3, 32, "parallel", "memory", 6000),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "%d-%s-%s" % (c[0], c[1], c[4]))
def test_fused_step_equals_separate_launches(case):
    from pfrl_b200.replay_buffer import batch_experiences
    from pfrl_b200.replay_buffers import PrioritizedReplayBuffer
    from pfrl_b200.utils.phi import Identity, ScaleU8

    capacity, kind, n_step, batch, mode, nb, prefill = case
    dev = torch.device("cuda")
    bufs = []
    for fused in (False, True):
        buf = PrioritizedReplayBuffer(capacity, alpha=0.5 if kind != "vectors" else 0.7,
                                      beta0=0.4, betasteps=50, normalize_by_max=nb,
                                      num_steps=n_step, max_batch=1024, sample_mode=mode,
                                      fused=fused, part_capacity=4 * capacity + 4096)
        rng = np.random.RandomState(5)
        if kind == "frames":
            _fill_frames(buf, rng, prefill)
        elif kind == "frames84":
            _fill_frames(buf, rng, prefill, hw=(84, 84))
        else:
            _fill_vectors(buf, rng, prefill)
        bufs.append((buf, rng))
    phi = Identity() if kind == "vectors" else ScaleU8()
    g = torch.Generator(device=dev)
    g.manual_seed(3)
    rounds = 7
    errs = [torch.rand(batch, device=dev, generator=g) * 1.7 for _ in range(rounds)]
    for r in range(rounds):
        outs = []
        for buf, rng in bufs:
            np.random.seed(100 + r)
            exps = buf.sample(batch)
            b = batch_experiences(exps, dev, phi, 0.97)
            outs.append((exps.index.clone(), {k: v.clone() for k, v in b.items()}))
            buf.update_errors(errs[r])
            if r % 3 == 1:  # appends between update and the next sample
                if kind.startswith("frames"):
                    _fill_frames(buf, rng, 37, hw=(84, 84) if kind == "frames84" else (12, 12))
                else:
                    _fill_vectors(buf, rng, 37)
        (ia, ba), (ib, bb) = outs
        assert torch.equal(ia, ib), "round %d indices" % r
        assert set(ba) == set(bb)
        for k in ba:
            assert ba[k].dtype == bb[k].dtype and ba[k].shape == bb[k].shape, k
            assert torch.equal(ba[k], bb[k]), "round %d %s" % (r, k)
    fa, fb = bufs[0][0], bufs[1][0]
    fa._flush()
    fb._flush()
    ia, ib = fa.store.info(), fb.store.info()
    for k in ("total", "min", "max_priority", "napp", "npop"):
        assert ia[k] == ib[k], k
    assert np.array_equal(fa.store.read_priorities(), fb.store.read_priorities())


@pytest.mark.parametrize("cap,levels_note", [(100, "smem tree"), (70000, "deep tree")])
def test_fused_step_draws_match_oracle(cap, levels_note):
    """b2rl_replay_step at the store level against the C oracle: indices, priorities,
    probabilities bit-identical, weights 2e-6, for every normalisation."""
    from oracle.replay import OraclePrioritizedBuffer
    from pfrl_b200 import _lib
    from pfrl_b200.store import DeviceReplayStore

    store = DeviceReplayStore(cap, part_bytes=16, part_capacity=64, max_batch=1024)
    ora = OraclePrioritizedBuffer(cap)
    rng = np.random.RandomState(11)
    n0 = min(cap, 5000)
    pr = rng.rand(n0) * 3 + 1e-3
    z = np.zeros((n0, 1), dtype=np.int32)
    store.append(z, z, np.zeros(n0, dtype=np.int64), np.zeros((n0, 1)), np.ones(n0, np.uint8),
                 np.zeros(n0, np.uint8), priority=pr)
    for p in pr:
        ora.append(None, float(p))
    for r in range(9):
        n = int(rng.randint(1, min(len(ora), 300) + 1))
        norm = r % 3
        beta = 0.4 + 0.05 * r
        u = rng.random_sample(n)
        oi, op, tot, mn = ora.sample_indices(n, u)
        res = store.step(u, [1.0, 0.9], beta, norm, mode=_lib.SAMPLE_EXACT, want_obs=False,
                         want_priority=True, want_prob=True)
        assert np.array_equal(res["index"].cpu().numpy(), oi), (r, n)
        assert res["priority"].cpu().numpy().tobytes() == op.tobytes()
        prob = op / tot
        assert res["prob"].cpu().numpy().tobytes() == prob.tobytes()
        if norm == _lib.NORM_NONE:
            w = (len(ora) * prob) ** -beta
        elif norm == _lib.NORM_BATCH:
            w = (prob / prob.min()) ** -beta
        else:
            w = (prob / (mn / tot)) ** -beta
        np.testing.assert_allclose(res["weights"].cpu().numpy(), w, rtol=2e-6)
        newp = rng.rand(n) * 2 + 1e-6
        ora.set_last_priority(newp)
        store.update_priorities(newp)
    info = store.info()
    assert info["total"] == ora.total() and info["min"] == ora.min()
    assert info["max_priority"] == ora.max_priority
    store.close()
