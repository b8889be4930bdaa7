"""GPU: the v6 exact sampler's ascent warps, on trees that make same-subtree revisits common.

v6 applies draw k to the exact tree on ascent warp k % V6_NASC, so draws of different
level-12 subtrees are applied concurrently.  Two draws of one subtree must never be: the
later one is decided fast only if the earlier one was inside the fenced prefix (the minimum
over the warps) when its scout copied the subtree, else it waits in the slow path for every
earlier draw.  Trees at heap levels 18 and 21 (v6 D = 6 and 9) whose mass sits on 8, 64 or
512 level-12 subtrees, and one whose draws alternate between two subtrees, hand revisits of a
subtree to different warps.  Every launch, stand-alone and fused, is bit-identical to the
oracle in indices and priorities, and the whole heap equals the oracle's after it.

The fast path must decide a real share of the revisits (scout_hits counts the fast draws):
otherwise the cross-warp ordering would only be exercised through the slow path.  The same
cases run again in a child pytest with B2RL_V6_SLOW_EVERY=3 and with B2RL_V6_EPS_SCALE=1e10
(the test hooks of test_v6_slow_path_gpu.py), where that share is not asserted."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle.replay import OraclePrioritizedBuffer
from test_replay_trees_gpu import (append_both, assert_heap_consistent, capacity_for_level,
                                   exact_round, make_store, oracle_heap)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NS = (1, 2, 3, 5, 31, 512, 4097)
# (heap level, heavy level-12 subtrees; "alt": two subtrees, draws alternate between them)
TREES = [(18, 8), (18, 64), (18, 512), (21, 8), (21, 64), (21, 512), (21, "alt")]
HOOKS = ("B2RL_V6_SLOW_EVERY", "B2RL_V6_EPS_SCALE")


def concentrated_tree(L, heavy, rng):
    """A full ring (npop = 0, so leaf slot = index) whose mass sits on `heavy` live level-12
    subtrees: their leaves 0.5..1.5, every other leaf 1e-9."""
    cap = capacity_for_level(L)
    D = L - 12
    store = make_store(cap, max_batch=8192)
    ora = OraclePrioritizedBuffer(cap)
    live = cap >> D  # level-12 subtrees with live leaves
    subs = rng.choice(live, 2 if heavy == "alt" else heavy, replace=False)
    prios = np.full(cap, 1e-9)
    for s in subs:
        prios[s << D:(s + 1) << D] = rng.uniform(0.5, 1.5, 1 << D)
    append_both(store, ora, prios)
    assert store.nslots == 1 << L and store.npop == 0 and len(store) == cap
    return store, ora, subs


def alternating_uniforms(store, ora, subs, n, L):
    """u that lands in subs[0] on even draws and in subs[1] on odd draws while both hold
    mass: the level-12 prefix of each heavy subtree over the root, nudged inside it."""
    D = L - 12
    leaves = oracle_heap(ora, 0, store.nslots)[store.nslots:]
    root = leaves.sum()
    pre = [leaves[:s << D].sum() for s in subs]
    mass = [leaves[s << D:(s + 1) << D].sum() for s in subs]
    k = np.arange(n)
    side = k % 2
    frac = 0.1 + 0.8 * ((k // 2) % 7) / 7.0
    u = (np.take(pre, side) + frac * np.take(mass, side) * 0.5) / root
    return np.clip(u, 0.0, 1.0 - 2.0 ** -53)


def revisits(idx, D):
    """Draws whose level-12 subtree an earlier draw of the same launch chose."""
    seen, r = set(), 0
    for s in (np.asarray(idx) >> D).tolist():
        r += s in seen
        seen.add(s)
    return r


@pytest.mark.parametrize("L,heavy", TREES, ids=["%d-%s" % t for t in TREES])
def test_ascent_warps_bit_identical(L, heavy):
    rng = np.random.RandomState(L * 1000 + (7 if heavy == "alt" else heavy))
    store, ora, subs = concentrated_tree(L, heavy, rng)
    D = L - 12
    drawn = {}  # the indices of the last launch, as the oracle drew them inside exact_round
    oracle_sample = ora.sample_indices

    def recording(n, u=None):
        out = oracle_sample(n, u)
        drawn["idx"] = out[0]
        return out

    ora.sample_indices = recording
    fast = non_revisit = rev = 0
    for fused in (False, True):
        for n in NS:
            if heavy == "alt":
                u = alternating_uniforms(store, ora, subs, n, L)
            else:
                u = rng.random_sample(n)
            drawn.clear()
            exact_round(store, ora, u, fused, "equal", rng)
            idx = drawn["idx"]
            hits = store.info()["scout_hits"]
            r = revisits(idx, D)
            fast += hits & 0xffff
            rev += r
            non_revisit += len(idx) - r
            assert (hits & 0xffff) + (hits >> 16) == len(idx)
    assert_heap_consistent(store, ora)
    store.close()
    if heavy in (64, 512) and not any(os.environ.get(h) for h in HOOKS):
        # at least this many revisits were decided on the fast path
        fast_revisits = fast - non_revisit
        assert fast_revisits >= 0.25 * rev, (fast, non_revisit, rev)


@pytest.mark.parametrize("var,value", [("B2RL_V6_SLOW_EVERY", "3"), ("B2RL_V6_EPS_SCALE", "1e10")])
def test_ascent_warps_through_the_slow_path(var, value):
    env = dict(os.environ)
    env[var] = value
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else [])
    cmd += ["-m", "pytest", "-q", "-p", "no:cacheprovider",
            "tests/test_v6_ascent_gpu.py::test_ascent_warps_bit_identical"]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, "%s=%s:\n%s\n%s" % (var, value, r.stdout[-4000:], r.stderr[-2000:])
    assert "%d passed" % len(TREES) in r.stdout, r.stdout[-2000:]
