"""The exact sampler's main warp reads a draw's table entries before the previous draw's
update is stored and applies that one update in registers (csrc/tree_dev.cuh,
exact_deep_v6).  On the CPU model of its decisions (tools/v6_model.py, prefetch=True),
every accepted decision equals the reference's sequential arithmetic when consecutive draws
fall on the same level-12 node, on nodes before and after it in the same block and in other
blocks, and when u * root lies on table boundaries.  The window of each draw is laid down
from a staged tree that still lacks the previous draw, so a draw at the previous draw's node
is only right because the conflict rule sends it down the exact path."""
import importlib.util
import os

import numpy as np
import pytest

_PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "v6_model.py")
_spec = importlib.util.spec_from_file_location("v6_model", _PATH)
v6 = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(v6)

FAMILIES = [name for name, _ in v6.families(np.random.RandomState(0))]
T_LEVELS = [4, 7, 8]  # 9, 6 and 5 levels staged per draw


def run(leaves, us, T, **kw):
    """run() asserts every accepted leaf against the exact chain, and the final trees"""
    stats = {}
    out, fallbacks = v6.run(leaves, us, T, None, older=2 + (T & 1), prefetch=True, stats=stats, **kw)
    assert len(out) == len(us)
    return out, fallbacks, stats


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("T", T_LEVELS)
def test_corrected_decisions_equal_the_exact_chain(family, T):
    rng = np.random.RandomState(FAMILIES.index(family) * 100 + T + 1)
    leaves = dict(v6.families(rng))[family]
    us = v6.draws(rng, leaves)
    _, _, st = run(leaves, us, T, mispredict=0.1, rng=rng)
    # not vacuous: decisions on entries that miss the previous draw's update were accepted
    assert st["accepted_before"] > 0 and st["accepted_after"] > 0


@pytest.mark.parametrize("T", T_LEVELS)
def test_consecutive_draws_at_one_node(T):
    """runs of three and more draws at the same level-12 node: the entries and the staged
    window of the second miss the first draw, and only the conflict rule keeps its leaf right"""
    rng = np.random.RandomState(T)
    leaves = rng.rand(1 << 12) + 0.01
    ntop = 1 << (T - 1)
    us = []
    for _ in range(24):
        x = rng.rand()
        us += [x, x + 0.1 / ntop, x - 0.1 / ntop]
    _, _, st = run(leaves, np.clip(us, 0.0, np.nextafter(1.0, 0.0)), T)
    assert st["same"] >= 24


@pytest.mark.parametrize("T", T_LEVELS)
@pytest.mark.parametrize("where", ["same block", "other blocks"])
def test_consecutive_draws_on_both_sides(T, where):
    """alternating draws at nodes before and after the previous draw's node, next to it
    inside one block of the prefix table or in blocks far apart"""
    rng = np.random.RandomState(10 * T + len(where))
    leaves = rng.rand(1 << 12) + 0.01
    ntop = 1 << (T - 1)
    step = 1.0 / ntop if where == "same block" else 0.5
    us = []
    for _ in range(48):
        x = rng.rand() * (1.0 - step) if where == "same block" else rng.rand() * 0.5
        us += [x + step, x]
    _, _, st = run(leaves, np.clip(us, 0.0, np.nextafter(1.0, 0.0)), T)
    assert st["accepted_before"] >= 10 and st["accepted_after"] >= 10


@pytest.mark.parametrize("T", T_LEVELS)
def test_u_on_table_boundaries(T):
    """equal leaves: u * root on node and block boundaries of the prefix tables, each after
    a draw at another node whose update the entries miss"""
    rng = np.random.RandomState(T + 50)
    leaves = np.ones(1 << 12)
    ntop = 1 << (T - 1)
    us = []
    for m in rng.randint(1, ntop, 40).tolist():
        us += [rng.rand(), m / ntop]
    _, _, st = run(leaves, np.array(us), T)
    assert st["before"] + st["after"] > 0
