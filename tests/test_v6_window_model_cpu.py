"""The exact sampler's leaf-window rule (csrc/tree_dev.cuh, exact_deep_v6) on the CPU model
of its decisions (tools/v6_model.py): every draw the rule accepts picks the leaf the
reference's sequential arithmetic picks, on adversarial trees (ties, 1e-30..1e+30, u on
node and leaf boundaries, mispredicted nodes and windows), and the window's bounds stay
inside the error budget the margin EPS = (n + 64) 2^-46 root is derived from."""
import importlib.util
import os
from fractions import Fraction

import numpy as np
import pytest

_PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "v6_model.py")
_spec = importlib.util.spec_from_file_location("v6_model", _PATH)
v6 = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(v6)

FAMILIES = [name for name, _ in v6.families(np.random.RandomState(0))]


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("T", [4, 7, 8])  # 9, 6 and 5 levels staged per draw
@pytest.mark.parametrize("eps_rel", [None, 2.0 ** -20])
def test_accepted_decisions_equal_the_exact_chain(family, T, eps_rel):
    rng = np.random.RandomState(FAMILIES.index(family) * 100 + T)
    leaves = dict(v6.families(rng))[family]
    us = v6.draws(rng, leaves)
    # run() asserts every accepted leaf against the exact chain, and the final trees
    out, fallbacks = v6.run(leaves, us, T, eps_rel, older=2 + (T & 1), mispredict=0.1, rng=rng)
    assert len(out) == len(us)
    if eps_rel is None:
        # not vacuous: most draws are decided by the window
        assert fallbacks < len(us) // 2


@pytest.mark.parametrize("T", [4, 7, 8])
def test_well_predicted_draws_rarely_fall_back(T):
    rng = np.random.RandomState(T)
    leaves = rng.rand(1 << 12) + 0.01
    us = rng.random_sample(256)
    _, fallbacks = v6.run(leaves, us, T, None, older=2 + (T & 1))
    assert fallbacks <= 0.02 * len(us)


@pytest.mark.parametrize("family", FAMILIES)
def test_window_bounds_within_the_error_budget(family):
    """each bound is within (D + 32) 2^-53 R of the exact sum of the leaves before it in
    the subtree, for windows at the subtree's edges and inside it"""
    rng = np.random.RandomState(7)
    leaves = dict(v6.families(rng))[family]
    E = v6.build(leaves)
    R = E[1]
    for D in (5, 6, 9):
        nleaf = 1 << D
        top = len(leaves) >> D  # heap indices of the nodes D levels above the leaves
        for node in rng.randint(top, 2 * top, 6).tolist():
            for x in (0.0, E[node] * 0.37, E[node]):
                lo, end, f = v6.leaf_window(E, node, D, x)
                assert 0 <= f <= nleaf - v6.WIN
                first = node << D
                exact = sum((Fraction(v) for v in E[first:first + f]), Fraction(0))
                bounds = list(lo) + [end]
                for c, b in enumerate(bounds):
                    if c:
                        exact += Fraction(E[first + f + c - 1])
                    assert abs(Fraction(b) - exact) <= (D + 32) * Fraction(R) / 2 ** 53
