"""GPU: the v6 exact sampler's slow path is bit-identical to the reference too.

v6 decides most draws on approximate tables and sends the rest (about 1 %) down
the slow path, which re-runs the reference's arithmetic on the exact tree.  Two
test hooks make the slow path carry the load: B2RL_V6_SLOW_EVERY=3 forces every
third draw through it, B2RL_V6_EPS_SCALE=1e10 widens the decision margin until no
draw passes the fast test.  The library reads them once per process, so the
v6-tree bit-identity cases run in a child pytest with the variable set, with
exactly the assertions of the parent suite."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# trees with leaves at heap levels 18 and 20 (v6), stand-alone and fused launches
V6_CASES = [
    "tests/test_per_gpu.py::test_exact_sampler_deep_trees_bit_identical[70000-3000-2000]",
    "tests/test_per_gpu.py::test_exact_sampler_deep_trees_bit_identical[300000-1500-9000]",
    "tests/test_fused_step_gpu.py::test_fused_step_draws_match_oracle[70000-deep tree]",
    # adversarial trees at levels 17..21 (v6 D = 5..9, n = 60000 included), stand-alone and fused
    "tests/test_replay_trees_gpu.py::test_samplers_at_level[17]",
    "tests/test_replay_trees_gpu.py::test_samplers_at_level[18]",
    "tests/test_replay_trees_gpu.py::test_samplers_at_level[19]",
    "tests/test_replay_trees_gpu.py::test_samplers_at_level[20]",
    "tests/test_replay_trees_gpu.py::test_samplers_at_level[21]",
    "tests/test_replay_trees_gpu.py::test_npop_at_the_half_boundary[40000-loguniform]",
    "tests/test_replay_trees_gpu.py::test_npop_at_the_half_boundary[40000-subnormal]",
]


@pytest.mark.parametrize("var,value", [("B2RL_V6_SLOW_EVERY", "3"), ("B2RL_V6_EPS_SCALE", "1e10")])
def test_v6_bit_identity_through_the_slow_path(var, value):
    env = dict(os.environ)
    env[var] = value
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else [])
    cmd += ["-m", "pytest", "-q", "-p", "no:cacheprovider"] + V6_CASES
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, "%s=%s:\n%s\n%s" % (var, value, r.stdout[-4000:], r.stderr[-2000:])
    assert "10 passed" in r.stdout, r.stdout[-2000:]
