"""Recurrent PPO replays the seeded runs of the REAL reference on CPU
(tests/golden/agent_trace_ppo_recurrent_*.npz, written by oracle/gen_golden_recurrent_ppo.py):
the actions of every step (equal for discrete, allclose for Gaussian), every minibatch's
schedule (episode, offset, length of each sequence, in order), the statistics after every
step and the final parameters."""
import os
import random

import numpy as np
import pytest
import torch

import pfrl_b200
from oracle.gen_golden_recurrent_ppo import (
    RPPO_KINDS, make_rppo_agent, record_schedule, run_rppo_trace,
)
from pfrl_b200.agents import ppo

GOLD = os.path.join(os.path.dirname(__file__), "golden")
RTOL, ATOL = 1e-5, 1e-6  # test_agent_traces_cpu.py's PPO bounds


def replay(kind, gpu=None, rtol=RTOL, atol=ATOL, use_fused=True):
    """Run this package's agent on the reference's trace; returns (golden, model, stats,
    schedule rows)."""
    g = np.load(os.path.join(GOLD, "agent_trace_ppo_recurrent_%s.npz" % kind))
    torch.manual_seed(3)
    model, agent = make_rppo_agent(pfrl_b200, kind, gpu=gpu)
    agent.use_fused = use_fused
    model.load_state_dict({k: torch.tensor(g["init_" + k]) for k in model.state_dict()})
    assert [n for n, _ in agent.get_statistics()] == g["stat_names"].tolist()
    log = []
    raw_yield = record_schedule(ppo, agent, log, spans=True)
    discrete = g["actions"].dtype.kind in "iu"

    def check(t, a):
        want = g["actions"][t]
        if discrete:
            assert a.tolist() == want.tolist(), "actions diverge at step %d" % t
        else:
            np.testing.assert_allclose(a, want, rtol=rtol, atol=atol,
                                       err_msg="actions diverge at step %d" % t)

    np.random.seed(9)
    torch.manual_seed(9)
    random.seed(9)
    try:
        _, stats = run_rppo_trace(agent, kind, steps=g["actions"].shape[0], check=check)
    finally:
        ppo._yield_subset_of_sequences_with_fixed_number_of_items = raw_yield
    return g, model, stats, np.asarray(log, dtype=np.int64).reshape(-1, 4)


def check_run(g, model, stats, schedule, rtol, atol):
    assert np.array_equal(schedule, g["schedule"]), "minibatch schedules differ"
    want = g["stats"]
    both_nan = np.isnan(stats) & np.isnan(want)
    np.testing.assert_allclose(np.where(both_nan, 0.0, stats), np.where(both_nan, 0.0, want),
                               rtol=rtol, atol=atol)
    for k, v in model.state_dict().items():
        np.testing.assert_allclose(v.detach().cpu().numpy(), g["final_" + k], rtol=rtol,
                                   atol=atol, err_msg=k)


def test_fixtures_cover_split_tails_and_dropped_remainders():
    g = np.load(os.path.join(GOLD, "agent_trace_ppo_recurrent_gru.npz"))
    s = g["schedule"]
    # max_recurrent_sequence_len = 3 cuts episodes at offsets 0, 3, 6 ...; a split tail
    # starts elsewhere
    assert np.any(s[:, 2] % 3 != 0)
    # 20 transitions per update and minibatches of 7: 2 minibatches per epoch, 6 dropped
    per_mb = np.bincount(s[:, 0], weights=s[:, 3])
    assert np.all(per_mb == 7)
    # whole episodes (no length limit): sequences longer than one step, several per minibatch
    lstm = np.load(os.path.join(GOLD, "agent_trace_ppo_recurrent_lstm.npz"))
    assert lstm["schedule"][:, 3].max() > 1
    assert np.bincount(lstm["schedule"][:, 0]).max() > 1


@pytest.mark.parametrize("kind", list(RPPO_KINDS))
def test_recurrent_ppo_reproduces_the_reference_run_on_cpu(kind):
    g, model, stats, schedule = replay(kind)
    check_run(g, model, stats, schedule, RTOL, ATOL)
