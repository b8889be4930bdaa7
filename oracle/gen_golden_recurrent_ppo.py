"""Golden traces for recurrent PPO, produced by the REAL reference on CPU (TEST
INFRASTRUCTURE ONLY).

    python -m oracle.gen_golden_recurrent_ppo

writes tests/golden/agent_trace_ppo_recurrent_<kind>.npz for every kind of RPPO_KINDS:
seeded runs of ``PPO(recurrent=True)`` on partially observable ABC envs.

- ``lstm``: the reference test's ``RecurrentBranched(LSTM pi, LSTM v)`` model (4 state
  leaves), ``max_recurrent_sequence_len=None``, standardised advantages,
  ``clip_eps_vf=0.2``; 3 envs driven through ``batch_act`` / ``batch_observe``: env 0
  episodic, env 1 a continuing task reset every 5 steps, env 2 episodic with resets
  every 7 steps (terminal episodes and resets mixed).
- ``gru``: continuous Gaussian head on a GRU trunk, ``max_recurrent_sequence_len=3``, an
  ``EmpiricalNormalization`` observation normaliser, lambda 0.5, and ``minibatch_size=7``
  over 2 envs, so minibatches end in split tails and each epoch drops a remainder.
- ``single``: the ``lstm`` model on one env driven through ``act`` / ``observe``.

Each file holds the initial and final parameters, the actions of every step, the
statistics after every step, and every minibatch's schedule: rows (minibatch number,
episode, offset, length) where the episode is its index in the update's memory order
and the offset is where the sequence starts in it, in the order the minibatch lists them.

The construction (``make_rppo_agent``), the driver (``run_rppo_trace``) and the schedule
recorder (``record_schedule``) are shared with tests/test_recurrent_ppo_traces_*.py.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

OUT = os.path.join(ROOT, "tests", "golden")

# kind -> number of envs, steps
RPPO_KINDS = {"lstm": (3, 90), "gru": (2, 90), "single": (1, 120)}
SIZE, HIDDEN = 3, 8


def make_rppo_agent(lib, kind, gpu=None):
    """The same agent for the reference (lib = pfrl) and the rebuild (lib = pfrl_b200).
    The parameters are seeded by the caller (torch.manual_seed before the call)."""
    import torch
    from torch import nn

    n_obs = SIZE + 2
    if kind in ("lstm", "single"):
        pi = lib.nn.RecurrentSequential(nn.LSTM(num_layers=1, input_size=n_obs, hidden_size=HIDDEN),
                                        nn.Linear(HIDDEN, SIZE),
                                        lib.policies.SoftmaxCategoricalHead())
        v = lib.nn.RecurrentSequential(nn.LSTM(num_layers=1, input_size=n_obs, hidden_size=HIDDEN),
                                       nn.Linear(HIDDEN, 1))
        model = lib.nn.RecurrentBranched(pi, v)
        kw = dict(update_interval=24 if kind == "lstm" else 20, minibatch_size=8, epochs=3,
                  lambd=0.95, clip_eps_vf=0.2, max_recurrent_sequence_len=None,
                  obs_normalizer=None)
    else:
        model = lib.nn.RecurrentSequential(
            nn.GRU(num_layers=1, input_size=n_obs, hidden_size=HIDDEN),
            lib.nn.Branched(
                nn.Sequential(nn.Linear(HIDDEN, SIZE),
                              lib.policies.GaussianHeadWithStateIndependentCovariance(
                                  action_size=SIZE, var_type="diagonal",
                                  var_func=lambda x: torch.exp(2 * x), var_param_init=0)),
                nn.Linear(HIDDEN, 1)))
        kw = dict(update_interval=20, minibatch_size=7, epochs=2, lambd=0.5, clip_eps_vf=None,
                  max_recurrent_sequence_len=3,
                  obs_normalizer=lib.nn.EmpiricalNormalization(n_obs, clip_threshold=5))
    opt = torch.optim.Adam(model.parameters(), lr=1e-2, eps=1e-5)
    agent = lib.agents.PPO(model, opt, gpu=gpu, gamma=0.9, standardize_advantages=True,
                           recurrent=True, max_grad_norm=1.0, **kw)
    return model, agent


def run_rppo_trace(agent, kind, steps=None, check=None):
    """Drive the kind's envs; returns the actions [steps, n_envs, ...] and the statistics
    after every step [steps, 6]."""
    from pfrl_b200.envs.abc import ABC

    n_envs, default_steps = RPPO_KINDS[kind]
    steps = default_steps if steps is None else steps
    discrete = kind != "gru"
    envs = [ABC(size=SIZE, discrete=discrete, partially_observable=True, deterministic=True,
                episodic=(i != 1)) for i in range(n_envs)]
    cut = {0: None, 1: 5, 2: 7}
    obs = [e.reset() for e in envs]
    age = [0] * n_envs
    actions, stats = [], []
    for t in range(steps):
        if kind == "single":
            a = np.asarray([agent.act(obs[0])])
        else:
            a = np.asarray(agent.batch_act(obs))
        if check is not None:
            check(t, a)
        actions.append(a)
        nobs, r, d, _ = zip(*[e.step(x) for e, x in zip(envs, a)])
        age = [n + 1 for n in age]
        resets = [cut[i] is not None and age[i] >= cut[i] and not d[i] for i in range(n_envs)]
        if kind == "single":
            agent.observe(nobs[0], r[0], d[0], resets[0])
        else:
            agent.batch_observe(list(nobs), list(r), list(d), resets)
        obs = list(nobs)
        for i in range(n_envs):
            if d[i] or resets[i]:
                obs[i] = envs[i].reset()
                age[i] = 0
        stats.append([float(v) for _, v in agent.get_statistics()])
    return np.asarray(actions), np.asarray(stats, dtype=np.float64)


def record_schedule(ppo_module, agent, log, spans=False):
    """Every minibatch the recurrent update serves, as rows (minibatch, episode, offset,
    length) appended to ``log``.  For the reference (``spans=False``) sequences are lists
    of transition dicts and the episodes are ``agent.memory`` when ``_update_recurrent``
    starts; for this package they are spans over the rollout and the episodes are
    ``agent._episode_spans`` when ``_update_recurrent_from_rollout`` starts."""
    where = {}
    raw_yield = ppo_module._yield_subset_of_sequences_with_fixed_number_of_items

    def key(seq):
        return (seq.env, seq.t0) if spans else id(seq[0])

    def yield_subsets(sequences, n_items):
        for sub in raw_yield(sequences, n_items):
            mb = len({r[0] for r in log})
            for seq in sub:
                ep, off = where[key(seq)]
                log.append((mb, ep, off, len(seq)))
            yield sub

    ppo_module._yield_subset_of_sequences_with_fixed_number_of_items = yield_subsets
    if spans:
        raw = agent._update_recurrent_from_rollout

        def update():
            T, E = len(agent._rewards), agent._rstates[0].shape[0]
            where.clear()
            for i, sp in enumerate(agent._episode_spans(T, E)):
                for j in range(len(sp)):
                    where[(sp.env, sp.t0 + j)] = (i, j)
            raw()

        agent._update_recurrent_from_rollout = update
    else:
        raw = agent._update_recurrent

        def update(dataset):
            where.clear()
            for i, ep in enumerate(agent.memory):
                for j, tr in enumerate(ep):
                    where[id(tr)] = (i, j)
            raw(dataset)

        agent._update_recurrent = update
    return raw_yield


def rppo_traces(out_dir):
    import random

    import torch

    from oracle.refimport import import_reference

    pfrl = import_reference()
    from pfrl.agents import ppo as ref_ppo

    for kind in RPPO_KINDS:
        torch.manual_seed(3)
        model, agent = make_rppo_agent(pfrl, kind)
        g = {"init_" + k: v.numpy().copy() for k, v in model.state_dict().items()}
        log = []
        raw_yield = record_schedule(ref_ppo, agent, log)
        np.random.seed(9)
        torch.manual_seed(9)
        random.seed(9)
        try:
            actions, stats = run_rppo_trace(agent, kind)
        finally:
            ref_ppo._yield_subset_of_sequences_with_fixed_number_of_items = raw_yield
        assert log, "the run made no update"
        g.update(actions=actions, stats=stats, schedule=np.asarray(log, dtype=np.int64),
                 stat_names=np.asarray([n for n, _ in agent.get_statistics()]))
        g.update({"final_" + k: v.detach().numpy().copy() for k, v in model.state_dict().items()})
        path = os.path.join(out_dir, "agent_trace_ppo_recurrent_%s.npz" % kind)
        np.savez(path, **g)
        print("wrote %s: %d minibatches, %d schedule rows, n_updates %d" % (
            path, len({r[0] for r in log}), len(log), int(stats[-1, 4])))


if __name__ == "__main__":
    rppo_traces(OUT)
