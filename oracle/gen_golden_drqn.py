"""Golden traces for recurrent DQN / DoubleDQN (DRQN), produced by the REAL reference on
CPU (TEST INFRASTRUCTURE ONLY).

    python -m oracle.gen_golden_drqn

writes tests/golden/agent_trace_drqn_<kind>.npz for every kind of DRQN_KINDS: seeded
runs of ``DQN`` / ``DoubleDQN(recurrent=True)`` over the reference's
``EpisodicReplayBuffer`` with the reference test's ``RecurrentSequential(Linear, ELU, RNN,
Linear, DiscreteActionValueHead)`` model or its LSTM variant, on two partially observable
ABC envs driven through ``batch_act`` / ``batch_observe``.  Env 0 is a continuing task cut
every 8 steps (interrupted episodes of 8 transitions, so ``episodic_update_len=3`` draws a
start), env 1 an episodic one (short terminal episodes); the 60-transition capacity evicts
whole episodes.  Each file holds the initial and final parameters, the actions of every
step, the statistics after every vector step, and the episodes every update sampled (their
commit number) with the start of each window.

The construction (``make_drqn_agent``) and the driver (``run_drqn_trace``,
``record_episode_samples``) are shared with tests/test_drqn_traces_*.py, which replay the
runs with this package's agents and buffers.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

OUT = os.path.join(ROOT, "tests", "golden")

# kind -> (agent class, recurrent layer, episodic_update_len)
DRQN_KINDS = {
    "dqn_rnn": ("DQN", "rnn", None),
    "dqn_lstm": ("DQN", "lstm", 3),
    "ddqn_rnn": ("DoubleDQN", "rnn", 3),
    "ddqn_lstm": ("DoubleDQN", "lstm", None),
}
STEPS = 150
CAPACITY = 60
MINIBATCH = 4
N_OBS, N_ACT, HIDDEN = 5, 3, 10


def make_drqn_agent(lib, kind, rbuf, gpu=None, phi=None):
    """The same agent for the reference (lib = pfrl) and the rebuild (lib = pfrl_b200).
    The parameters are seeded by the caller (torch.manual_seed before the call)."""
    import torch
    from torch import nn

    cls_name, cell, ep_len = DRQN_KINDS[kind]
    rnn = nn.RNN(HIDDEN, HIDDEN) if cell == "rnn" else nn.LSTM(HIDDEN, HIDDEN)
    q = lib.nn.RecurrentSequential(nn.Linear(N_OBS, HIDDEN), nn.ELU(), rnn,
                                   nn.Linear(HIDDEN, N_ACT),
                                   lib.q_functions.DiscreteActionValueHead())
    opt = torch.optim.Adam(q.parameters(), 1e-2, eps=1e-2)
    explorer = lib.explorers.LinearDecayEpsilonGreedy(1.0, 0.1, 200,
                                                      lambda: np.random.randint(N_ACT))
    if phi is None:
        phi = lambda x: x.astype(np.float32, copy=False)  # noqa: E731
    agent = getattr(lib.agents, cls_name)(
        q, opt, rbuf, gamma=0.9, explorer=explorer, gpu=gpu, replay_start_size=30,
        minibatch_size=MINIBATCH, update_interval=1, target_update_interval=20, phi=phi,
        recurrent=True, episodic_update_len=ep_len)
    return q, agent


def run_drqn_trace(agent, steps=STEPS, check=None):
    """Drive two ABC(partially_observable=True) envs; returns the actions [steps, 2] and
    the statistics after every vector step [steps, 4] (average_q, average_loss, n_updates,
    rlen)."""
    from pfrl_b200.envs.abc import ABC

    envs = [ABC(size=3, partially_observable=True, episodic=False, deterministic=True),
            ABC(size=3, partially_observable=True, episodic=True, deterministic=True)]
    obs = [e.reset() for e in envs]
    age = [0, 0]
    actions, stats = [], []
    for t in range(steps):
        a = [int(x) for x in agent.batch_act(obs)]
        if check is not None:
            check(t, a)
        actions.append(a)
        nobs, r, d, _ = zip(*[e.step(x) for e, x in zip(envs, a)])
        age = [n + 1 for n in age]
        resets = [age[0] == 8, False]
        agent.batch_observe(list(nobs), list(r), list(d), resets)
        obs = list(nobs)
        for i in range(2):
            if d[i] or resets[i]:
                obs[i] = envs[i].reset()
                age[i] = 0
        st = dict(agent.get_statistics())
        stats.append([st["average_q"], st["average_loss"], st["n_updates"], st["rlen"]])
    return np.asarray(actions), np.asarray(stats, dtype=np.float64)


def record_episode_samples(rbuf, log):
    """Wrap a list-of-dicts episodic buffer (the reference's EpisodicReplayBuffer or
    pfrl_b200's HostEpisodicReplayBuffer) so that every sample_episodes call appends
    (episode commit numbers, window starts) to ``log``."""
    committed = [0]
    raw_stop = rbuf.stop_current_episode
    raw_sample = rbuf.sample_episodes

    def stop(env_id=0):
        if rbuf.current_episode[env_id]:
            committed[0] += 1
        raw_stop(env_id=env_id)

    def sample_episodes(n_episodes, max_len=None):
        episodes = raw_sample(n_episodes, max_len)
        memory = list(rbuf.episodic_memory)
        popped = committed[0] - len(memory)
        ids, starts = [], []
        for seq in episodes:
            for i, ep in enumerate(memory):
                hit = [j for j, tr in enumerate(ep) if tr is seq[0]]
                if hit:
                    ids.append(popped + i)
                    starts.append(hit[0])
                    break
        assert len(ids) == len(episodes)
        log.append((ids, starts))
        return episodes

    rbuf.stop_current_episode = stop
    rbuf.sample_episodes = sample_episodes


def drqn_traces(out_dir):
    import torch

    from oracle.refimport import import_reference

    pfrl = import_reference()
    for kind in DRQN_KINDS:
        rbuf = pfrl.replay_buffers.EpisodicReplayBuffer(CAPACITY)
        log = []
        record_episode_samples(rbuf, log)
        torch.manual_seed(3)
        q, agent = make_drqn_agent(pfrl, kind, rbuf)
        g = {"init_" + k: v.numpy().copy() for k, v in q.state_dict().items()}
        np.random.seed(9)
        torch.manual_seed(9)
        actions, stats = run_drqn_trace(agent)
        assert log, "the run made no update"
        g.update(actions=actions, stats=stats,
                 sample_ids=np.asarray([ids for ids, _ in log], dtype=np.int64),
                 sample_starts=np.asarray([s for _, s in log], dtype=np.int64))
        g.update({"final_" + k: v.detach().numpy().copy() for k, v in q.state_dict().items()})
        path = os.path.join(out_dir, "agent_trace_drqn_%s.npz" % kind)
        np.savez(path, **g)
        print("wrote %s: %d updates, final rlen %d" % (
            path, len(log), int(stats[-1, 3])))


if __name__ == "__main__":
    drqn_traces(OUT)
