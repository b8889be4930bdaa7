"""Seeded single-process runs of the reference's ACER on its ABC toy environment ->
tests/golden/agent_trace_acer_<kind>.npz.

Each run goes through ``experiments.train_agent`` after moving the agent's
``shared_attributes`` to shared memory the way the reference's train_agent_async does
(its ACER asserts shared memory on every update).  Recorded: the initial parameters of
the shared model, the action and the statistics after every step, and the final
parameters of the shared and average models.

The kinds cover the discrete and the Gaussian heads, feed-forward and LSTM
(``RecurrentSequential``) models, the trust region on and off, truncation 10 and None,
``disable_online_update``, ``n_times_replay`` 0 and 2, continuing episodes cut by
``max_episode_len`` (a reset without a terminal, so the replay and online updates
bootstrap) and a replay_start_size small enough that replay starts early.  The runs are
short, so that fp32 rounding on CUDA cannot flip a sampled discrete action.

    python oracle/gen_golden_acer.py tests/golden
"""
import importlib
import os
import random
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

# kind -> (discrete, lstm, episodic, constructor overrides)
KINDS = {
    "discrete_ff": (True, False, False, dict(max_grad_norm=40)),
    "discrete_ff_plain": (True, False, True, dict(use_trust_region=False,
                                                  truncation_threshold=None)),
    "discrete_ff_replay_only": (True, False, False, dict(disable_online_update=True)),
    "discrete_ff_online_only": (True, False, True, dict(n_times_replay=0)),
    "discrete_lstm": (True, True, False, dict(t_max=5)),
    "gauss_ff": (False, False, False, dict()),
}
ACER_KINDS = tuple(KINDS)
STEPS = 200


def make_env(lib, kind, test=False):
    discrete, lstm, episodic, _ = KINDS[kind]
    ABC = importlib.import_module(lib.__name__ + ".envs.abc").ABC
    return ABC(size=2, discrete=discrete, episodic=episodic or test,
               partially_observable=lstm, deterministic=test)


def make_model(lib, kind, hidden=20):
    import torch  # noqa: F401
    from torch import nn

    discrete, lstm, _, _ = KINDS[kind]
    env = make_env(lib, kind)
    obs_size = env.observation_space.low.size
    acer = lib.agents.acer
    if discrete:
        n = env.action_space.n
        head = acer.ACERDiscreteActionHead(
            pi=nn.Sequential(nn.Linear(hidden, n), lib.policies.SoftmaxCategoricalHead()),
            q=nn.Sequential(nn.Linear(hidden, n), lib.q_functions.DiscreteActionValueHead()))
    else:
        a = env.action_space.low.size
        head = acer.ACERContinuousActionHead(
            pi=nn.Sequential(nn.Linear(hidden, a * 2),
                             lib.policies.GaussianHeadWithDiagonalCovariance()),
            v=nn.Sequential(nn.Linear(hidden, 1)),
            adv=nn.Sequential(lib.nn.ConcatObsAndAction(), nn.Linear(hidden + a, 1)))
    if lstm:
        return lib.nn.RecurrentSequential(
            nn.Linear(obs_size, hidden), nn.LeakyReLU(),
            nn.LSTM(num_layers=1, input_size=hidden, hidden_size=hidden), head)
    return nn.Sequential(nn.Linear(obs_size, hidden), nn.LeakyReLU(), head)


def make_acer_agent(lib, kind, device=None, rbuf=None, **extra):
    _, lstm, _, over = KINDS[kind]
    model = make_model(lib, kind)
    if device is not None:
        model.to(device)
    opt = lib.optimizers.SharedRMSpropEpsInsideSqrt(model.parameters(), lr=1e-3, eps=1e-8,
                                                    alpha=0.99)
    kw = dict(t_max=2, n_times_replay=2, replay_start_size=20, beta=1e-2)
    kw.update(over)
    kw.update(extra)
    if rbuf is None:
        rbuf = lib.replay_buffers.EpisodicReplayBuffer(10 ** 4)
    return lib.agents.acer.ACER(model, opt, gamma=0.5, replay_buffer=rbuf,
                                act_deterministically=True, recurrent=lstm, **kw)


def share_memory(agent):
    """train_agent_async.py's preparation of the shared attributes (CPU models)."""
    import torch

    for attr in agent.shared_attributes:
        value = getattr(agent, attr)
        if isinstance(value, torch.nn.Module):
            for v in value.state_dict().values():
                v.share_memory_()
        elif isinstance(value, torch.optim.Optimizer):
            for state in value.state_dict()["state"].values():
                for v in state.values():
                    if isinstance(v, torch.Tensor):
                        v.share_memory_()


class _Recorder:
    """The env seen by train_agent, recording every action; a step hook records the
    statistics after every step."""

    def __init__(self, env, check):
        self.env = env
        self.actions = []
        self.stats = []
        self.check = check

    def reset(self):
        return self.env.reset()

    def step(self, action):
        if self.check is not None:
            self.check(len(self.actions), action)
        self.actions.append(np.array(action, copy=True))
        return self.env.step(action)

    def hook(self, env, agent, step):
        self.stats.append([v for _, v in agent.get_statistics()])

    def __getattr__(self, name):
        return getattr(self.env, name)


def run(lib, kind, device=None, rbuf=None, check=None, init=None, steps=STEPS, setup=None,
        **extra):
    import torch

    torch.manual_seed(3)
    agent = make_acer_agent(lib, kind, device=device, rbuf=rbuf, **extra)
    if setup is not None:
        setup(agent)
    if init is not None:
        sd = {k[len("init_shared_model__"):]: torch.tensor(init[k]) for k in init.files
              if k.startswith("init_shared_model__")}
        for name in ("shared_model", "shared_average_model", "model"):
            getattr(agent, name).load_state_dict(sd)
    if agent.device.type == "cpu":
        share_memory(agent)
    g = {"init_shared_model__" + k: v.detach().cpu().numpy().copy()
         for k, v in agent.shared_model.state_dict().items()}
    np.random.seed(9)
    torch.manual_seed(9)
    random.seed(9)
    _, _, episodic, _ = KINDS[kind]
    env = _Recorder(make_env(lib, kind), check)
    with tempfile.TemporaryDirectory() as outdir:
        lib.experiments.train_agent(agent, env, steps, outdir,
                                    max_episode_len=None if episodic else 3,
                                    step_hooks=[env.hook])
    g.update(actions=np.array(env.actions), stats=np.array(env.stats, dtype=np.float64),
             stat_names=np.array([n for n, _ in agent.get_statistics()]))
    for name in ("shared_model", "shared_average_model"):
        for k, v in getattr(agent, name).state_dict().items():
            g["final_%s__%s" % (name, k)] = v.detach().cpu().numpy().copy()
    return agent, g


def main(out_dir):
    from oracle.refimport import import_reference

    pfrl = import_reference()
    for kind in ACER_KINDS:
        _, g = run(pfrl, kind)
        np.savez_compressed(os.path.join(out_dir, "agent_trace_acer_%s.npz" % kind), **g)
        print("wrote agent_trace_acer_%s.npz" % kind, dict(zip(g["stat_names"], g["stats"][-1])))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(HERE), "tests",
                                                             "golden"))
