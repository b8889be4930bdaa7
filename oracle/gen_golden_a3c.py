"""Seeded single-process runs of the reference's A3C on its ABC toy environment ->
tests/golden/agent_trace_a3c_<kind>.npz.

The models are the reference test's (tests/agents_tests/test_a3c.py): ``Branched`` (or
``RecurrentBranched`` of LSTMs) of a 20-unit policy with a softmax or a state-independent
diagonal Gaussian head and a value branch, output layers scaled by 0.1.  The optimizer is
``SharedRMSpropEpsInsideSqrt``, gamma 0.8 and beta 1e-2 as there.  Each run goes through
``experiments.train_agent`` after moving the shared attributes to shared memory as the
reference's train_agent_async does (A3C asserts shared memory on every update).

The kinds cover the discrete and Gaussian heads, feed-forward and LSTM models, t_max 1 and
5, an episodic env and a continuing one cut by ``max_episode_len`` = 2 (a reset without a
terminal, so the update bootstraps), and one run each with ``keep_loss_scale_same``,
``normalize_grad_by_t_max`` and ``max_grad_norm``.  Recorded: the initial parameters, the
action of every step, the statistics after every step, the number of updates and the shared
model's parameters after every update (after every fifth or tenth for the LSTM models, whose
parameters would otherwise make the fixtures large).  The runs are short, so that fp32
rounding on CUDA cannot flip a sampled discrete action.

    python oracle/gen_golden_a3c.py tests/golden
"""
import importlib
import os
import random
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle.gen_golden_acer import share_memory  # noqa: E402

# kind -> (discrete, lstm, episodic, constructor overrides)
KINDS = {
    "discrete_ff_t5": (True, False, True, dict(t_max=5)),
    "discrete_ff_t1": (True, False, False, dict(t_max=1)),
    "discrete_ff_keep_scale": (True, False, True, dict(t_max=5, keep_loss_scale_same=True)),
    "discrete_ff_norm_t_max": (True, False, False, dict(t_max=5, normalize_grad_by_t_max=True)),
    "discrete_ff_clip": (True, False, False, dict(t_max=5, max_grad_norm=1.0)),
    "discrete_lstm_t5": (True, True, False, dict(t_max=5)),
    "gauss_ff_t5": (False, False, False, dict(t_max=5)),
    "gauss_lstm_t1": (False, True, True, dict(t_max=1)),
}
A3C_KINDS = tuple(KINDS)
STEPS = 150
# record the parameters after every PARAM_STRIDE-th update
PARAM_STRIDE = {"discrete_lstm_t5": 5, "gauss_lstm_t1": 10}


def make_env(lib, kind, test=False):
    discrete, lstm, episodic, _ = KINDS[kind]
    ABC = importlib.import_module(lib.__name__ + ".envs.abc").ABC
    return ABC(size=2, discrete=discrete, episodic=episodic or test,
               partially_observable=lstm, deterministic=test)


def make_model(lib, discrete, lstm, obs_size, out_size, hidden=20):
    """tests/agents_tests/test_a3c.py:50-111."""
    import torch
    from torch import nn

    def weight_scale(layer, scale):
        with torch.no_grad():
            layer.weight.mul_(scale)
        return layer

    if discrete:
        head = lib.policies.SoftmaxCategoricalHead()
    else:
        head = lib.policies.GaussianHeadWithStateIndependentCovariance(
            action_size=out_size, var_type="diagonal", var_func=lambda x: torch.exp(2 * x),
            var_param_init=0)
    if lstm:
        v = lib.nn.RecurrentSequential(
            nn.LSTM(num_layers=1, input_size=obs_size, hidden_size=hidden),
            weight_scale(nn.Linear(hidden, 1), 1e-1))
        pi = lib.nn.RecurrentSequential(
            nn.LSTM(num_layers=1, input_size=obs_size, hidden_size=hidden),
            weight_scale(nn.Linear(hidden, out_size), 1e-1), head)
        return lib.nn.RecurrentBranched(pi, v)
    v = nn.Sequential(nn.Linear(obs_size, hidden), nn.Tanh(),
                      weight_scale(nn.Linear(hidden, 1), 1e-1))
    pi = nn.Sequential(nn.Linear(obs_size, hidden), nn.Tanh(),
                       weight_scale(nn.Linear(hidden, out_size), 1e-1), head)
    return lib.nn.Branched(pi, v)


def make_a3c_agent(lib, kind, device=None, **extra):
    discrete, lstm, _, over = KINDS[kind]
    env = make_env(lib, kind)
    out = env.action_space.n if discrete else env.action_space.low.size
    model = make_model(lib, discrete, lstm, env.observation_space.low.size, out)
    if device is not None:
        model.to(device)
    opt = lib.optimizers.SharedRMSpropEpsInsideSqrt(model.parameters())
    kw = dict(gamma=0.8, beta=1e-2, act_deterministically=True, recurrent=lstm)
    kw.update(over)
    kw.update(extra)
    return lib.agents.a3c.A3C(model, opt, **kw)


def flat_params(model):
    return np.concatenate([p.detach().cpu().numpy().ravel() for p in model.parameters()])


class _Recorder:
    """The env seen by train_agent, recording every action; a step hook records the
    statistics after every step, and the optimizer's step counts the updates and records the
    shared parameters after every ``stride``-th one."""

    def __init__(self, env, check):
        self.env = env
        self.actions = []
        self.stats = []
        self.params = []
        self.n_updates = 0
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

    def watch(self, agent, stride):
        step = agent.optimizer.step

        def recorded(*args, **kwargs):
            out = step(*args, **kwargs)
            self.n_updates += 1
            if self.n_updates % stride == 0:
                self.params.append(flat_params(agent.shared_model))
            return out

        agent.optimizer.step = recorded

    def __getattr__(self, name):
        return getattr(self.env, name)


def run(lib, kind, device=None, check=None, init=None, steps=STEPS, setup=None, **extra):
    import torch

    torch.manual_seed(3)
    agent = make_a3c_agent(lib, kind, device=device, **extra)
    if setup is not None:
        setup(agent)
    if init is not None:
        sd = {k[len("init__"):]: torch.tensor(init[k]) for k in init.files
              if k.startswith("init__")}
        agent.shared_model.load_state_dict(sd)
        agent.model.load_state_dict(sd)
    if agent.device.type == "cpu":
        share_memory(agent)
    g = {"init__" + k: v.detach().cpu().numpy().copy()
         for k, v in agent.shared_model.state_dict().items()}
    np.random.seed(9)
    torch.manual_seed(9)
    random.seed(9)
    _, _, episodic, _ = KINDS[kind]
    env = _Recorder(make_env(lib, kind), check)
    env.watch(agent, PARAM_STRIDE.get(kind, 1))
    with tempfile.TemporaryDirectory() as outdir:
        lib.experiments.train_agent(agent, env, steps, outdir,
                                    max_episode_len=None if episodic else 2,
                                    step_hooks=[env.hook])
    g.update(actions=np.array(env.actions), stats=np.array(env.stats, dtype=np.float64),
             stat_names=np.array([n for n, _ in agent.get_statistics()]),
             n_updates=np.array(env.n_updates),
             params=np.array(env.params).reshape(len(env.params), -1))
    return agent, g


def main(out_dir):
    from oracle.refimport import import_reference

    pfrl = import_reference()
    for kind in A3C_KINDS:
        _, g = run(pfrl, kind)
        np.savez_compressed(os.path.join(out_dir, "agent_trace_a3c_%s.npz" % kind), **g)
        print("wrote agent_trace_a3c_%s.npz" % kind, int(g["n_updates"]), "updates",
              dict(zip(g["stat_names"], g["stats"][-1])))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(HERE), "tests",
                                                             "golden"))
