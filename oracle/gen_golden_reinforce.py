"""Seeded runs of the reference's REINFORCE on its ABC toy environment ->
tests/golden/agent_trace_reinforce_<kind>.npz.

The models are the reference test's (tests/agents_tests/test_reinforce.py): a 20-unit
MLP or an LSTM ``RecurrentSequential``, with a softmax head or a state-independent
diagonal Gaussian head, Adam and beta = 1e-2.  The kinds cover batchsize 1 and 10,
``backward_separately`` on and off, ``max_grad_norm``, and episodes cut by
``train_max_episode_len`` = 2 (a reset without a terminal, which throws the episode
away).  Recorded: the initial parameters, the action of every step, ``average_entropy``
after every step and the parameters after every optimizer step.  The runs are short, so
that fp32 rounding on CUDA cannot flip a sampled discrete action.

    python oracle/gen_golden_reinforce.py tests/golden
"""
import importlib
import os
import random
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

# kind -> (discrete, lstm, max_episode_len, constructor overrides)
KINDS = {
    "discrete_ff_b1": (True, False, 2, dict(batchsize=1)),
    "discrete_ff_b10": (True, False, None, dict(batchsize=10, max_grad_norm=0.5)),
    "discrete_ff_b10_sep": (True, False, 2, dict(batchsize=10, backward_separately=True)),
    "discrete_lstm_b10": (True, True, 2, dict(batchsize=10)),
    "discrete_lstm_b10_sep": (True, True, None, dict(batchsize=10, backward_separately=True)),
    "gauss_ff_b1": (False, False, 2, dict(batchsize=1)),
    "gauss_ff_b10_sep": (False, False, None, dict(batchsize=10, backward_separately=True,
                                                   max_grad_norm=0.5)),
    "gauss_lstm_b10": (False, True, 2, dict(batchsize=10)),
}
REINFORCE_KINDS = tuple(KINDS)
STEPS = 200


def make_env(lib, kind, test=False):
    discrete, lstm, _, _ = KINDS[kind]
    ABC = importlib.import_module(lib.__name__ + ".envs.abc").ABC
    return ABC(size=2, discrete=discrete, episodic=True, partially_observable=lstm,
               deterministic=test)


def make_model(lib, discrete, lstm, obs_size, output_size, hidden=20):
    from torch import nn

    if discrete:
        head = lib.policies.SoftmaxCategoricalHead()
    else:
        head = lib.policies.GaussianHeadWithStateIndependentCovariance(
            output_size, var_type="diagonal")
    if lstm:
        return lib.nn.RecurrentSequential(
            nn.LSTM(num_layers=1, input_size=obs_size, hidden_size=hidden),
            nn.Linear(hidden, hidden), nn.LeakyReLU(), nn.Linear(hidden, output_size), head)
    return nn.Sequential(nn.Linear(obs_size, hidden), nn.LeakyReLU(),
                         nn.Linear(hidden, output_size), head)


def make_reinforce_agent(lib, kind, gpu=None, **extra):
    import torch

    discrete, lstm, _, over = KINDS[kind]
    env = make_env(lib, kind)
    out = env.action_space.n if discrete else env.action_space.low.size
    model = make_model(lib, discrete, lstm, env.observation_space.low.size, out)
    opt = torch.optim.Adam(model.parameters())
    kw = dict(beta=1e-2, act_deterministically=True, recurrent=lstm)
    kw.update(over)
    kw.update(extra)
    return lib.agents.REINFORCE(model, opt, gpu=gpu, **kw)


def flat_params(model):
    return np.concatenate([p.detach().cpu().numpy().ravel() for p in model.parameters()])


class _Recorder:
    """The env seen by train_agent, recording every action; a step hook records the
    statistics after every step, and the optimizer's step the parameters after it."""

    def __init__(self, env, check):
        self.env = env
        self.actions = []
        self.stats = []
        self.params = []
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

    def watch(self, agent):
        step = agent.optimizer.step

        def recorded(*args, **kwargs):
            out = step(*args, **kwargs)
            self.params.append(flat_params(agent.model))
            return out

        agent.optimizer.step = recorded

    def __getattr__(self, name):
        return getattr(self.env, name)


def run(lib, kind, gpu=None, check=None, init=None, steps=STEPS, setup=None, **extra):
    import torch

    torch.manual_seed(3)
    agent = make_reinforce_agent(lib, kind, gpu=gpu, **extra)
    if setup is not None:
        setup(agent)
    if init is not None:
        sd = {k[len("init__"):]: torch.tensor(init[k]) for k in init.files
              if k.startswith("init__")}
        agent.model.load_state_dict(sd)
    g = {"init__" + k: v.detach().cpu().numpy().copy()
         for k, v in agent.model.state_dict().items()}
    np.random.seed(9)
    torch.manual_seed(9)
    random.seed(9)
    env = _Recorder(make_env(lib, kind), check)
    env.watch(agent)
    with tempfile.TemporaryDirectory() as outdir:
        lib.experiments.train_agent(agent, env, steps, outdir,
                                    max_episode_len=KINDS[kind][2], step_hooks=[env.hook])
    g.update(actions=np.array(env.actions), stats=np.array(env.stats, dtype=np.float64),
             stat_names=np.array([n for n, _ in agent.get_statistics()]),
             params=np.array(env.params).reshape(len(env.params), -1))
    return agent, g


def main(out_dir):
    import warnings

    from oracle.refimport import import_reference

    pfrl = import_reference()
    warnings.simplefilter("ignore")  # the discarded episodes' warning
    for kind in REINFORCE_KINDS:
        _, g = run(pfrl, kind)
        np.savez_compressed(os.path.join(out_dir, "agent_trace_reinforce_%s.npz" % kind), **g)
        print("wrote agent_trace_reinforce_%s.npz" % kind, len(g["params"]), "updates",
              dict(zip(g["stat_names"], g["stats"][-1])))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(HERE), "tests",
                                                             "golden"))
