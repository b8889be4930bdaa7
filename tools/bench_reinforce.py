"""REINFORCE update time: the reference's formulation (use_fused = False, each step's
graph kept from acting) against the fused path, alternated in one process on cuda:0.

Shapes (batchsize 10, Adam, beta 1e-4 as in examples/gym/train_reinforce_gym.py):
  * abc-mlp: the reference test's ABC network (one 20-unit layer, 2 actions) on
    episodes of 3 steps;
  * cartpole-mlp: the gym example's network (two 200-unit LeakyReLU layers, 2 actions)
    on 4-float observations, episodes of 200 steps;
  * abc-lstm: the reference test's LSTM model (20 units) on episodes of 20 steps.
An update is the ``observe`` of the batch's last terminal, timed with CUDA events around
it after a device synchronise; the host synchronisations torch reports inside it (sync
debug mode "warn") are counted, and so are those of one ordinary act + observe step,
with the source lines torch attributes them to.
Medians over --reps updates after --warmup.  One JSON line, with the card's name and
power limit.

    python tools/bench_reinforce.py --reps 20
"""
import argparse
import json
import os
import subprocess
import sys
import warnings

import numpy as np
import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

BATCHSIZE = 10
SHAPES = {  # name -> (obs size, episode length, recurrent)
    "abc-mlp": (4, 3, False),
    "cartpole-mlp": (4, 200, False),
    "abc-lstm": (4, 20, True),
}


def make(shape, fused):
    import pfrl_b200 as pfrl

    obs_size, ep_len, lstm = SHAPES[shape]
    torch.manual_seed(0)
    head = pfrl.policies.SoftmaxCategoricalHead()
    if shape == "cartpole-mlp":
        model = nn.Sequential(nn.Linear(obs_size, 200), nn.LeakyReLU(0.2), nn.Linear(200, 200),
                              nn.LeakyReLU(0.2), nn.Linear(200, 2), head)
    elif lstm:
        model = pfrl.nn.RecurrentSequential(nn.LSTM(num_layers=1, input_size=obs_size,
                                                    hidden_size=20),
                                            nn.Linear(20, 20), nn.LeakyReLU(), nn.Linear(20, 2),
                                            head)
    else:
        model = nn.Sequential(nn.Linear(obs_size, 20), nn.LeakyReLU(), nn.Linear(20, 2), head)
    agent = pfrl.agents.REINFORCE(model, torch.optim.Adam(model.parameters(), lr=1e-3), gpu=0,
                                  beta=1e-4, batchsize=BATCHSIZE, recurrent=lstm)
    agent.use_fused = fused
    return agent, np.random.RandomState(0)


def _short(path):
    """A source path relative to this repository or to torch's package directory."""
    for root in (os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                 os.path.dirname(os.path.dirname(os.path.abspath(torch.__file__)))):
        if os.path.abspath(path).startswith(root + os.sep):
            return os.path.relpath(path, root)
    return os.path.basename(path)


class Timer:
    def __init__(self):
        self.ms, self.syncs = [], []
        self.sites = set()  # where in the source torch reported each synchronisation

    def __call__(self, fn):
        torch.cuda.synchronize()
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            start.record()
            try:
                fn()
            finally:
                end.record()
                torch.cuda.set_sync_debug_mode(0)
        torch.cuda.synchronize()
        self.ms.append(start.elapsed_time(end))
        syncs = [x for x in w if "synchroniz" in str(x.message)]
        self.syncs.append(len(syncs))
        self.sites.update("%s:%d" % (_short(x.filename), x.lineno) for x in syncs)


def one_update(agent, rng, shape, timers):
    """A batch of episodes; the last terminal's observe (the update) and one ordinary
    step are timed."""
    obs_size, ep_len, _ = SHAPES[shape]
    obs = lambda: rng.randn(obs_size).astype(np.float32)  # noqa: E731
    for e in range(BATCHSIZE):
        for t in range(ep_len):
            last = e == BATCHSIZE - 1 and t == ep_len - 1
            s = obs()
            if e == 0 and t == 0 and ep_len > 1:
                def step():
                    agent.act(s)
                    agent.observe(obs(), 0.0, False, False)

                timers["step"](step)
                continue
            agent.act(s)
            r, done = float(rng.randn()), t == ep_len - 1
            if last:
                timers["update"](lambda: agent.observe(obs(), r, True, False))
            else:
                agent.observe(obs(), r, done, False)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_reinforce.py measures on a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    res = {}
    for shape in SHAPES:
        arms = {}
        for name, fused in (("reference", False), ("fused", True)):
            agent, rng = make(shape, fused)
            arms[name] = (agent, rng, {"update": Timer(), "step": Timer()})
        for _ in range(args.warmup + args.reps):
            for agent, rng, timers in arms.values():
                one_update(agent, rng, shape, timers)
        res[shape] = {}
        for name, (agent, _, timers) in arms.items():
            assert agent._fused_record == (name == "fused")
            out = {}
            for part, tm in timers.items():
                out[part + "_ms_median"] = round(float(np.median(tm.ms[args.warmup:])), 3)
                out[part + "_syncs_median"] = int(np.median(tm.syncs[args.warmup:]))
                out[part + "_sync_sites"] = sorted(tm.sites)
            res[shape][name] = out
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                                "-i", "0"], capture_output=True, text=True).stdout.strip()
    except OSError:
        limit = "unknown"
    print(json.dumps({"card": name, "power_limit": limit, "batchsize": BATCHSIZE,
                      "reps": args.reps, "results": res}))


if __name__ == "__main__":
    main()
