"""ACER update time: one replay update and one online update, the reference's formulation
(use_fused = False) against the fused path, alternated in one process on cuda:0.

Shapes:
  * atari-K4 / atari-K18: the Atari example's network (examples/atari/train_acer_ale.py:
    two convolutions, a 256-unit layer, the discrete head) on 4x84x84 uint8 frames with
    phi = ScaleU8(), t_max = 5, max_grad_norm = 40, trust region and truncation 10;
  * abc-mlp: the reference test's ABC network (one 20-unit layer, 2 actions), t_max 5.
Each update is timed with CUDA events around it (after a device synchronise), and the
host synchronisations torch reports inside it (sync debug mode "warn") are counted.
Medians over --reps updates after --warmup.  One JSON line, with the card's name and
power limit.

    python tools/bench_acer.py --reps 20
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

T_MAX = 5


def atari_model(pfrl, n_actions):
    acer = pfrl.agents.acer
    return nn.Sequential(
        nn.Conv2d(4, 16, 8, stride=4), nn.ReLU(), nn.Conv2d(16, 32, 4, stride=2), nn.ReLU(),
        nn.Flatten(), nn.Linear(2592, 256), nn.ReLU(),
        acer.ACERDiscreteActionHead(
            pi=nn.Sequential(nn.Linear(256, n_actions), pfrl.policies.SoftmaxCategoricalHead()),
            q=nn.Sequential(nn.Linear(256, n_actions),
                            pfrl.q_functions.DiscreteActionValueHead())))


def abc_model(pfrl):
    acer = pfrl.agents.acer
    return nn.Sequential(
        nn.Linear(4, 20), nn.LeakyReLU(),
        acer.ACERDiscreteActionHead(
            pi=nn.Sequential(nn.Linear(20, 2), pfrl.policies.SoftmaxCategoricalHead()),
            q=nn.Sequential(nn.Linear(20, 2), pfrl.q_functions.DiscreteActionValueHead())))


def make(shape, fused):
    import pfrl_b200 as pfrl
    from pfrl_b200.utils.phi import Identity, ScaleU8

    torch.manual_seed(0)
    if shape.startswith("atari"):
        K = int(shape.split("K")[1])
        model, phi, max_grad_norm = atari_model(pfrl, K), ScaleU8(), 40
        rng = np.random.RandomState(0)
        obs = lambda: rng.randint(0, 256, size=(4, 84, 84), dtype=np.uint8)  # noqa: E731
    else:
        K, model, phi, max_grad_norm = 2, abc_model(pfrl), Identity(), None
        rng = np.random.RandomState(0)
        obs = lambda: rng.randn(4).astype(np.float32)  # noqa: E731
    model.to("cuda:0")
    opt = pfrl.optimizers.SharedRMSpropEpsInsideSqrt(model.parameters(), lr=7e-4, eps=4e-3,
                                                     alpha=0.99)
    rbuf = pfrl.replay_buffers.EpisodicReplayBuffer(10 ** 4, device=0)
    agent = pfrl.agents.acer.ACER(model, opt, t_max=10 ** 9, gamma=0.99, replay_buffer=rbuf,
                                  phi=phi, n_times_replay=0, replay_start_size=1,
                                  max_grad_norm=max_grad_norm)
    agent.use_fused = fused
    # 300 transitions in episodes of 30 (cut without a terminal: the replay bootstraps)
    for t in range(300):
        s = obs()
        agent.act(s)
        agent.observe(obs(), float(rng.randn()), False, (t + 1) % 30 == 0)
    return agent, obs, rng


class Timer:
    def __init__(self):
        self.ms, self.syncs = [], []

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
        self.syncs.append(sum("synchroniz" in str(x.message) for x in w))


def one_round(agent, obs, rng, timers):
    from pfrl_b200.utils.batch_states import batch_states

    s = obs()
    for _ in range(T_MAX):  # the online history of t_max steps
        agent.act(s)
        s = obs()
        agent.observe(s, float(rng.randn()), False, False)
    statevar = batch_states([s], agent.device, agent.phi)
    agent.replay_buffer._flush()
    timers["online"](lambda: agent.update_on_policy(statevar))
    timers["replay"](agent.update_from_replay)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_acer.py measures on a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    res = {}
    for shape in ("atari-K4", "atari-K18", "abc-mlp"):
        arms = {}
        for name, fused in (("reference", False), ("fused", True)):
            agent, obs, rng = make(shape, fused)
            arms[name] = (agent, obs, rng, {"online": Timer(), "replay": Timer()})
        for _ in range(args.warmup + args.reps):
            for agent, obs, rng, timers in arms.values():
                one_round(agent, obs, rng, timers)
        res[shape] = {}
        for name, (_, _, _, timers) in arms.items():
            out = {}
            for part, tm in timers.items():
                ms = np.array(tm.ms[args.warmup:])
                out[part + "_ms_median"] = round(float(np.median(ms)), 3)
                out[part + "_syncs_median"] = int(np.median(tm.syncs[args.warmup:]))
            res[shape][name] = out
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                                "-i", "0"], capture_output=True, text=True).stdout.strip()
    except OSError:
        limit = "unknown"
    print(json.dumps({"card": name, "power_limit": limit, "t_max": T_MAX, "reps": args.reps,
                      "results": res}))


if __name__ == "__main__":
    main()
