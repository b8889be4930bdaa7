"""Recurrent PPO update on one GPU: the pack kernel and one whole update.

    python tools/bench_recurrent_ppo.py [--shape atari|mlp|both] [--reps 3]

Shapes:
  atari  8 envs, update_interval 1024 (T = 128), minibatch 256, 4 epochs, 1x84x84 u8 obs,
         Nature conv -> GRU-512 -> policy / value heads
  mlp    256 envs, update_interval 2048 (T = 8), minibatch 64, 10 epochs, obs 376, 17
         Gaussian actions, GRU-64

Per shape it prints, in one JSON line with the card name and power limit:
  - k_rollout_seq_gather's mean time per launch from torch.profiler (a separate run),
    with the bytes it moves (computed from the shapes) over that time against 3.35 TB/s;
  - one full update (dataset pass + every minibatch step), host clock around a device
    synchronise, the kernel path and use_fused=False alternated in the same process.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from pfrl_b200 import nn as pnn  # noqa: E402
from pfrl_b200.agents.ppo import PPO  # noqa: E402
from pfrl_b200.policies import GaussianHeadWithStateIndependentCovariance, SoftmaxCategoricalHead  # noqa: E402

HBM_BYTES_PER_S = 3.35e12

SHAPES = {
    "atari": dict(E=8, interval=1024, mb=256, epochs=4, obs=(1, 84, 84), u8=True, hidden=512,
                  n_actions=6),
    "mlp": dict(E=256, interval=2048, mb=64, epochs=10, obs=(376,), u8=False, hidden=64,
                n_actions=17),
}


def make_model(s):
    if s["u8"]:
        trunk = nn.Sequential(nn.Conv2d(1, 32, 8, 4), nn.ReLU(), nn.Conv2d(32, 64, 4, 2),
                              nn.ReLU(), nn.Conv2d(64, 64, 3, 1), nn.ReLU(), nn.Flatten(),
                              nn.Linear(3136, 512), nn.ReLU())
        pi = nn.Sequential(nn.Linear(s["hidden"], s["n_actions"]), SoftmaxCategoricalHead())
        return pnn.RecurrentSequential(trunk, nn.GRU(512, s["hidden"]),
                                       pnn.Branched(pi, nn.Linear(s["hidden"], 1)))
    pi = nn.Sequential(nn.Linear(s["hidden"], s["n_actions"]),
                       GaussianHeadWithStateIndependentCovariance(
                           action_size=s["n_actions"], var_type="diagonal",
                           var_func=lambda x: torch.exp(2 * x), var_param_init=0))
    return pnn.RecurrentSequential(nn.GRU(s["obs"][0], s["hidden"]),
                                   pnn.Branched(pi, nn.Linear(s["hidden"], 1)))


def make_agent(s, seed=0):
    torch.manual_seed(seed)
    model = make_model(s)
    phi = (lambda x: np.asarray(x, dtype=np.float32) / 255.0) if s["u8"] else (lambda x: x)
    return PPO(model, torch.optim.Adam(model.parameters(), lr=2.5e-4), gpu=0, phi=phi,
               update_interval=10 ** 12, minibatch_size=s["mb"], epochs=s["epochs"],
               recurrent=True, max_recurrent_sequence_len=None)


def fill(agent, s, seed=0):
    """One rollout of T = interval / E steps with episodes of random length."""
    rng = np.random.RandomState(seed)
    E, T = s["E"], s["interval"] // s["E"]

    def obs():
        if s["u8"]:
            return [rng.randint(0, 256, s["obs"]).astype(np.uint8) for _ in range(E)]
        return [rng.randn(*s["obs"]).astype(np.float32) for _ in range(E)]

    o = obs()
    for _ in range(T):
        agent.batch_act(o)
        o = obs()
        agent.batch_observe(o, rng.randn(E).astype(np.float32), rng.rand(E) < 0.01,
                            np.zeros(E, bool))
    return {k: list(getattr(agent, k)) if isinstance(getattr(agent, k), list)
            else getattr(agent, k)
            for k in ("_states", "_next_states", "_actions", "_rewards", "_nonterminal", "_cut",
                      "_rstates", "_rpresent", "_segments", "_seg_start")}


def restore(agent, saved):
    for k, v in saved.items():
        setattr(agent, k, list(v))


def one_update(agent, saved):
    restore(agent, saved)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    agent._update_recurrent_from_rollout()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def pack_bytes(s, agent, saved):
    """Bytes the update's packs read and write: the dataset pass (2 obs + action, index,
    2 state sides) and the minibatches (obs, action, 4 f32 scalars, 1 state side)."""
    N = s["interval"]
    obs_b = int(np.prod(s["obs"])) * (1 if s["u8"] else 4)
    act_b = 8 if s["u8"] else 4 * s["n_actions"]
    D = agent._state_spec.row_floats
    n_eps = len(saved["_segments"]) + s["E"]
    data = N * (2 * obs_b + act_b + 8) + 2 * n_eps * D * 4
    mbs = (N // s["mb"]) * s["epochs"]
    minib = s["epochs"] * N * (obs_b + act_b + 16)
    return 2 * data, 2 * minib, mbs


def bench(name, reps):
    s = SHAPES[name]
    agent = make_agent(s)
    saved = fill(agent, s)
    one_update(agent, saved)  # warm-up (and lazy allocations)
    agent.use_fused = False
    one_update(agent, saved)
    times = {"kernel": [], "torch": []}
    for _ in range(reps):
        for fused in (True, False):
            agent.use_fused = fused
            times["kernel" if fused else "torch"].append(one_update(agent, saved))
    agent.use_fused = True
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        one_update(agent, saved)
    k = [e for e in prof.key_averages() if "k_rollout_seq_gather" in e.key]
    launches = k[0].count if k else 0
    dev_us = (k[0].device_time_total if k else float("nan"))
    data_b, mb_b, n_mb = pack_bytes(s, agent, saved)
    moved = data_b + mb_b
    return {
        "shape": name,
        "update_s_kernel": min(times["kernel"]),
        "update_s_torch": min(times["torch"]),
        "pack_launches_per_update": launches,
        "pack_us_per_update": dev_us,
        "pack_bytes_per_update": moved,
        "pack_fraction_of_hbm_peak": moved / (dev_us * 1e-6) / HBM_BYTES_PER_S if k else None,
        "minibatches_per_update": n_mb,
    }


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                                "-i", "0"], capture_output=True, text=True, timeout=30).stdout
        limit = limit.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="both", choices=["atari", "mlp", "both"])
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    names = ["atari", "mlp"] if args.shape == "both" else [args.shape]
    name, limit = card()
    out = {"card": name, "power_limit": limit, "results": [bench(n, args.reps) for n in names]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
