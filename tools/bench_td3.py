"""One TD3 and one DDPG update at MuJoCo sizes on one GPU, in three modes; one JSON line.

    python tools/bench_td3.py [--window 1.0] [--windows 5]

Shapes: obs 17, action 6, 256 x 256 policy and critics, minibatch 256, a device replay
buffer holding 10^4 transitions, device-side phi.  Modes:

* ``torch``: ``use_fused = False``, the reference's eager formulation;
* ``fused``: the fused critic update (k_td3_smooth, k_td3_critic_loss), eager;
* ``graph``: the fused update with ``cuda_graph=True``.

Each update is timed with a host clock around a device synchronise, after a warm-up (which
includes the graph captures), over windows of ``--window`` seconds that alternate between the
six agents; the median window is reported.  Kernel times come from torch.profiler in a process
of its own (``--profile``, started by the default run), so the profiler does not touch the
timed runs.  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

OBS, ACT, HIDDEN, BATCH, FILL = 17, 6, 256, 256, 10 ** 4
MODES = (("torch", False, False), ("fused", True, False), ("graph", True, True))
KERNELS = ("k_td3_smooth", "k_td3_critic_loss", "k_polyak")


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True).stdout
    return out.strip().splitlines()[0] if out.strip() else torch.cuda.get_device_name()


def make_agent(kind, fused, graph):
    from pfrl_b200 import agents, explorers, policies
    from pfrl_b200 import nn as pnn
    from pfrl_b200.replay_buffers import ReplayBuffer
    from pfrl_b200.utils.phi import Identity

    torch.manual_seed(0)

    def mlp(n_in, n_out):
        return [nn.Linear(n_in, HIDDEN), nn.ReLU(), nn.Linear(HIDDEN, HIDDEN), nn.ReLU(),
                nn.Linear(HIDDEN, n_out)]

    def critic():
        return nn.Sequential(pnn.ConcatObsAndAction(), *mlp(OBS + ACT, 1))

    policy = nn.Sequential(*mlp(OBS, ACT), nn.Tanh(), policies.DeterministicHead())
    rbuf = ReplayBuffer(10 ** 5, device=0)
    adam = lambda m: torch.optim.Adam(m.parameters(), lr=3e-4)  # noqa: E731
    ex = explorers.AdditiveGaussian(0.1, -1, 1)
    common = dict(gpu=0, replay_start_size=BATCH, minibatch_size=BATCH, phi=Identity(),
                  cuda_graph=graph)
    if kind == "td3":
        q1, q2 = critic(), critic()
        agent = agents.TD3(policy, q1, q2, adam(policy), adam(q1), adam(q2), rbuf, 0.99, ex,
                           **common)
    else:
        q = critic()
        agent = agents.DDPG(policy, q, adam(policy), adam(q), rbuf, 0.99, ex,
                            target_update_method="soft", soft_update_tau=5e-3, **common)
    agent.use_fused = fused
    rng = np.random.RandomState(0)
    s = rng.randn(FILL + 1, OBS).astype(np.float32)
    a = rng.uniform(-1, 1, size=(FILL, ACT)).astype(np.float32)
    r = rng.randn(FILL).astype(np.float32)
    for t in range(FILL):
        done = t % 1000 == 999
        rbuf.append(state=s[t], action=a[t], reward=float(r[t]), next_state=s[t + 1],
                    next_action=None, is_state_terminal=done)
        if done:
            rbuf.stop_current_episode()
    return agent


def one_update(agent):
    agent.update(agent.replay_buffer.sample(BATCH))


def arms():
    return [(kind, mode, make_agent(kind, fused, graph))
            for kind in ("td3", "ddpg") for mode, fused, graph in MODES]


def window_ms(agent, seconds):
    """Milliseconds per update over at least ``seconds`` of back-to-back updates."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n = 0
    while True:
        for _ in range(20):
            one_update(agent)
        n += 20
        if time.perf_counter() - t0 >= seconds:
            break
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / n


def profile(updates=50):
    """Device time per update of each kernel of KERNELS, and of all kernels, per arm."""
    from torch.profiler import ProfilerActivity, profile as tprofile

    out = {}
    for kind, mode, agent in arms():
        for _ in range(10):  # warm-up, and the graph captures
            one_update(agent)
        torch.cuda.synchronize()
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(updates):
                one_update(agent)
            torch.cuda.synchronize()
        row = {"kernels_per_update": 0.0, "kernel_us_per_update": 0.0}
        for e in prof.events():
            if e.device_type != torch.autograd.DeviceType.CUDA or e.name.startswith("Memcpy") \
                    or e.name.startswith("Memset"):
                continue
            row["kernels_per_update"] += 1 / updates
            row["kernel_us_per_update"] += e.time_range.elapsed_us() / updates
            for k in KERNELS:
                if k + "(" in e.name or e.name.endswith(k):
                    row.setdefault(k + "_us", []).append(e.time_range.elapsed_us())
        for k in KERNELS:
            if k + "_us" in row:
                t = row[k + "_us"]
                row[k + "_calls_per_update"] = len(t) / updates
                row[k + "_us"] = round(statistics.median(t), 3)
        row["kernels_per_update"] = round(row["kernels_per_update"], 2)
        row["kernel_us_per_update"] = round(row["kernel_us_per_update"], 2)
        out["%s_%s" % (kind, mode)] = row
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=1.0, help="seconds per timed window")
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--profile", action="store_true",
                    help="only the torch.profiler kernel times (run in a process of its own)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_td3.py measures on a CUDA device; none found")
    torch.backends.cuda.matmul.allow_tf32 = False
    if args.profile:
        print(json.dumps(profile()), flush=True)
        return
    result = dict(bench="td3_ddpg_update", card=card(), torch=torch.__version__, obs=OBS,
                  action=ACT, hidden="256x256", minibatch=BATCH,
                  replay="device ReplayBuffer, %d transitions" % FILL)
    runs = arms()
    for _, _, agent in runs:
        for _ in range(10):
            one_update(agent)
    times = {(kind, mode): [] for kind, mode, _ in runs}
    for _ in range(args.windows):
        for kind, mode, agent in runs:
            times[kind, mode].append(window_ms(agent, args.window))
    result["update_ms"] = {"%s_%s" % k: round(statistics.median(v), 4) for k, v in times.items()}
    result["update_ms_spread"] = {"%s_%s" % k: [round(min(v), 4), round(max(v), 4)]
                                  for k, v in times.items()}
    prof = subprocess.run([sys.executable, os.path.abspath(__file__), "--profile"],
                          capture_output=True, text=True, check=True)
    result["kernels"] = json.loads(prof.stdout.strip().splitlines()[-1])
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
