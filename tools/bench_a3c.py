"""A3C update time: the reference's formulation (use_fused = False) against the fused path,
alternated in one process on cuda:0.

Shapes (gamma 0.99, beta 1e-2, SharedRMSpropEpsInsideSqrt as in
examples/atari/reproduction/a3c/train_a3c.py):
  * abc-mlp: the reference test's ABC network (20-unit policy and value branches, 2
    actions) at t_max 5;
  * atari-t5 / atari-t20: the Atari example's network (conv 16 8x8/4, conv 32 4x4/2, a
    256-unit layer, a Branched softmax head over 18 actions and a value head) on synthetic
    uint8 84x84x4 observations scaled by 1/255, at t_max 5 and 20;
  * abc-lstm: the reference test's LSTM model (20 units) at t_max 5.
An update is the ``observe`` that completes a segment of t_max steps (no terminal, so it
bootstraps), timed with CUDA events around it after a device synchronise; the host
synchronisations torch reports inside it (sync debug mode "warn") are counted, and so are
those of one ordinary act + observe step, with the source lines torch attributes them to.
Medians over --reps updates after --warmup.  One JSON line, with the card's name and
power limit.

    python tools/bench_a3c.py --reps 30
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_reinforce import Timer  # noqa: E402

SHAPES = {  # name -> (t_max, network)
    "abc-mlp": (5, "mlp"),
    "atari-t5": (5, "atari"),
    "atari-t20": (20, "atari"),
    "abc-lstm": (5, "lstm"),
}
N_ACTIONS_ATARI = 18


def make(shape, fused):
    import pfrl_b200 as pfrl
    from oracle.gen_golden_a3c import make_model

    t_max, net = SHAPES[shape]
    torch.manual_seed(0)
    phi = lambda x: x  # noqa: E731
    if net == "atari":
        model = nn.Sequential(
            nn.Conv2d(4, 16, 8, stride=4), nn.ReLU(), nn.Conv2d(16, 32, 4, stride=2), nn.ReLU(),
            nn.Flatten(), nn.Linear(2592, 256), nn.ReLU(),
            pfrl.nn.Branched(nn.Sequential(nn.Linear(256, N_ACTIONS_ATARI),
                                           pfrl.policies.SoftmaxCategoricalHead()),
                             nn.Linear(256, 1)))
        phi = lambda x: np.asarray(x, dtype=np.float32) / 255  # noqa: E731
    else:
        model = make_model(pfrl, True, net == "lstm", 4, 2)
    model.to("cuda:0")
    opt = pfrl.optimizers.SharedRMSpropEpsInsideSqrt(model.parameters(), lr=7e-4, eps=1e-1,
                                                     alpha=0.99)
    agent = pfrl.agents.A3C(model, opt, t_max=t_max, gamma=0.99, beta=1e-2, phi=phi,
                            recurrent=net == "lstm")
    agent.use_fused = fused
    return agent, np.random.RandomState(0)


def observation(rng, shape):
    if SHAPES[shape][1] == "atari":
        return rng.randint(0, 256, (4, 84, 84), dtype=np.uint8)
    return rng.randn(4).astype(np.float32)


def one_update(agent, rng, shape, timers):
    """One segment of t_max steps; its first step and its last observe (the update) are
    timed."""
    t_max = SHAPES[shape][0]
    for t in range(t_max):
        s, s2, r = observation(rng, shape), observation(rng, shape), float(rng.randn())
        if t == t_max - 1:
            agent.act(s)
            timers["update"](lambda: agent.observe(s2, r, False, False))
        elif t == 0:
            def step():
                agent.act(s)
                agent.observe(s2, r, False, False)

            timers["step"](step)
        else:
            agent.act(s)
            agent.observe(s2, r, False, False)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_a3c.py measures on a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    from pfrl_b200.ops import a3c as fused_ops

    launches = []
    real = fused_ops.loss_grads

    def counted(*a, **kw):
        launches.append(1)
        return real(*a, **kw)

    fused_ops.loss_grads = counted
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
            out = {}
            for part, tm in timers.items():
                out[part + "_ms_median"] = round(float(np.median(tm.ms[args.warmup:])), 3)
                out[part + "_syncs_median"] = int(np.median(tm.syncs[args.warmup:]))
                out[part + "_sync_sites"] = sorted(tm.sites)
            res[shape][name] = out
        res[shape]["speedup"] = round(res[shape]["reference"]["update_ms_median"]
                                      / res[shape]["fused"]["update_ms_median"], 2)
    # every fused update launched the kernel once; no reference update did
    assert len(launches) == len(SHAPES) * (args.warmup + args.reps), len(launches)
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                                "-i", "0"], capture_output=True, text=True).stdout.strip()
    except OSError:
        limit = "unknown"
    print(json.dumps({"card": name, "power_limit": limit, "reps": args.reps,
                      "results": res}))


if __name__ == "__main__":
    main()
