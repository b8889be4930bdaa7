"""TRPO update time on the MuJoCo reproduction shape: the fused path with cuda_graph=True,
the fused path eager, and the torch formulation (use_fused=False), alternated in one
process.

Shape: obs 17, 6 Gaussian actions (state-independent covariance), 64-64 tanh policy and
value function, update_interval 5000 (10 envs x 500 steps of
SyntheticContinuousVectorEnv), vf_epochs 5, vf_batch_size 64, 20 CG iterations with
damping 0.1, 10 backtracks.  Per update: the policy part and the value-function part,
each timed with a host clock around a device synchronise, and the host synchronisations
torch reports (sync debug mode "warn") in each part.  One JSON line with the card name
and power limit.

    python tools/bench_trpo.py --reps 5
"""
import argparse
import json
import os
import subprocess
import sys
import time
import warnings

import numpy as np
import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def make_agent(fused, graph):
    import pfrl_b200 as pfrl

    torch.manual_seed(0)
    policy = nn.Sequential(nn.Linear(17, 64), nn.Tanh(), nn.Linear(64, 64), nn.Tanh(),
                           nn.Linear(64, 6),
                           pfrl.policies.GaussianHeadWithStateIndependentCovariance(
                               action_size=6, var_type="diagonal",
                               var_func=lambda x: torch.exp(2 * x), var_param_init=0))
    vf = nn.Sequential(nn.Linear(17, 64), nn.Tanh(), nn.Linear(64, 64), nn.Tanh(),
                       nn.Linear(64, 1))
    agent = pfrl.agents.TRPO(
        policy, vf, torch.optim.Adam(vf.parameters(), lr=1e-3),
        obs_normalizer=pfrl.nn.EmpiricalNormalization(17, clip_threshold=5), gpu=0,
        update_interval=5000, vf_epochs=5, vf_batch_size=64, conjugate_gradient_max_iter=20,
        conjugate_gradient_damping=0.1, line_search_max_backtrack=10, max_kl=0.01,
        cuda_graph=graph)
    agent.use_fused = fused
    return agent


class Timed:
    """Wraps an agent method: host clock around a device synchronise, and the number of
    synchronisations torch reports inside it."""

    def __init__(self, agent, name):
        self.fn = getattr(agent, name)
        self.times, self.syncs = [], []
        setattr(agent, name, self)

    def __call__(self, *a, **k):
        torch.cuda.synchronize()
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            t0 = time.perf_counter()
            try:
                out = self.fn(*a, **k)
            finally:
                torch.cuda.set_sync_debug_mode(0)
            torch.cuda.synchronize()
            self.times.append(time.perf_counter() - t0)
        self.syncs.append(sum("synchroniz" in str(x.message) for x in w))
        return out


def rollout_and_update(agent, env, steps):
    obs = env.reset()
    for _ in range(steps):
        a = agent.batch_act(obs)
        obs, r, d, info = env.step(a)
        agent.batch_observe(obs, r, d, [False] * len(d))


def main():
    from pfrl_b200.envs.synthetic import SyntheticContinuousVectorEnv

    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    arms = {}
    for name, fused, graph in (("fused_graph", True, True), ("fused", True, False),
                               ("torch", False, False)):
        agent = make_agent(fused, graph)
        arms[name] = (agent, Timed(agent, "_update_policy_fused" if fused else
                                   "_update_policy_torch"), Timed(agent, "_update_vf"),
                      SyntheticContinuousVectorEnv(10, 17, 6, seed=1))
    # the first three rounds warm every arm up (the graphed arm captures on its third)
    for rep in range(args.reps + 3):
        for name in arms:
            agent, _, _, env = arms[name]
            rollout_and_update(agent, env, 500)
    res = {}
    for name, (agent, pol, vf, _) in arms.items():
        p, v = np.array(pol.times[3:]) * 1e3, np.array(vf.times[3:]) * 1e3
        res[name] = dict(
            policy_ms=[round(x, 2) for x in p], vf_ms=[round(x, 2) for x in v],
            policy_ms_median=round(float(np.median(p)), 2),
            vf_ms_median=round(float(np.median(v)), 2),
            update_ms_median=round(float(np.median(p + v)), 2),
            policy_syncs=pol.syncs[3:], vf_syncs=vf.syncs[3:])
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                                "-i", "0"], capture_output=True, text=True).stdout.strip()
    except OSError:
        limit = "unknown"
    print(json.dumps({"card": name, "power_limit": limit, "shape": "obs17-act6-64x64-N5000",
                      "results": res}))


if __name__ == "__main__":
    main()
