"""Per-call times of the Rainbow training loop with graphs on (dev tool, GPU box):
batch_act / env.step / batch_observe (= append + 4 updates) for a GPU env and a host env."""
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from pfrl_b200.envs import SyntheticAtariVectorEnv  # noqa: E402
from pfrl_b200.replay_buffers import PrioritizedReplayBuffer  # noqa: E402

dev = torch.device("cuda", 0)
cap, B = 200000, 512
buf = PrioritizedReplayBuffer(cap, alpha=0.5, beta0=0.4, betasteps=None, normalize_by_max="memory",
                              num_steps=3, device=0, max_batch=512, part_capacity=cap + 4096)
g = torch.Generator(device=dev)
g.manual_seed(0)
rng = np.random.RandomState(0)
done = 0
while done < cap + 2:
    m = min(1 << 16, cap + 2 - done)
    fr = torch.randint(0, 256, (m + 4, 84, 84), dtype=torch.uint8, device=dev, generator=g)
    term = np.zeros(m, bool)
    term[-1] = True
    buf.append_trajectory(fr, rng.randint(0, 18, m).astype(np.int64),
                          rng.randint(-1, 2, m).astype(float), term)
    done += m
torch.backends.cudnn.allow_tf32 = False
agent = bench.make_rainbow_agent(buf, 0, B, cuda_graph=True)
for env_dev in (dev, "cpu", dev):
    env = SyntheticAtariVectorEnv(16, device=env_dev, seed=1)
    bench.rainbow_loop(agent, env, 4)
    torch.cuda.synchronize()
    obss = env.reset()
    t = {"act": 0.0, "step": 0.0, "observe": 0.0, "reset": 0.0}
    n = 12
    for _ in range(n):
        torch.cuda.synchronize(); t0 = time.perf_counter()
        a = agent.batch_act(obss)
        torch.cuda.synchronize(); t1 = time.perf_counter()
        obss, rs, dones, infos = env.step(a)
        torch.cuda.synchronize(); t2 = time.perf_counter()
        agent.batch_observe(obss, rs, dones, np.zeros(16, bool))
        torch.cuda.synchronize(); t3 = time.perf_counter()
        obss = env.reset(np.logical_not(dones))
        torch.cuda.synchronize(); t4 = time.perf_counter()
        t["act"] += t1 - t0; t["step"] += t2 - t1; t["observe"] += t3 - t2; t["reset"] += t4 - t3
    print("env on", env_dev, {k: round(v / n * 1e3, 3) for k, v in t.items()}, "ms per vector step;",
          "act graph:", agent._act_graph.graph is not None, "key", agent._act_graph.key)
