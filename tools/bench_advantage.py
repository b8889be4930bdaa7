"""Timings of the advantage-learning and DPP targets on one GPU (stand-alone; prints JSON lines).

(a) kernel: ops.losses.adv_td_loss forward + backward (k_adv_td_fwd + k_td_bwd) against the
    torch chain of the reference's target expression (pfrl/agents/al.py, pal.py,
    double_pal.py, dpp.py) plus compute_weighted_value_loss and its backward, for each mode
    at B in {32, 512, 4096}, nA = 18, with importance weights.  CUDA events around windows
    of at least --window-s seconds (the call count is sized from a calibration run), the
    two variants alternated, the median window reported.  With --count-launches the script
    instead counts the launches per call with torch.profiler: run it as a process of its
    own, so that tracing does not touch the timings.
(b) update: one PAL.update at the Nature-DQN Atari shape (84x84x4 uint8, nA = 18, B = 32,
    device PER with the fused replay step), fused loss vs use_fused_loss = False, each with
    and without cuda_graph.

    python tools/bench_advantage.py [--window-s 0.5] [--windows 7]
    python tools/bench_advantage.py --count-launches
"""
import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pfrl_b200.agents.dqn import compute_weighted_value_loss  # noqa: E402
from pfrl_b200.ops.losses import ADV_MODES, adv_td_loss  # noqa: E402

ALPHA, ETA = 0.9, 2.0


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or torch.cuda.get_device_name(0)


def torch_chain(mode, q, action, tq, tnq, nq, reward, discount, terminal, weights):
    """The reference's _compute_y_and_t target and weighted value loss, in torch."""
    def gather(x, a):
        return x.gather(1, a[:, None])[:, 0]

    def vmax(x):
        return gather(x, x.argmax(dim=1))

    y = gather(q, action)
    with torch.no_grad():
        if mode in ("al", "pal", "double_pal"):
            next_v = gather(tnq, nq.argmax(dim=1)) if mode == "double_pal" else vmax(tnq)
            t = reward + discount * (1.0 - terminal) * next_v
            adv = gather(tq, action) - vmax(tq)
            if mode != "al":
                adv = torch.max(adv, gather(tnq, action) - vmax(tnq))
            t = t + ALPHA * adv
        else:
            if mode == "dpp":
                L = lambda x: torch.sum(F.softmax(ETA * x, dim=1) * x, dim=1)  # noqa: E731
            elif mode == "dppl":
                L = lambda x: torch.logsumexp(ETA * x, dim=1) / ETA  # noqa: E731
            else:
                L = vmax
            t = gather(tq, action) + (reward + discount * (1 - terminal) * L(tnq)) - L(tq)
    return compute_weighted_value_loss(y, t, weights)


def fused(mode, q, action, tq, tnq, nq, reward, discount, terminal, weights):
    return adv_td_loss(q, action, tq, tnq, reward, discount, terminal, weights, mode,
                       alpha=ALPHA, eta=ETA, next_q=nq if mode == "double_pal" else None)[0]


def calls_per_window(fn, window_s):
    """Calls of fn that fill window_s seconds, from a timed calibration run."""
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 10
    while True:
        start.record()
        for _ in range(n):
            fn()
        end.record()
        torch.cuda.synchronize()
        s = start.elapsed_time(end) / 1e3
        if s >= 0.05:
            return max(n, int(math.ceil(n * window_s / s)))
        n *= 4


def time_windows(fns, window_s, windows):
    """Median ms per call of each fn over windows of >= window_s seconds, alternated
    between the fns; also returns the calls per window."""
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
          for _ in fns]
    res = [[] for _ in fns]
    for fn in fns:  # warm-up of every shape
        for _ in range(10):
            fn()
    iters = [calls_per_window(fn, window_s) for fn in fns]
    torch.cuda.synchronize()
    for _ in range(windows):
        for k, fn in enumerate(fns):
            ev[k][0].record()
            for _ in range(iters[k]):
                fn()
            ev[k][1].record()
            torch.cuda.synchronize()
            res[k].append(ev[k][0].elapsed_time(ev[k][1]) / iters[k])
    return [float(np.median(r)) for r in res], iters


def count_launches(fn):
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
               and "memcpy" not in e.name.lower() and "memset" not in e.name.lower())


def bench_kernel(window_s, windows, count):
    nA, dev = 18, "cuda"
    for B in (32, 512, 4096):
        g = torch.Generator(device=dev).manual_seed(B)
        q = torch.randn(B, nA, device=dev, generator=g).requires_grad_(True)
        tq, tnq, nq = (torch.randn(B, nA, device=dev, generator=g) for _ in range(3))
        action = torch.randint(0, nA, (B,), device=dev, generator=g)
        reward = torch.randn(B, device=dev, generator=g)
        discount = torch.full((B,), 0.99, device=dev)
        terminal = (torch.rand(B, device=dev, generator=g) < 0.1).float()
        weights = torch.rand(B, device=dev, generator=g) + 0.1
        for mode in ADV_MODES:
            args = (mode, q, action, tq, tnq, nq, reward, discount, terminal, weights)

            def step(f):
                def run():
                    q.grad = None
                    f(*args).backward()
                return run

            runs = [step(fused), step(torch_chain)]
            if count:
                print(json.dumps(dict(bench="adv_td_loss launches", mode=mode, B=B, nA=nA,
                                      fused=count_launches(runs[0]),
                                      torch=count_launches(runs[1]))), flush=True)
                continue
            ms, iters = time_windows(runs, window_s, windows)
            print(json.dumps(dict(
                bench="adv_td_loss", mode=mode, B=B, nA=nA, fused_us=round(ms[0] * 1e3, 2),
                torch_us=round(ms[1] * 1e3, 2), speedup=round(ms[1] / ms[0], 2),
                calls_per_window=iters)), flush=True)


def bench_update(window_s, windows):
    from pfrl_b200 import agents, explorers, q_functions
    from pfrl_b200.replay_buffers import PrioritizedReplayBuffer
    from pfrl_b200.utils import set_random_seed
    from pfrl_b200.utils.phi import ScaleU8

    rbuf = PrioritizedReplayBuffer(10 ** 5, alpha=0.5, beta0=0.4, betasteps=10 ** 6,
                                   num_steps=3, normalize_by_max="memory")
    rng = np.random.RandomState(0)
    n = 20000
    term = rng.rand(n) < 0.005
    term[-1] = True
    rbuf.append_trajectory(rng.randint(0, 256, size=(n + 4, 84, 84), dtype=np.uint8),
                           rng.randint(0, 18, size=n).astype(np.int64),
                           rng.randint(-1, 2, size=n).astype(np.float64), term)
    variants = []
    for use_fused in (True, False):
        for graph in (False, True):
            set_random_seed(0)
            q = q_functions.DuelingDQN(18)
            agent = agents.PAL(q, torch.optim.Adam(q.parameters(), 6.25e-5, eps=1.5e-4,
                                                   capturable=graph),
                               rbuf, 0.99, explorers.Greedy(), gpu=0, minibatch_size=32,
                               replay_start_size=1000, target_update_interval=10 ** 9,
                               phi=ScaleU8(), cuda_graph=graph)
            agent.use_fused_loss = use_fused

            def run(agent=agent):
                agent.update(rbuf.sample(32))
            variants.append(("fused" if use_fused else "torch", graph, run))
    ms, iters = time_windows([v[2] for v in variants], window_s, windows)
    for (loss, graph, _), t, n in zip(variants, ms, iters):
        print(json.dumps(dict(bench="PAL.update", loss=loss, cuda_graph=graph, B=32, nA=18,
                              us_per_update=round(t * 1e3, 1), calls_per_window=n)),
              flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window-s", type=float, default=0.5, help="seconds per timed window")
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--count-launches", action="store_true",
                    help="count launches per call with torch.profiler instead of timing")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_advantage needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    print(json.dumps(dict(card=card(), torch=torch.__version__)), flush=True)
    bench_kernel(args.window_s, args.windows, args.count_launches)
    if not args.count_launches:
        bench_update(args.window_s, args.windows)


if __name__ == "__main__":
    main()
