"""DRQN measurement at the shapes of the reference's Atari DRQN example
(examples/atari/train_drqn_ale.py): B = 32 sequences of L = 10, 84x84x4 uint8 frames
(LazyFrames sharing), a Nature conv stack + LSTM-512 DoubleDQN, a 10^6-transition
EpisodicReplayBuffer.  Needs a GPU; prints one JSON line.

  * gather: k_seq_gather alone -- its kernel time from torch.profiler, and the bytes the
    algorithm moves (frames read once per packed row and side, f32 rows written, the
    first records' LSTM states read and written) over that time, against the H100 SXM
    data-sheet HBM3 bandwidth (3.35 TB/s);
  * update: one full update_from_episodes (sample, batch, forwards, loss, backward, Adam),
    host clock around a device synchronise, on the device path (EpisodicReplayBuffer +
    k_seq_gather) and on the host path (HostEpisodicReplayBuffer + batch_recurrent_
    experiences + H2D on the same GPU; numpy states, as the reference stores them).  The
    host buffer holds --host-fill transitions: its per-update cost does not depend on its
    size, only on the sampled batch.

    python tools/bench_drqn.py [--fill 1000000] [--iters 200]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import pfrl_b200  # noqa: E402
from pfrl_b200 import replay_buffers  # noqa: E402
from pfrl_b200.replay_buffer import batch_recurrent_experiences  # noqa: E402
from pfrl_b200.utils.lazy_frames import LazyFrames  # noqa: E402

HBM_PEAK_GBS = 3350.0
B, L, STACK, H = 32, 10, 4, 512


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.splitlines()[0].split(",")]
        return name, power
    except Exception:  # noqa: BLE001
        return torch.cuda.get_device_name(0), "unknown"


def fill(buf, n, device, ep_len=200, seed=0, host=False):
    """n transitions of episodes of ep_len steps: one new 84x84 frame per step, LSTM-512
    (h, c) states for both sides of every transition."""
    g = torch.Generator(device=device).manual_seed(seed)
    pool = torch.randint(0, 256, (4096, 1, 84, 84), dtype=torch.uint8, device=device,
                         generator=g)
    states = torch.randn(256, 2, 1, H, device=device, generator=g)  # [layers, H] per env, as the agent stores
    if host:
        pool, states = pool.cpu().numpy(), states.cpu().numpy()
    rng = np.random.RandomState(seed)
    frames = [pool[i] for i in range(STACK)]
    for t in range(n):
        s = LazyFrames(list(frames), stack_axis=0)
        frames = frames[1:] + [pool[(t + STACK) % len(pool)]]
        ns = LazyFrames(list(frames), stack_axis=0)
        k = t % len(states)
        # one entry per recurrent child of the model: the LSTM's (h, c)
        rs = ((states[k, 0], states[k, 1]),)
        k1 = (k + 1) % len(states)
        nrs = ((states[k1, 0], states[k1, 1]),)
        end = (t + 1) % ep_len == 0
        buf.append(s, int(rng.randint(18)), float(rng.randn()), ns, is_state_terminal=end,
                   recurrent_state=rs, next_recurrent_state=nrs)


def make_agent(rbuf):
    from torch import nn

    torch.manual_seed(0)
    q = pfrl_b200.nn.RecurrentSequential(
        nn.Conv2d(4, 32, 8, stride=4), nn.ReLU(), nn.Conv2d(32, 64, 4, stride=2), nn.ReLU(),
        nn.Conv2d(64, 64, 3, stride=1), nn.Flatten(), nn.Linear(3136, 512), nn.ReLU(),
        nn.LSTM(512, H), nn.Linear(H, 18), pfrl_b200.q_functions.DiscreteActionValueHead())
    return pfrl_b200.agents.DoubleDQN(
        q, torch.optim.Adam(q.parameters(), 1e-4, eps=1e-2), rbuf, 0.99,
        pfrl_b200.explorers.Greedy(), gpu=0, replay_start_size=10 ** 9 if rbuf.capacity is None
        else rbuf.capacity, minibatch_size=B, target_update_interval=10 ** 6, recurrent=True,
        episodic_update_len=L, phi=pfrl_b200.utils.phi.ScaleU8())


def time_updates(agent, rbuf, iters, warmup=10):
    for _ in range(warmup):
        agent.update_from_episodes(rbuf.sample_episodes(B, L))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        agent.update_from_episodes(rbuf.sample_episodes(B, L))
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / iters * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--fill", type=int, default=10 ** 6)
    ap.add_argument("--host-fill", type=int, default=20000)
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_drqn needs a GPU")
    dev = torch.device("cuda:0")
    name, power = card()
    np.random.seed(0)

    buf = replay_buffers.EpisodicReplayBuffer(10 ** 6, device=dev)
    t0 = time.perf_counter()
    fill(buf, args.fill, dev)
    buf._flush()
    torch.cuda.synchronize()
    fill_s = time.perf_counter() - t0
    phi = pfrl_b200.utils.phi.ScaleU8()

    # gather alone
    eps = [buf.sample_episodes(B, L).sorted_by_length() for _ in range(64)]
    for e in eps[:8]:
        batch_recurrent_experiences(e, dev, phi, 0.99)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for e in eps:
            batch_recurrent_experiences(e, dev, phi, 0.99)
        torch.cuda.synchronize()
    times = [ev.device_time for ev in prof.events() if ev.name.startswith("k_seq_gather")]
    gather_us = float(np.mean(times)) if times else float("nan")
    rows = B * L
    part = 84 * 84
    D = 2 * H  # floats per stored state: (h, c) of one layer
    nbytes = (2 * rows * STACK * part              # u8 frames read, both sides
              + 2 * rows * STACK * part * 4        # f32 rows written
              + rows * (8 + 8 + 4 + 4)             # action, reward (fp64) read; action, f32 out
              + 2 * B * D * 4 * 2)                 # first records' states read + written
    gather = dict(kernel_us=gather_us, launches_timed=len(times), bytes=nbytes,
                  gbs=nbytes / gather_us / 1e3, hbm_share=nbytes / gather_us / 1e3 / HBM_PEAK_GBS)

    # full update, device path
    agent = make_agent(buf)
    dev_ms = time_updates(agent, buf, args.iters)

    # full update, host path on the same GPU
    hbuf = replay_buffers.HostEpisodicReplayBuffer(args.host_fill)
    fill(hbuf, args.host_fill, dev, host=True)
    hagent = make_agent(hbuf)
    host_ms = time_updates(hagent, hbuf, max(20, args.iters // 4))

    print(json.dumps(dict(
        bench="drqn", card=name, power_limit=power, B=B, L=L, capacity=10 ** 6,
        filled=len(buf), fill_seconds=fill_s, gather=gather,
        update_ms=dict(device_path=dev_ms, host_path=host_ms),
        host_path_buffer=args.host_fill, hbm_peak_gbs_datasheet=HBM_PEAK_GBS)))


if __name__ == "__main__":
    main()
