"""NAF kernels against the reference's torch chains on one GPU; one JSON line per result.

    python tools/bench_naf.py [--reps 200] [--windows 7]

* loss: the fused target-and-loss forward + backward (ops.naf.td_loss) against the reference's
  formulation (QuadraticActionValue members, the target, the Huber loss, autograd), per mode,
  at B in {32, 512, 4096} and n in {1, 6, 17};
* head: P = L L^T forward + backward (ops.naf.head) against exp + lower_triangular_matrix +
  matmul;
* update: one DQN update at a MuJoCo-like shape (obs 17, n = 6, 2 x 256 hidden, B = 256) on the
  device PrioritizedReplayBuffer with the fused replay step (sample, gather and the previous
  update's priority write-back in one launch): the fused NAF kernels against
  ``use_fused_loss = False``, each eager and with ``cuda_graph=True``;
* ``--count-launches``: kernel and graph launches per update of each arm, counted by
  torch.profiler in a process of its own (the default run starts it), so the profiler does not
  touch the timed runs.

Both arms run on the same inputs; the arms alternate window by window, each window is timed
with CUDA events over ``--reps`` calls, and the median window is reported.  The first line
names the card and its power limit, read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from pfrl_b200.action_value import QuadraticActionValue  # noqa: E402
from pfrl_b200.agents.dqn import compute_weighted_value_loss  # noqa: E402
from pfrl_b200.functions.lower_triangular_matrix import lower_triangular_matrix  # noqa: E402
from pfrl_b200.ops import naf  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True).stdout
    return out.strip().splitlines()[0] if out.strip() else torch.cuda.get_device_name()


def timed(fns, reps, windows):
    """Median per-call milliseconds of each fn, windows alternating between the fns."""
    for f in fns:
        for _ in range(5):  # past a graphed arm's warm-up and capture
            f()
    times = [[] for _ in fns]
    for _ in range(windows):
        for k, f in enumerate(fns):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(reps):
                f()
            b.record()
            b.synchronize()
            times[k].append(a.elapsed_time(b) / reps)
    return [sorted(t)[len(t) // 2] for t in times]


def problem(B, n):
    g = torch.Generator(device="cuda").manual_seed(B + n)

    def net():
        L = torch.tril(torch.randn(B, n, n, device="cuda", generator=g) * 0.3)
        return (torch.randn(B, n, device="cuda", generator=g),
                L @ L.transpose(1, 2) + 0.1 * torch.eye(n, device="cuda"),
                torch.randn(B, 1, device="cuda", generator=g))

    lo, hi = -torch.ones(n, device="cuda"), torch.ones(n, device="cuda")
    batch = dict(action=torch.randn(B, n, device="cuda", generator=g),
                 reward=torch.randn(B, device="cuda", generator=g),
                 discount=torch.full((B,), 0.99, device="cuda"),
                 is_state_terminal=(torch.rand(B, device="cuda", generator=g) < 0.1).float(),
                 weights=torch.rand(B, device="cuda", generator=g))
    return [net() for _ in range(4)], lo, hi, batch


def torch_target(mode, b, tq, tnq, nq, alpha):
    """The reference agents' targets (dqn.py, double_dqn.py, al.py, pal.py, double_pal.py,
    dpp.py) over QuadraticActionValue."""
    a = b["action"]
    if mode in ("double_dqn", "double_pal"):
        next_v = tnq.evaluate_actions(nq.greedy_actions)
    else:
        next_v = tnq.max
    bell = b["reward"] + b["discount"] * (1.0 - b["is_state_terminal"]) * next_v
    if mode in ("dqn", "double_dqn"):
        return bell
    if mode == "dpp_greedy":
        return tq.evaluate_actions(a) + bell - tq.max
    adv = tq.compute_advantage(a)
    if mode != "al":
        adv = torch.max(adv, tnq.compute_advantage(a))
    return bell + alpha * adv


def bench_loss(mode, B, n, reps, windows):
    nets, lo, hi, b = problem(B, n)
    (mu, mat, v), t, tn, nx = nets
    mu, mat, v = (x.clone().requires_grad_() for x in (mu, mat, v))
    q = lambda m, p, vv: QuadraticActionValue(m, p, vv, min_action=lo, max_action=hi)  # noqa
    tq, tnq, nq = q(*t), q(*tn), q(*nx)

    def fused():
        loss = naf.td_loss(q(mu, mat, v), b["action"], tnq, b["reward"], b["discount"],
                           b["is_state_terminal"], b["weights"], mode, target=tq,
                           next_online=nq, alpha=0.9)[0]
        loss.backward()

    def reference():
        y = q(mu, mat, v).evaluate_actions(b["action"]).reshape(B, 1)
        with torch.no_grad():
            tgt = torch_target(mode, b, q(*t), q(*tn), q(*nx), 0.9).reshape(B, 1)
        compute_weighted_value_loss(y, tgt, b["weights"]).backward()

    f, r = timed([fused, reference], reps, windows)
    return dict(bench="naf_loss_fwd_bwd", mode=mode, B=B, n=n, fused_us=round(f * 1e3, 2),
                torch_us=round(r * 1e3, 2), speedup=round(r / f, 2))


def bench_head(B, n, reps, windows):
    g = torch.Generator(device="cuda").manual_seed(B * n)
    dp = torch.randn(B, n, device="cuda", generator=g).requires_grad_()
    nd = (torch.randn(B, n * (n - 1) // 2, device="cuda", generator=g).requires_grad_()
          if n > 1 else None)
    G = torch.randn(B, n, n, device="cuda", generator=g)

    def fused():
        naf.head(dp, nd).backward(G)

    def reference():  # state_q_functions.py FCQuadraticStateQFunction.forward, after the heads
        d = torch.exp(dp)
        if nd is None:
            mat = torch.unsqueeze(d ** 2, dim=2)
        else:
            tril = lower_triangular_matrix(d, nd)
            mat = torch.matmul(tril, torch.transpose(tril, 1, 2))
        mat.backward(G)

    f, r = timed([fused, reference], reps, windows)
    return dict(bench="naf_head_fwd_bwd", B=B, n=n, fused_us=round(f * 1e3, 2),
                torch_us=round(r * 1e3, 2), speedup=round(r / f, 2))


UPDATE_ARMS = (("fused", True, False), ("fused_graph", True, True),
               ("torch", False, False), ("torch_graph", False, True))


def update_agent(use_fused_loss, graph, obs=17, n=6, hidden=256, batch=256, fill=5000):
    """A DQN with FCQuadraticStateQFunction on a device PER holding ``fill`` transitions."""
    import numpy as np

    from pfrl_b200 import explorers
    from pfrl_b200.agents import DQN
    from pfrl_b200.q_functions import FCQuadraticStateQFunction
    from pfrl_b200.replay_buffers import PrioritizedReplayBuffer

    torch.manual_seed(0)
    space = types.SimpleNamespace(low=-np.ones(n, np.float32), high=np.ones(n, np.float32))
    q = FCQuadraticStateQFunction(obs, n, hidden, 2, space).cuda()
    rbuf = PrioritizedReplayBuffer(10 ** 5, num_steps=3, device=0, fused=True)
    agent = DQN(q, torch.optim.Adam(q.parameters(), lr=1e-4, capturable=True), rbuf, 0.99,
                explorers.Greedy(), gpu=0, replay_start_size=batch, minibatch_size=batch,
                target_update_interval=10 ** 9, cuda_graph=graph)
    agent.use_fused_loss = use_fused_loss
    rng = np.random.RandomState(0)
    s = rng.randn(fill + 1, obs).astype(np.float32)
    a = rng.uniform(-1, 1, size=(fill, n)).astype(np.float32)
    r = rng.randn(fill).astype(np.float32)
    for t in range(fill):
        done = t % 200 == 199
        rbuf.append(state=s[t], action=a[t], reward=float(r[t]), next_state=s[t + 1],
                    next_action=None, is_state_terminal=done)
        if done:
            rbuf.stop_current_episode()
    return agent


def one_update(agent):
    agent.replay_updater.update_if_necessary(agent.replay_updater.update_interval)


def bench_update(reps, windows):
    agents = [update_agent(f, g) for _, f, g in UPDATE_ARMS]
    times = timed([lambda ag=ag: one_update(ag) for ag in agents], reps, windows)
    return [dict(bench="naf_dqn_update", arm=name, obs=17, n=6, hidden="2x256", B=256,
                 replay="device PER, fused replay step", ms=round(t, 4))
            for (name, _, _), t in zip(UPDATE_ARMS, times)]


def count_launches(updates=20):
    """Kernel launches (cudaLaunchKernel and friends) and graph launches per update."""
    from torch.profiler import ProfilerActivity, profile

    out = []
    for name, fused, graph in UPDATE_ARMS:
        agent = update_agent(fused, graph, fill=2000)
        for _ in range(5):  # warm-up, and the capture of the graphed arms
            one_update(agent)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for _ in range(updates):
                one_update(agent)
            torch.cuda.synchronize()
        names = [e.name for e in prof.events()]
        kernels = sum(1 for x in names if x in ("cudaLaunchKernel", "cudaLaunchKernelExC",
                                                "cuLaunchKernel", "cuLaunchKernelEx"))
        graphs = sum(1 for x in names if x in ("cudaGraphLaunch", "cuGraphLaunch"))
        out.append(dict(bench="naf_dqn_update_launches", arm=name, kernel_launches=kernels / updates,
                        graph_launches=graphs / updates))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--count-launches", action="store_true",
                    help="only count the launches per update (run in a process of its own)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_naf.py measures on a CUDA device; none found")
    torch.backends.cuda.matmul.allow_tf32 = False
    if args.count_launches:
        for row in count_launches():
            print(json.dumps(row), flush=True)
        return
    print(json.dumps(dict(card=card(), torch=torch.__version__)), flush=True)
    for row in bench_update(max(args.reps // 4, 20), args.windows):
        print(json.dumps(row), flush=True)
    subprocess.run([sys.executable, os.path.abspath(__file__), "--count-launches"], check=True)
    for B in (32, 512, 4096):
        for n in (1, 6, 17):
            print(json.dumps(bench_head(B, n, args.reps, args.windows)), flush=True)
            for mode in naf.NAF_MODES:
                print(json.dumps(bench_loss(mode, B, n, args.reps, args.windows)), flush=True)


if __name__ == "__main__":
    main()
