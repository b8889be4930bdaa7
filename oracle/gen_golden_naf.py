"""Golden vectors for NAF (FCQuadraticStateQFunction, QuadraticActionValue,
lower_triangular_matrix) and the DQN-family agents on it, produced by the REAL reference on
CPU (TEST INFRASTRUCTURE ONLY).

    python -m oracle.gen_golden_naf

writes tests/golden/naf_values.npz (the Q-function's outputs and every QuadraticActionValue
member at several action sizes, with scale_mu on and off, bounds none / scalar / array and mu
planted outside the box), tests/golden/naf_losses.npz (each agent's _compute_loss on fixed
batches, as oracle/gen_golden_advantage.py:advantage_losses) and
tests/golden/agent_trace_naf_<kind>.npz (seeded runs of the six agents with 3-step prioritised
replay and AdditiveOU exploration on two continuous chain environments, as
oracle/gen_golden_advantage.py:adv_agent_traces)."""
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

OUT = os.path.join(ROOT, "tests", "golden")

VALUE_N = (1, 2, 3, 6, 17)
VALUE_OBS, VALUE_B = 7, 9
# bounds handed to QuadraticActionValue directly
BOUND_KINDS = ("none", "scalar", "array", "lower_only")

NAF_AGENTS = {
    "dqn": ("dqn", "DQN", dict(batch_accumulator="sum")),
    "double_dqn": ("double_dqn", "DoubleDQN", dict(clip_delta=False)),
    "al": ("al", "AL", dict(alpha=1.0 / 3)),
    "pal": ("pal", "PAL", dict(alpha=0.99)),
    "double_pal": ("double_pal", "DoublePAL", dict(clip_delta=False, batch_accumulator="sum")),
    "dpp_greedy": ("dpp", "DPPGreedy", {}),
}
LOSS_OBS, LOSS_B, LOSS_N = 10, 48, (1, 3)


def action_space(n):
    """The attributes of a Box the Q-function reads: an asymmetric box, so the tanh scale and
    mean both matter."""
    low = np.linspace(-1.0, -0.25, n).astype(np.float32)
    high = np.linspace(0.5, 2.0, n).astype(np.float32)
    return types.SimpleNamespace(low=low, high=high, shape=(n,), dtype=np.dtype(np.float32))


def bounds(kind, n):
    if kind == "none":
        return None, None
    if kind == "scalar":
        return -0.5, 0.75
    if kind == "array":
        return action_space(n).low, action_space(n).high
    return action_space(n).low, None


def value_inputs(n):
    rng = np.random.RandomState(100 + n)
    return dict(state=rng.randn(VALUE_B, VALUE_OBS).astype(np.float32),
                actions=(rng.randn(VALUE_B, n) * 1.5).astype(np.float32),
                actions2=(rng.randn(VALUE_B, n) * 1.5).astype(np.float32),
                # mu planted around and outside every box above
                mu=(rng.randn(VALUE_B, n) * 2.0).astype(np.float32),
                diag=rng.randn(VALUE_B, n).astype(np.float32),
                non_diag=rng.randn(VALUE_B, n * (n - 1) // 2).astype(np.float32),
                mat_raw=rng.randn(VALUE_B, n, n).astype(np.float32),  # not symmetric
                v=rng.randn(VALUE_B, 1).astype(np.float32))


def action_value_members(av, inp):
    import torch

    a = torch.tensor(inp["actions"])
    a2 = torch.tensor(inp["actions2"])
    out = dict(greedy=av.greedy_actions, max=av.max, eval=av.evaluate_actions(a),
               adv=av.compute_advantage(a), dadv=av.compute_double_advantage(a, a2))
    sl = av[2:5]
    out.update(slice_greedy=sl.greedy_actions, slice_max=sl.max,
               slice_eval=sl.evaluate_actions(a[2:5]))
    return {k: v.detach().numpy().copy() for k, v in out.items()}


def naf_values(out_dir):
    import torch

    import pfrl
    from pfrl.functions.lower_triangular_matrix import lower_triangular_matrix

    g = {}
    for n in VALUE_N:
        inp = value_inputs(n)
        g.update({"n%d_%s" % (n, k): v for k, v in inp.items()})
        if n > 1:
            g["n%d_tril" % n] = lower_triangular_matrix(
                torch.tensor(inp["diag"]), torch.tensor(inp["non_diag"])).numpy()
        for scale_mu in (1, 0):
            torch.manual_seed(n)
            q = pfrl.q_functions.FCQuadraticStateQFunction(VALUE_OBS, n, 16, 2, action_space(n),
                                                           scale_mu=bool(scale_mu))
            name = "n%d_s%d" % (n, scale_mu)
            for k, v in q.state_dict().items():
                g["%s_param_%s" % (name, k)] = v.numpy().copy()
            av = q(torch.tensor(inp["state"]))
            g.update({"%s_%s" % (name, k): v.detach().numpy().copy()
                      for k, v in zip(("mu", "mat", "v"), av.params)})
            g.update({"%s_%s" % (name, k): v for k, v in action_value_members(av, inp).items()})
        for kind in BOUND_KINDS:
            lo, hi = bounds(kind, n)
            for which in ("tril", "raw"):
                mat = (torch.tensor(inp["mat_raw"]) if which == "raw" else
                       torch.tensor(inp["diag"]).exp().diag_embed())
                av = pfrl.action_value.QuadraticActionValue(
                    torch.tensor(inp["mu"]), mat, torch.tensor(inp["v"]), min_action=lo,
                    max_action=hi)
                g.update({"n%d_%s_%s_%s" % (n, kind, which, k): v
                          for k, v in action_value_members(av, inp).items()})
    np.savez_compressed(os.path.join(out_dir, "naf_values.npz"), **g)
    print("wrote naf_values.npz:", len(g), "arrays")


def _agent_class(lib, kind):
    from importlib import import_module

    module, name, kw = NAF_AGENTS[kind]
    return getattr(import_module("%s.agents.%s" % (lib.__name__, module)), name), dict(kw)


def loss_batch(n):
    rng = np.random.RandomState(31 + n)
    B = LOSS_B
    return dict(
        state=rng.randn(B, LOSS_OBS).astype(np.float32),
        next_state=rng.randn(B, LOSS_OBS).astype(np.float32),
        action=rng.uniform(-1.5, 2.5, size=(B, n)).astype(np.float32),
        reward=rng.choice([-1.0, 0.0, 1.0, 0.3], size=B).astype(np.float32),
        discount=(0.99 ** rng.randint(1, 4, size=B)).astype(np.float32),
        is_state_terminal=(rng.rand(B) < 0.2).astype(np.float32),
        weights=(rng.rand(B) + 0.2).astype(np.float32))


def make_loss_agent(lib, kind, n, gpu=None):
    import torch

    cls, kw = _agent_class(lib, kind)
    qf = lib.q_functions.FCQuadraticStateQFunction(LOSS_OBS, n, 32, 2, action_space(n))
    if gpu is not None:
        kw["gpu"] = gpu
    buf = (lib.replay_buffers.PrioritizedReplayBuffer(100) if lib.__name__ == "pfrl"
           else lib.replay_buffers.HostReplayBuffer(100))
    return cls(qf, torch.optim.SGD(qf.parameters(), lr=0.0), buf, 0.99, lib.explorers.Greedy(),
               replay_start_size=10, minibatch_size=8, **kw)


def naf_losses(out_dir):
    """End-to-end _compute_loss of each agent on a fixed batch, with and without weights, the
    target net perturbed away from the online net, at n = 1 and 3 (fp32, CPU)."""
    import torch

    import pfrl

    g = {}
    for n in LOSS_N:
        batch = loss_batch(n)
        g.update({"batch%d_%s" % (n, k): v for k, v in batch.items()})
        tb = {k: torch.tensor(v) for k, v in batch.items()}
        for kind in NAF_AGENTS:
            torch.manual_seed(7 + n)
            agent = make_loss_agent(pfrl, kind, n)
            with torch.no_grad():
                for p in agent.target_model.parameters():
                    p.add_(torch.randn_like(p) * 0.05)
            name = "%s_%d" % (kind, n)
            for which, mod in (("model", agent.model), ("target", agent.target_model)):
                for k, v in mod.state_dict().items():
                    g["%s_%s_%s" % (name, which, k)] = v.numpy().copy()
            for use_w in (1, 0):
                eb = dict(tb)
                if not use_w:
                    del eb["weights"]
                errs = []
                agent.model.zero_grad()
                loss = agent._compute_loss(eb, errors_out=errs)
                loss.backward()
                gn = torch.sqrt(sum((p.grad ** 2).sum() for p in agent.model.parameters()))
                g["%s_w%d_loss" % (name, use_w)] = np.float32(loss.item())
                g["%s_w%d_errors" % (name, use_w)] = np.asarray(errs, dtype=np.float32)
                g["%s_w%d_gradnorm" % (name, use_w)] = np.float64(gn.item())
    np.savez_compressed(os.path.join(out_dir, "naf_losses.npz"), **g)
    print("wrote naf_losses.npz:", len(g), "arrays")


# -------------------------------------------------------------------------------- traces
TRACE_OBS, TRACE_N = 5, 3


def make_trace_agent(lib, kind, rbuf, gpu=None):
    """Construction shared by the reference (lib = pfrl) and the rebuild (lib = pfrl_b200).
    The Q-function acts in a 3-dimensional box [-1, 1]^3; the chain reads component 0, so the
    off-diagonal entries of P take part in every update."""
    import torch

    space = types.SimpleNamespace(low=-np.ones(TRACE_N, np.float32),
                                  high=np.ones(TRACE_N, np.float32), shape=(TRACE_N,),
                                  dtype=np.dtype(np.float32))
    q = lib.q_functions.FCQuadraticStateQFunction(TRACE_OBS, TRACE_N, 32, 2, space)
    cls, kw = _agent_class(lib, kind)
    kw = {k: v for k, v in kw.items() if k == "alpha"}
    if gpu is not None:
        kw["gpu"] = gpu
    opt = torch.optim.Adam(q.parameters(), lr=1e-3, eps=1e-4)
    phi = lambda x: x.astype(np.float32, copy=False)  # noqa: E731
    return q, cls(q, opt, rbuf, 0.95, lib.explorers.AdditiveOU(sigma=0.5), replay_start_size=40,
                  minibatch_size=16, update_interval=1, target_update_interval=20, phi=phi, **kw)


def run_trace(agent, steps=260, n_envs=2, check=None):
    """oracle/gen_golden_losses.py:_run_trace on ChainEnv(continuous=True): the actions are
    float vectors."""
    from pfrl_b200.envs import ChainEnv

    envs = [ChainEnv(seed=i, continuous=True) for i in range(n_envs)]
    obs = [e.reset() for e in envs]
    actions, stats = [], []
    for t in range(steps):
        a = np.stack([np.asarray(x, dtype=np.float32).reshape(-1) for x in agent.batch_act(obs)])
        if check is not None:
            check(t, a)
        actions.append(a)
        nobs, r, d, info = zip(*[e.step(x) for e, x in zip(envs, a)])
        resets = [i["needs_reset"] for i in info]
        agent.batch_observe(list(nobs), list(r), list(d), resets)
        obs = [e.reset() if (dd or rr) else o for e, o, dd, rr in zip(envs, nobs, d, resets)]
        st = dict(agent.get_statistics())
        stats.append([st["average_q"], st["average_loss"], st["n_updates"], st["rlen"]])
    return np.asarray(actions), np.asarray(stats, dtype=np.float64)


def naf_traces(out_dir):
    import torch

    import pfrl
    from oracle.gen_golden_losses import TRACE_PER

    for kind in NAF_AGENTS:
        rbuf = pfrl.replay_buffers.PrioritizedReplayBuffer(150, **TRACE_PER)
        raw_update = rbuf.update_errors
        rbuf.update_errors = lambda errors, raw=raw_update: raw([float(e) for e in errors])
        torch.manual_seed(3)
        q, agent = make_trace_agent(pfrl, kind, rbuf)
        g = {"init_" + k: v.numpy().copy() for k, v in q.state_dict().items()}
        sampled, sample = [], rbuf.sample

        def recording_sample(n, sample=sample, rbuf=rbuf, sampled=sampled):
            out = sample(n)
            sampled.append(list(rbuf.memory.sampled_indices))
            return out

        rbuf.sample = recording_sample
        np.random.seed(9)
        torch.manual_seed(9)
        actions, stats = run_trace(agent)
        g.update(actions=actions, stats=stats, sampled=np.asarray(sampled, dtype=np.int64),
                 total=np.float64(rbuf.memory.priority_sums.sum()),
                 min=np.float64(rbuf.memory.priority_mins.min()),
                 max_priority=np.float64(rbuf.memory.max_priority), beta=np.float64(rbuf.beta))
        for k, v in q.state_dict().items():
            g["final_" + k] = v.numpy().copy()
        np.savez_compressed(os.path.join(out_dir, "agent_trace_naf_%s.npz" % kind), **g)
        print("wrote agent_trace_naf_%s.npz:" % kind, int(stats[-1][2]), "updates")


def main():
    from oracle.refimport import import_reference

    import_reference()
    os.makedirs(OUT, exist_ok=True)
    naf_values(OUT)
    naf_losses(OUT)
    naf_traces(OUT)


if __name__ == "__main__":
    main()
