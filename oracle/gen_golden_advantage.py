"""Golden vectors for the advantage-learning and DPP agents (AL, PAL, DoublePAL, DPP, DPPL,
DPPGreedy), produced by the REAL reference on CPU (TEST INFRASTRUCTURE ONLY).

    python -m oracle.gen_golden_advantage

writes tests/golden/agent_trace_<kind>.npz for every kind of ADV_TRACE_KINDS (seeded runs
with 3-step prioritised replay, as oracle/gen_golden_losses.py:agent_traces) and
tests/golden/advantage_losses.npz (each agent's _compute_loss on fixed batches, as
oracle/gen_golden_losses.py:agent_losses)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.gen_golden_losses import TRACE_PER, _run_trace  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")

# kind -> (module, class, keyword arguments); eta != 1 so that the fp32 rounding of eta counts
ADV_AGENTS = {
    "al": ("al", "AL", {}),
    "pal": ("pal", "PAL", {}),
    "double_pal": ("double_pal", "DoublePAL", {}),
    "dpp": ("dpp", "DPP", dict(eta=2.0)),
    "dppl": ("dpp", "DPPL", dict(eta=2.0)),
    "dpp_greedy": ("dpp", "DPPGreedy", {}),
}
# the noisy DoublePAL run checks the order of the four network forwards (noise stream)
ADV_TRACE_KINDS = tuple(ADV_AGENTS) + ("double_pal_noisy",)


def _agent_class(lib, kind):
    from importlib import import_module

    module, name, kw = ADV_AGENTS[kind]
    return getattr(import_module("%s.agents.%s" % (lib.__name__, module)), name), kw


def _make_adv_trace_agent(lib, kind, rbuf):
    """Construction shared by the reference (lib = pfrl) and the rebuild (lib = pfrl_b200),
    as oracle/gen_golden_losses.py:_make_trace_agent."""
    import torch

    phi = lambda x: x.astype(np.float32, copy=False)  # noqa: E731
    q = lib.q_functions.FCStateQFunctionWithDiscreteAction(5, 2, 32, 2)
    if kind == "double_pal_noisy":
        lib.nn.to_factorized_noisy(q, sigma_scale=0.5)
        explorer = lib.explorers.Greedy()
        cls, kw = _agent_class(lib, "double_pal")
    else:
        explorer = lib.explorers.LinearDecayEpsilonGreedy(1.0, 0.1, 150,
                                                          lambda: np.random.randint(2))
        cls, kw = _agent_class(lib, kind)
    opt = torch.optim.Adam(q.parameters(), lr=1e-3, eps=1e-4)
    return q, cls(q, opt, rbuf, 0.95, explorer, replay_start_size=40, minibatch_size=16,
                  update_interval=1, target_update_interval=20, phi=phi, **kw)


def adv_agent_traces(out_dir):
    import torch

    import pfrl

    for kind in ADV_TRACE_KINDS:
        rbuf = pfrl.replay_buffers.PrioritizedReplayBuffer(150, **TRACE_PER)
        raw_update = rbuf.update_errors
        # TD errors enter update_errors as Python floats (see gen_golden_losses.agent_traces)
        rbuf.update_errors = lambda errors, raw=raw_update: raw([float(e) for e in errors])
        torch.manual_seed(3)
        q, agent = _make_adv_trace_agent(pfrl, kind, rbuf)
        g = {"init_" + k: v.numpy().copy() for k, v in q.state_dict().items()}
        np.random.seed(9)
        torch.manual_seed(9)
        actions, stats = _run_trace(agent, rbuf)
        g.update(actions=actions, stats=stats,
                 total=np.float64(rbuf.memory.priority_sums.sum()),
                 min=np.float64(rbuf.memory.priority_mins.min()),
                 max_priority=np.float64(rbuf.memory.max_priority), beta=np.float64(rbuf.beta))
        for k, v in q.state_dict().items():
            g["final_" + k] = v.numpy().copy()
        np.savez_compressed(os.path.join(out_dir, "agent_trace_%s.npz" % kind), **g)
        print("wrote agent_trace_%s.npz:" % kind, int(stats[-1][2]), "updates")


# per agent: (alpha / eta / loss keywords) of the fixed-batch cases
LOSS_CASES = {
    "al": dict(alpha=1.0 / 3),
    "pal": dict(alpha=0.99),
    "double_pal": dict(clip_delta=False, batch_accumulator="sum"),
    "dpp": dict(eta=2.0),
    "dppl": dict(eta=0.5, clip_delta=False),
    "dpp_greedy": dict(batch_accumulator="sum"),
}
LOSS_OBS, LOSS_B, LOSS_NA = 10, 48, (4, 18)


def loss_batch(nA):
    rng = np.random.RandomState(11 + nA)
    B = LOSS_B
    return dict(
        state=rng.randn(B, LOSS_OBS).astype(np.float32),
        next_state=rng.randn(B, LOSS_OBS).astype(np.float32),
        action=rng.randint(0, nA, size=B).astype(np.int64),
        reward=rng.choice([-1.0, 0.0, 1.0, 0.3], size=B).astype(np.float32),
        discount=(0.99 ** rng.randint(1, 4, size=B)).astype(np.float32),
        is_state_terminal=(rng.rand(B) < 0.2).astype(np.float32),
        weights=(rng.rand(B) + 0.2).astype(np.float32))


def make_loss_agent(lib, kind, nA, gpu=None):
    import torch

    cls, _ = _agent_class(lib, kind)
    qf = lib.q_functions.FCStateQFunctionWithDiscreteAction(LOSS_OBS, nA, 32, 2)
    kw = dict(LOSS_CASES[kind])
    if gpu is not None:
        kw["gpu"] = gpu
    buf = (lib.replay_buffers.PrioritizedReplayBuffer(100) if lib.__name__ == "pfrl"
           else lib.replay_buffers.HostReplayBuffer(100))
    return cls(qf, torch.optim.SGD(qf.parameters(), lr=0.0), buf, 0.99, lib.explorers.Greedy(),
               replay_start_size=10, minibatch_size=8, **kw)


def advantage_losses(out_dir):
    """End-to-end _compute_loss of each agent on a fixed batch, with and without weights, the
    target net perturbed away from the online net, at nA = 4 and 18 (fp32, CPU)."""
    import torch

    import pfrl

    g = {}
    for nA in LOSS_NA:
        batch = loss_batch(nA)
        g.update({"batch%d_%s" % (nA, k): v for k, v in batch.items()})
        tb = {k: torch.tensor(v) for k, v in batch.items()}
        for kind in ADV_AGENTS:
            torch.manual_seed(7 + nA)
            agent = make_loss_agent(pfrl, kind, nA)
            with torch.no_grad():
                for p in agent.target_model.parameters():
                    p.add_(torch.randn_like(p) * 0.05)
            name = "%s_%d" % (kind, nA)
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
                g["%s_w%d_loss" % (name, use_w)] = loss.detach().numpy()
                g["%s_w%d_errors" % (name, use_w)] = np.asarray(errs, dtype=np.float32)
                g["%s_w%d_gradnorm" % (name, use_w)] = np.float32(
                    torch.sqrt(sum((p.grad ** 2).sum() for p in agent.model.parameters())))
    np.savez_compressed(os.path.join(out_dir, "advantage_losses.npz"), **g)
    print("wrote advantage_losses.npz with", len(g), "arrays")


def main():
    from oracle.refimport import import_reference

    import_reference()
    print("numpy", np.__version__)
    advantage_losses(OUT)
    adv_agent_traces(OUT)


if __name__ == "__main__":
    main()
