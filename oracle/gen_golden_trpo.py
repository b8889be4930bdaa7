"""Seeded runs of the reference's TRPO on the CPU -> tests/golden/agent_trace_trpo_{gauss,softmax}.npz.

Two chain environments (oracle/gen_golden_losses.py's runner): a Gaussian
state-independent-covariance policy on the continuous chain and a softmax policy on
the discrete chain, with the observation normaliser, standardised advantages,
max_grad_norm and update_interval 64.  Recorded: initial and final parameters, the
actions and statistics at every step, and per update every line-search candidate's
gain improvement and KL and the accepted step size (read from the reference's own log
lines by a handler on its logger).

The line search is discontinuous, so the generator also stores the decision margin:
the smallest |improve| (absolute: the gains of standardised advantages are O(0.01 .. 1))
and the smallest |kl - max_kl| / max_kl over all candidates, and asserts both exceed
MIN_MARGIN.  tests/test_trpo_gpu.py measures how far every candidate's improvement and
KL on CUDA move from these values (fp32 rounding of the forwards, the CG and the
reductions, accumulated over the run) and requires that distance to stay below a
quarter of the stored margins, so that no decision can flip.

    python oracle/gen_golden_trpo.py tests/golden
"""
import logging
import os
import random
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle.gen_golden_losses import _module_attrs, _run_more_trace  # noqa: E402

TRPO_KINDS = ("gauss", "softmax")
TRPO_STEPS = 260
MIN_MARGIN = 1e-3


def make_trpo_agent(lib, kind, gpu=None, logger=None, **extra):
    import torch
    from torch import nn

    phi = lambda x: x.astype(np.float32, copy=False)  # noqa: E731
    if kind == "gauss":
        policy = nn.Sequential(nn.Linear(5, 32), nn.Tanh(), nn.Linear(32, 1),
                               lib.policies.GaussianHeadWithStateIndependentCovariance(
                                   action_size=1, var_type="diagonal",
                                   var_func=lambda x: torch.exp(2 * x), var_param_init=-0.5))
    else:
        policy = nn.Sequential(nn.Linear(5, 32), nn.Tanh(), nn.Linear(32, 2),
                               lib.policies.SoftmaxCategoricalHead())
    vf = nn.Sequential(nn.Linear(5, 32), nn.Tanh(), nn.Linear(32, 1))
    kw = dict(extra) if logger is None else dict(extra, logger=logger)
    return lib.agents.TRPO(
        policy, vf, torch.optim.Adam(vf.parameters(), lr=3e-3),
        obs_normalizer=lib.nn.EmpiricalNormalization(5, clip_threshold=5), gpu=gpu, gamma=0.95,
        lambd=0.9, phi=phi, entropy_coef=0.01, update_interval=64, max_kl=0.01, vf_epochs=2,
        vf_batch_size=16, standardize_advantages=True, line_search_max_backtrack=6,
        conjugate_gradient_max_iter=8, conjugate_gradient_damping=0.1, max_grad_norm=0.5, **kw)


class LineSearchLog(logging.Handler):
    """Per update: [(improve, kl), ...] and the accepted step size, from the log lines of
    trpo.py:649-693."""

    def __init__(self):
        super().__init__(logging.INFO)
        self.updates = []
        self._cur = None

    def emit(self, record):
        msg = record.getMessage()
        if msg.startswith("Line search iteration: "):
            i = int(msg.split()[3])
            step = float(msg.split()[-1])
            if i == 0:
                self._cur = dict(cands=[], step=0.0)
                self.updates.append(self._cur)
            self._cur["cands"].append([step, np.nan, np.nan])
        elif msg.startswith("Surrogate objective improve: "):
            self._cur["cands"][-1][1] = float(msg.split()[-1])
        elif msg.startswith("KL divergence: "):
            self._cur["cands"][-1][2] = float(msg.split()[-1])


def run(lib, kind, gpu=None, check=None, init=None):
    import torch

    log = logging.getLogger("b2rl.trpo_trace.%s" % kind)
    log.setLevel(logging.INFO)
    log.propagate = False
    handler = LineSearchLog()
    log.handlers = [handler]
    torch.manual_seed(3)
    agent = make_trpo_agent(lib, kind, gpu=gpu, logger=log)
    if init is not None:
        for name, mod in _module_attrs(agent):
            mod.load_state_dict({k: torch.tensor(init["init_%s__%s" % (name, k)])
                                 for k in mod.state_dict()})
    g = {}
    for name, mod in _module_attrs(agent):
        for k, v in mod.state_dict().items():
            g["init_%s__%s" % (name, k)] = v.detach().cpu().numpy().copy()
    np.random.seed(9)
    torch.manual_seed(9)
    random.seed(9)
    actions, stats = _run_more_trace(agent, "sac" if kind == "gauss" else "ppo", TRPO_STEPS,
                                     check=check)
    g.update(actions=actions, stats=stats,
             stat_names=np.array([n for n, _ in agent.get_statistics()]))
    for name, mod in _module_attrs(agent):
        for k, v in mod.state_dict().items():
            g["final_%s__%s" % (name, k)] = v.detach().cpu().numpy().copy()
    return agent, g, handler.updates


def line_search_arrays(updates, max_kl):
    """cands [U, C, 3] (step, improve, kl; NaN past the decision) and accepted [U]."""
    C = max(len(u["cands"]) for u in updates)
    cands = np.full((len(updates), C, 3), np.nan)
    accepted = np.zeros(len(updates))
    for j, u in enumerate(updates):
        cands[j, :len(u["cands"])] = u["cands"]
        last = u["cands"][-1]
        ok = np.isfinite(last[1]) and np.isfinite(last[2]) and last[1] >= 0 and last[2] <= max_kl
        accepted[j] = last[0] if ok else 0.0
    return cands, accepted


def margin(cands, stats_scale, max_kl):
    imp, kl = cands[..., 1], cands[..., 2]
    ok = np.isfinite(imp) & np.isfinite(kl)
    m_imp = float(np.min(np.abs(imp[ok]))) / stats_scale
    m_kl = float(np.min(np.abs(kl[ok] - max_kl))) / max_kl
    return m_imp, m_kl


def main(out_dir):
    from oracle.refimport import import_reference

    pfrl = import_reference()
    for kind in TRPO_KINDS:
        agent, g, updates = run(pfrl, kind)
        cands, accepted = line_search_arrays(updates, agent.max_kl)
        m_imp, m_kl = margin(cands, 1.0, agent.max_kl)
        print(kind, "updates", len(updates), "accepted", accepted.tolist(),
              "margin improve %.3g kl %.3g" % (m_imp, m_kl))
        assert len(updates) >= 4 and m_imp > MIN_MARGIN and m_kl > MIN_MARGIN, (m_imp, m_kl)
        g.update(ls_cands=cands, ls_accepted=accepted, margin=np.array([m_imp, m_kl]),
                 max_kl=np.float64(agent.max_kl))
        np.savez_compressed(os.path.join(out_dir, "agent_trace_trpo_%s.npz" % kind), **g)
        print("wrote agent_trace_trpo_%s.npz" % kind, dict(zip(g["stat_names"], g["stats"][-1])))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(HERE), "tests",
                                                             "golden"))
