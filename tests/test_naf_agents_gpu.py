"""GPU: the DQN-family agents with a NAF Q-function on CUDA.

* the fixed-batch losses of tests/golden/naf_losses.npz through the fused path and through
  ``use_fused_loss = False``;
* training on the device PER with the fused replay step and with separate launches: same
  indices, trees and parameters, bit for bit;
* ``cuda_graph=True`` against eager, update and acting;
* the six seeded reference runs (tests/golden/agent_trace_naf_<kind>.npz) on cuda:0, within the
  tolerances tests/test_agent_traces_gpu.py allows for fp32 GEMM rounding differences
  (cuBLAS against the CPU the fixtures were made on) over a few hundred Adam steps."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_naf_cpu import check_fixed_batch_losses, replay_trace  # noqa: E402

from oracle.gen_golden_naf import LOSS_N, NAF_AGENTS, action_space  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture
def no_tf32(monkeypatch):
    """fp32 GEMMs in full precision for this test only."""
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)


@pytest.mark.parametrize("kind", list(NAF_AGENTS))
def test_agent_on_cuda_reproduces_the_reference_run(kind, no_tf32):
    """Prioritised sampling reads fp32 TD errors, and cuBLAS rounds GEMMs differently from the
    CPU the fixture was made on, so a draw near a leaf boundary can pick the neighbouring leaf
    (tests/test_agent_traces_gpu.py).  Up to the first such update the run must match the
    reference step for step; a run without one must match to the end (parameters and trees)."""
    diverged, worst = replay_trace(kind, device=0, rtol=2e-3, atol=2e-4)
    print("\n[naf trace %s on cuda] first update with other indices: %s, max |action diff| "
          "before it %.3g" % (kind, diverged, worst))


@pytest.mark.parametrize("n", LOSS_N)
@pytest.mark.parametrize("kind", list(NAF_AGENTS))
def test_fused_fixed_batch_losses_match_reference_and_torch_path(kind, n, no_tf32):
    agent, fused = check_fixed_batch_losses(kind, n, "cuda", rtol=1e-4)
    assert agent.use_fused_loss
    _, torch_path = check_fixed_batch_losses(kind, n, "cuda", rtol=1e-4, use_fused_loss=False)
    for use_w in (1, 0):
        np.testing.assert_allclose(fused[use_w][0], torch_path[use_w][0], rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(fused[use_w][1], torch_path[use_w][1], rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(fused[use_w][2], torch_path[use_w][2], rtol=1e-5)


def _agent_class(kind):
    from importlib import import_module

    module, name, _ = NAF_AGENTS[kind]
    return getattr(import_module("pfrl_b200.agents.%s" % module), name)


def _train(kind, fused_step=True, graph=False, steps=80, n=3):
    """A seeded run on 4 device environments with 3-step prioritised replay; returns the
    sampled indices of every update, the parameters, the statistics, the buffer and the
    actions taken."""
    from pfrl_b200 import explorers, q_functions
    from pfrl_b200.envs import SyntheticContinuousVectorEnv
    from pfrl_b200.replay_buffers import PrioritizedReplayBuffer
    from pfrl_b200.utils import set_random_seed
    from pfrl_b200.utils.phi import Identity

    set_random_seed(3)
    q = q_functions.FCQuadraticStateQFunction(12, n, 64, 2, action_space(n))
    rbuf = PrioritizedReplayBuffer(4096, alpha=0.6, beta0=0.4, betasteps=200, num_steps=3,
                                   fused=fused_step)
    kw = {k: v for k, v in NAF_AGENTS[kind][2].items() if k == "alpha"}
    agent = _agent_class(kind)(
        q.cuda(), torch.optim.Adam(q.parameters(), lr=1e-3, capturable=True), rbuf, 0.99,
        explorers.Greedy(), gpu=0, replay_start_size=64, minibatch_size=32,
        target_update_interval=40, phi=Identity(), cuda_graph=graph, **kw)
    indices, actions = [], []
    sample = rbuf.sample

    def recording_sample(k):
        exps = sample(k)
        indices.append(exps.index.clone())
        return exps

    rbuf.sample = recording_sample
    env = SyntheticContinuousVectorEnv(4, 12, n, device="cuda", seed=5, mean_episode_len=20)
    obs = env.reset()
    for _ in range(steps):
        a = agent.batch_act(obs)
        actions.append(np.asarray(a).copy())
        obs, r, d, info = env.step(a)
        agent.batch_observe(obs, r, d, np.zeros(4, dtype=bool))
        obs = env.reset(np.logical_not(d))
    assert agent.optim_t > 200
    assert (agent._graph is not None and agent._graph.graph is not None) == graph
    params = [p.detach().clone() for p in agent.model.parameters()]
    return indices, params, dict(agent.get_statistics()), rbuf, actions


@pytest.mark.parametrize("kind", ["dqn", "double_pal"])
def test_fused_replay_step_matches_separate_launches(kind):
    (ia, pa, sa, ba, _), (ib, pb, sb, bb, _) = [_train(kind, fused_step=f) for f in (True, False)]
    assert len(ia) == len(ib) and all(torch.equal(x, y) for x, y in zip(ia, ib))
    assert all(torch.equal(x, y) for x, y in zip(pa, pb))
    ba._flush()
    bb._flush()
    fa, fb = ba.store.info(), bb.store.info()
    for k in ("total", "min", "max_priority", "napp", "npop"):
        assert fa[k] == fb[k], k
    assert np.array_equal(ba.store.read_priorities(), bb.store.read_priorities())
    assert sa["average_loss"] == sb["average_loss"] and np.isfinite(sa["average_loss"])


@pytest.mark.parametrize("kind", list(NAF_AGENTS))
def test_update_and_acting_as_cuda_graph_match_eager(kind):
    """cuda_graph=True replays the forwards, the NAF head and loss kernels, backward and Adam
    as one graph, and the acting forward as another: bit-equal to eager."""
    ie, eager, se, _, ae = _train(kind, graph=False)
    ig, graphed, sg, _, ag = _train(kind, graph=True)
    assert all(torch.equal(x, y) for x, y in zip(ie, ig))
    assert all(np.array_equal(x, y) for x, y in zip(ae, ag))
    assert all(torch.equal(a, b) for a, b in zip(eager, graphed))
    assert se["average_loss"] == sg["average_loss"]


def test_naf_update_does_not_synchronise():
    """One fused NAF update has no host round trip (sync debug mode "error")."""
    from test_naf_cpu import LOSSES

    from oracle.gen_golden_naf import make_loss_agent

    import pfrl_b200

    agent = make_loss_agent(pfrl_b200, "double_pal", 3, gpu=0)
    prefix = "batch3_"
    eb = {k[len(prefix):]: torch.tensor(LOSSES[k]).cuda() for k in LOSSES.files
          if k.startswith(prefix)}
    agent._learn(eb, want_errors=True)  # warm-up
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        agent._learn(eb, want_errors=True)
    finally:
        torch.cuda.set_sync_debug_mode(0)


@pytest.mark.parametrize("kind", list(NAF_AGENTS))
def test_fp64_model_keeps_the_reference_formulation(kind):
    """A NAF model in fp64 is not rounded through the fp32 kernel: its loss and gradients
    equal those of use_fused_loss = False, bit for bit."""
    from oracle.gen_golden_naf import make_loss_agent
    from test_naf_cpu import LOSSES

    import pfrl_b200

    # n = 1: with n > 1 the reference's lower_triangular_matrix is fp32 only
    eb = {k[len("batch1_"):]: torch.tensor(LOSSES[k]).cuda().double()
          if LOSSES[k].dtype == np.float32 else torch.tensor(LOSSES[k]).cuda()
          for k in LOSSES.files if k.startswith("batch1_")}
    out = []
    for fused in (True, False):
        torch.manual_seed(0)
        agent = make_loss_agent(pfrl_b200, kind, 1, gpu=0)
        agent.model.double()
        agent.target_model.double()
        agent.use_fused_loss = fused
        loss, delta = agent._compute_loss(eb, want_errors=True)
        loss.backward()
        assert loss.dtype == torch.float64
        out.append([loss.detach(), delta.detach()] + [p.grad for p in agent.model.parameters()])
    assert all(torch.equal(a, b) for a, b in zip(*out))
