"""GPU: recurrent PPO on cuda:0 replays the seeded runs of the REAL reference
(tests/golden/agent_trace_ppo_recurrent_*.npz, written by oracle/gen_golden_recurrent_ppo.py
on the CPU) through k_rollout_seq_gather, the fused GAE and the fused PPO loss.  Random
numbers are injected as in tests/test_agent_traces_gpu.py: the policy's draws are made on
the CPU generator, as the reference made them, and moved to the device.  Every minibatch's
schedule must be identical; actions equal (discrete) or within PPO's GPU bounds
(Gaussian); statistics and final parameters within PPO's GPU bounds there."""
import pytest
import torch

from oracle.gen_golden_recurrent_ppo import RPPO_KINDS
from test_agent_traces_gpu import TOL, host_rng
from test_recurrent_ppo_traces_cpu import check_run, replay

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("use_fused", [True, False], ids=["kernel", "torch"])
@pytest.mark.parametrize("kind", list(RPPO_KINDS))
def test_recurrent_ppo_reproduces_the_reference_run_on_cuda(kind, use_fused):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    rtol, atol = TOL["ppo"]
    with host_rng():
        g, model, stats, schedule = replay(kind, gpu=0, rtol=rtol, atol=atol,
                                           use_fused=use_fused)
    assert next(model.parameters()).is_cuda
    check_run(g, model, stats, schedule, rtol, atol)
