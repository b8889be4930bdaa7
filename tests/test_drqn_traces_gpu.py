"""GPU: recurrent DQN / DoubleDQN on cuda:0 replay the seeded runs of the REAL reference
(tests/golden/agent_trace_drqn_*.npz, written by oracle/gen_golden_drqn.py on the CPU):
actions at every step and the sampled episodes and window starts exactly; statistics and
final parameters within the bounds tests/test_agent_traces_gpu.py uses for its
uniform-replay agents.  With the device EpisodicReplayBuffer (k_seq_gather, HBM state ring,
fused TD loss over the packed rows) and with the host buffer."""
import numpy as np
import pytest
import torch

from oracle.gen_golden_drqn import DRQN_KINDS
from test_drqn_traces_cpu import check_samples, replay

pytestmark = pytest.mark.gpu

RTOL, ATOL = 2e-3, 2e-4  # fp32 GEMM rounding, cuBLAS / cuDNN vs the CPU (test_agent_traces_gpu.py)


@pytest.mark.parametrize("buffer", ["device", "host"])
@pytest.mark.parametrize("kind", list(DRQN_KINDS))
def test_drqn_reproduces_the_reference_run_on_cuda(kind, buffer):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    g, q, stats, log = replay(kind, buffer, gpu=0)
    assert next(q.parameters()).is_cuda
    check_samples(g, log)
    assert np.array_equal(stats[:, 2:], g["stats"][:, 2:])
    live = ~np.isnan(g["stats"][:, 0])
    np.testing.assert_allclose(stats[live, :2], g["stats"][live, :2], rtol=RTOL, atol=ATOL)
    worst = 0.0
    for k, v in q.state_dict().items():
        worst = max(worst, float(np.abs(v.cpu().numpy() - g["final_" + k]).max()))
        np.testing.assert_allclose(v.cpu().numpy(), g["final_" + k], rtol=RTOL, atol=ATOL,
                                   err_msg=k)
    print("\n[drqn trace %s/%s on cuda] max |param diff| %.3g" % (kind, buffer, worst))
