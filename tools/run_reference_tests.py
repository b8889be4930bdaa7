"""Run the REFERENCE's own unit tests against this package.

Build-container tool (needs /root/reference; nothing here ships or runs on the
GPU box).  The name ``pfrl`` is aliased to ``pfrl_b200`` module by module, the
gym shim of oracle/gym_shim stands in for gym, and -- because there is no GPU
here -- the CUDA store behind the device replay buffers is replaced by
tests/fake_store.OracleBackedStore, so that the reference's replay-buffer tests
exercise the device buffers' real host logic.  Then pytest runs the reference's
test files unmodified from where they lie.

    python tools/run_reference_tests.py            # the default file list below
    python tools/run_reference_tests.py experiments_tests/test_evaluator.py -k batch

Files that test subsystems outside the rebuilt path (async training, persistent
buffers, ALE wrappers, ...) are not in the list.
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_TESTS = os.environ.get("PFRL_REFERENCE_ROOT", "/root/reference") + "/tests"

DEFAULT = [
    "test_agent.py", "test_action_value.py",
    "experiments_tests/test_train_agent_batch.py", "experiments_tests/test_train_agent.py",
    "experiments_tests/test_evaluator.py", "experiments_tests/test_hooks.py",
    "explorers_tests/test_additive_gaussian.py", "explorers_tests/test_additive_ou.py",
    "explorers_tests/test_boltzmann.py", "explorers_tests/test_epsilon_greedy.py",
    "nn_tests/test_branched.py", "nn_tests/test_empirical_normalization.py",
    "nn_tests/test_lmbda.py", "nn_tests/test_noisy_chain.py", "nn_tests/test_noisy_linear.py",
    "utils_tests/test_batch_states.py", "utils_tests/test_clip_l2_grad_norm.py",
    "utils_tests/test_contexts.py", "utils_tests/test_copy_param.py",
    "utils_tests/test_mode_of_distribution.py", "utils_tests/test_random.py",
    "utils_tests/test_random_seed.py", "wrappers_tests/test_vector_frame_stack.py",
    # envs_tests/test_vector_envs.py needs gym.make("CartPole-v0"): see tests/test_vector_envs_cpu.py
    "replay_buffers_test/test_replay_buffer.py", "collections_tests/test_random_access_queue.py",
    "collections_tests/test_prioritized.py",
    "agents_tests/test_dqn.py", "agents_tests/test_double_dqn.py",
    "agents_tests/test_categorical_dqn.py", "agents_tests/test_double_categorical_dqn.py",
    "agents_tests/test_iqn.py", "agents_tests/test_ppo.py", "agents_tests/test_a2c.py",
    "agents_tests/test_soft_actor_critic.py", "agents_tests/test_td3.py",
    "agents_tests/test_ddpg.py",
    "agents_tests/test_al.py", "agents_tests/test_pal.py", "agents_tests/test_double_pal.py",
    "agents_tests/test_dpp.py",
    # recurrent TRPO is out of scope: the non-recurrent classes only
    "agents_tests/test_trpo.py::TestHessianVectorProduct",
    "agents_tests/test_trpo.py::TestTRPONonRecurrent",
    "utils_tests/test_conjugate_gradient.py",
    "nn_tests/test_recurrent_sequential.py", "nn_tests/test_recurrent_branched.py",
    "utils_tests/test_recurrent.py",
    # ACER's function-level tests; _TestACER needs train_agent_async
    "agents_tests/test_acer.py::TestDegenerateDistribution",
    "agents_tests/test_acer.py::test_bias_correction_gaussian",
    "agents_tests/test_acer.py::test_bias_correction_softmax",
    "agents_tests/test_acer.py::test_compute_loss_with_kl_constraint_gaussian",
    "agents_tests/test_acer.py::test_compute_loss_with_kl_constraint_softmax",
    "agents_tests/test_reinforce.py",
]

PLUGIN = '''
import importlib, pkgutil, sys
from unittest import mock
sys.dont_write_bytecode = True
sys.path[:0] = [%(root)r, %(root)r + "/tests", %(root)r + "/oracle/gym_shim"]
import pfrl_b200
for m in pkgutil.walk_packages(pfrl_b200.__path__, "pfrl_b200."):
    if ".csrc" not in m.name:
        importlib.import_module(m.name)
sys.modules["pfrl"] = pfrl_b200
for name, mod in list(sys.modules.items()):
    if name.startswith("pfrl_b200."):
        sys.modules["pfrl." + name[len("pfrl_b200."):]] = mod

def _out_of_scope(module_name):
    """Names the reference has and this package does not (recurrent models,
    episodic buffers, other agents ...): importing them works, using them fails."""
    def getter(name):
        if name.startswith("__"):
            raise AttributeError(name)
        def init(self, *a, **k):
            raise NotImplementedError("%%s.%%s is out of scope of pfrl_b200" %% (module_name, name))
        return type(name, (), {"__init__": init, "_b2rl_stub": True})
    return getter

for name, mod in list(sys.modules.items()):
    if name.startswith("pfrl_b200") and not hasattr(mod, "__getattr__"):
        mod.__getattr__ = _out_of_scope(name)

from fake_store import OracleBackedStore
from fake_episodic_store import EpisodicOracleStore
mock.patch("pfrl_b200.replay_buffers.device_buffer.DeviceReplayStore", EpisodicOracleStore).start()
mock.patch("pfrl_b200.collections.prioritized.DeviceReplayStore", OracleBackedStore).start()
mock.patch("torch.cuda.current_device", return_value=0).start()

def pytest_configure(config):
    for m in ("gpu", "slow", "async_"):
        config.addinivalue_line("markers", m + ": reference marker")
'''


def main(argv):
    files = [a for a in argv if a.endswith(".py")] or DEFAULT
    extra = [a for a in argv if not a.endswith(".py")]
    work = os.path.join("/tmp", "b2rl_reference_tests")
    os.makedirs(work, exist_ok=True)
    with open(os.path.join(work, "b2rl_alias_plugin.py"), "w") as f:
        f.write(PLUGIN % {"root": ROOT})
    env = dict(os.environ, PYTHONPATH=work, PYTHONDONTWRITEBYTECODE="1")
    totals = {}
    for rel in files:
        cmd = [sys.executable, "-m", "pytest", "-p", "b2rl_alias_plugin", "-p", "no:cacheprovider",
               "--rootdir", work, "-c", "/dev/null", os.path.join(REF_TESTS, rel), "-q",
               "-m", "not gpu and not slow"] + extra
        try:
            out = subprocess.run(cmd, cwd=work, env=env, capture_output=True, text=True,
                                 timeout=int(os.environ.get("B2RL_FILE_TIMEOUT", "300"))).stdout
        except subprocess.TimeoutExpired:
            out = "TIMEOUT"
        tail = [ln for ln in out.strip().splitlines() if ln.strip()]
        summary = tail[-1] if tail else "(no output)"
        print("%-50s %s" % (rel, summary), flush=True)
        if "-v" in extra or os.environ.get("B2RL_SHOW_FAILURES"):
            print("\\n".join(ln for ln in tail if ln.startswith(("FAILED", "ERROR", "E "))))
        totals[rel] = summary
    return totals


if __name__ == "__main__":
    main(sys.argv[1:])
