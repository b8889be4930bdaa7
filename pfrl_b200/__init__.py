"""pfrl_b200 -- an H100-native (sm_90a) batched-RL hot path behind PFRL's
public surface.

Python/PyTorch host code mirrors the reference's class names and signatures
(`pfrl_b200.replay_buffers.PrioritizedReplayBuffer`, `pfrl_b200.agents.DQN`,
`pfrl_b200.experiments.train_agent_batch`, ...) and calls hand-written CUDA
through the C ABI of include/b2rl.h (libb2rl.so, loaded with ctypes).
"""
__version__ = "0.1.0"

# `import pfrl_b200 as pfrl` then `pfrl.agents.DQN`, `pfrl.replay_buffers...`:
# the sub-packages are attributes of the package, like pfrl/__init__.py:1-20.
# Nothing here touches CUDA; libb2rl.so is loaded on first use of a device class.
from pfrl_b200 import action_value  # NOQA
from pfrl_b200 import agent  # NOQA
from pfrl_b200 import agents  # NOQA
from pfrl_b200 import collections  # NOQA
from pfrl_b200 import distributions  # NOQA
from pfrl_b200 import env  # NOQA
from pfrl_b200 import envs  # NOQA
from pfrl_b200 import experiments  # NOQA
from pfrl_b200 import explorer  # NOQA
from pfrl_b200 import explorers  # NOQA
from pfrl_b200 import functions  # NOQA
from pfrl_b200 import initializers  # NOQA
from pfrl_b200 import nn  # NOQA
from pfrl_b200 import optimizers  # NOQA
from pfrl_b200 import policies  # NOQA
from pfrl_b200 import q_function  # NOQA
from pfrl_b200 import q_functions  # NOQA
from pfrl_b200 import replay_buffer  # NOQA
from pfrl_b200 import replay_buffers  # NOQA
from pfrl_b200 import utils  # NOQA
from pfrl_b200 import wrappers  # NOQA
