from pfrl_b200.agents.a2c import A2C  # NOQA
from pfrl_b200.agents.al import AL  # NOQA
from pfrl_b200.agents.categorical_double_dqn import CategoricalDoubleDQN  # NOQA
from pfrl_b200.agents.categorical_dqn import CategoricalDQN  # NOQA
from pfrl_b200.agents.double_dqn import DoubleDQN  # NOQA
from pfrl_b200.agents.double_pal import DoublePAL  # NOQA
from pfrl_b200.agents.dpp import DPP  # NOQA
from pfrl_b200.agents.dqn import DQN  # NOQA
from pfrl_b200.agents.iqn import IQN  # NOQA
from pfrl_b200.agents.pal import PAL  # NOQA
from pfrl_b200.agents.ppo import PPO  # NOQA
from pfrl_b200.agents.soft_actor_critic import SoftActorCritic  # NOQA
from pfrl_b200.agents.td3 import DDPG, TD3  # NOQA
from pfrl_b200.agents import ddpg  # NOQA  (module path of the reference)
from pfrl_b200.agents.trpo import TRPO  # NOQA
from pfrl_b200.agents.acer import ACER  # NOQA
from pfrl_b200.agents.reinforce import REINFORCE  # NOQA
from pfrl_b200.agents.a3c import A3C  # NOQA
