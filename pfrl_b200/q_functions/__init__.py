from pfrl_b200.q_functions.dueling_dqn import DistributionalDuelingDQN, DuelingDQN  # NOQA
from pfrl_b200.q_functions.state_q_functions import (  # NOQA
    DiscreteActionValueHead,
    DistributionalFCStateQFunctionWithDiscreteAction,
    DistributionalSingleModelStateQFunctionWithDiscreteAction,
    FCQuadraticStateQFunction,
    FCStateQFunctionWithDiscreteAction,
    SingleModelStateQFunctionWithDiscreteAction,
)
