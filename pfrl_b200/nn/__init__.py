from pfrl_b200.nn.atari_cnn import LargeAtariCNN, SmallAtariCNN  # NOQA
from pfrl_b200.nn.empirical_normalization import EmpiricalNormalization  # NOQA
from pfrl_b200.nn.mlp import MLP  # NOQA
from pfrl_b200.nn.noisy_chain import to_factorized_noisy  # NOQA
from pfrl_b200.nn.noisy_linear import FactorizedNoisyLinear  # NOQA
from pfrl_b200.nn.containers import BoundByTanh, Branched, ConcatObsAndAction, Lambda  # NOQA
from pfrl_b200.nn import bound_by_tanh, branched, concat_obs_and_action, lmbda  # NOQA  (module paths of the reference)
from pfrl_b200.nn.recurrent import Recurrent, RecurrentBranched, RecurrentSequential  # NOQA
from pfrl_b200.nn import recurrent  # NOQA
