from pfrl_b200.utils.batch_states import batch_states  # NOQA
from pfrl_b200.utils.clip_l2_grad_norm import clip_l2_grad_norm_  # NOQA
from pfrl_b200.utils.conjugate_gradient import conjugate_gradient  # NOQA
from pfrl_b200.utils.modes import evaluating  # NOQA
from pfrl_b200.utils.copy_param import synchronize_parameters  # NOQA
from pfrl_b200.utils.random import sample_n_k  # NOQA
from pfrl_b200.utils.random_seed import set_random_seed  # NOQA
from pfrl_b200.utils.mode_of_distribution import mode_of_distribution  # NOQA
from pfrl_b200.utils import copy_param  # NOQA  (the module, as in the reference)
from pfrl_b200.utils import phi  # NOQA  (ScaleU8 / Identity / AsFloat32: phi objects the gather kernel understands)
from pfrl_b200.utils import recurrent  # NOQA  (the module, as in the reference)
