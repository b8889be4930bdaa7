"""Q-function heads for vector observations
(pfrl/q_functions/state_q_functions.py)."""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from pfrl_b200.action_value import (
    DiscreteActionValue, DistributionalDiscreteActionValue, QuadraticActionValue,
)
from pfrl_b200.functions.lower_triangular_matrix import lower_triangular_matrix
from pfrl_b200.initializers import init_chainer_default
from pfrl_b200.nn.mlp import MLP
from pfrl_b200.q_function import StateQFunction


def scale_by_tanh(x, low, high):
    scale = (high - low) / 2
    mean = (high + low) / 2
    return torch.tanh(x) * scale + mean


class SingleModelStateQFunctionWithDiscreteAction(nn.Module, StateQFunction):
    """Wrap a module whose output is [batch, n_actions] Q-values."""

    def __init__(self, model):
        super().__init__()
        self.model = model

    def forward(self, x):
        return DiscreteActionValue(self.model(x))


class FCStateQFunctionWithDiscreteAction(SingleModelStateQFunctionWithDiscreteAction):
    """MLP Q-function: ndim_obs -> hidden^layers -> n_actions."""

    def __init__(self, ndim_obs, n_actions, n_hidden_channels, n_hidden_layers,
                 nonlinearity=F.relu, last_wscale=1.0):
        super().__init__(model=MLP(
            in_size=ndim_obs, out_size=n_actions,
            hidden_sizes=[n_hidden_channels] * n_hidden_layers, nonlinearity=nonlinearity,
            last_wscale=last_wscale))


class DistributionalSingleModelStateQFunctionWithDiscreteAction(nn.Module, StateQFunction):
    """Wrap a module producing [batch, n_actions, n_atoms] probabilities."""

    def __init__(self, model, z_values):
        super().__init__()
        self.model = model
        self.register_buffer("z_values", z_values)

    def forward(self, x):
        return DistributionalDiscreteActionValue(self.model(x), self.z_values)


class DistributionalFCStateQFunctionWithDiscreteAction(
        DistributionalSingleModelStateQFunctionWithDiscreteAction):
    """C51 MLP Q-function over ``n_atoms`` atoms in [v_min, v_max]."""

    def __init__(self, ndim_obs, n_actions, n_atoms, v_min, v_max, n_hidden_channels,
                 n_hidden_layers, nonlinearity=F.relu, last_wscale=1.0):
        assert n_atoms >= 2
        assert v_min < v_max
        # numpy linspace (fp64 then cast), as in the reference (state_q_functions.py:128)
        z_values = torch.from_numpy(np.linspace(v_min, v_max, num=n_atoms, dtype=np.float32))

        class _Head(nn.Module):
            def forward(self, h):
                return F.softmax(h.reshape(-1, n_actions, n_atoms), dim=2)

        model = nn.Sequential(
            MLP(in_size=ndim_obs, out_size=n_actions * n_atoms,
                hidden_sizes=[n_hidden_channels] * n_hidden_layers, nonlinearity=nonlinearity,
                last_wscale=last_wscale),
            _Head())
        super().__init__(model=model, z_values=z_values)


class FCQuadraticStateQFunction(nn.Module, StateQFunction):
    """NAF Q-function for continuous actions (arXiv:1603.00748;
    pfrl/q_functions/state_q_functions.py FCQuadraticStateQFunction): ReLU hidden layers, then
    linear heads for V, mu (scaled into the action box by tanh when ``scale_mu``) and the
    diagonal and lower part of L, with P = L L^T.  Same parameters and ``state_dict`` keys as
    the reference.

    The tanh scale and mean and the action bounds are non-persistent buffers: they follow the
    module to its device once instead of being copied from the host on every forward.  On CUDA
    with fp32 parameters, P is built by one kernel (ops.naf.head); elsewhere by the
    reference's torch formulation."""

    def __init__(self, n_input_channels, n_dim_action, n_hidden_channels, n_hidden_layers,
                 action_space, scale_mu=True):
        self.n_input_channels = n_input_channels
        self.n_hidden_layers = n_hidden_layers
        self.n_hidden_channels = n_hidden_channels
        self.n_dim_action = n_dim_action
        assert action_space is not None
        self.scale_mu = scale_mu
        self.action_space = action_space
        super().__init__()
        hidden_layers = nn.ModuleList()
        assert n_hidden_layers >= 1
        hidden_layers.append(init_chainer_default(nn.Linear(n_input_channels, n_hidden_channels)))
        for _ in range(n_hidden_layers - 1):
            hidden_layers.append(
                init_chainer_default(nn.Linear(n_hidden_channels, n_hidden_channels)))
        self.hidden_layers = hidden_layers

        self.v = init_chainer_default(nn.Linear(n_hidden_channels, 1))
        self.mu = init_chainer_default(nn.Linear(n_hidden_channels, n_dim_action))
        self.mat_diag = init_chainer_default(nn.Linear(n_hidden_channels, n_dim_action))
        non_diag_size = n_dim_action * (n_dim_action - 1) // 2
        if non_diag_size > 0:
            self.mat_non_diag = init_chainer_default(nn.Linear(n_hidden_channels, non_diag_size))

        high, low = action_space.high, action_space.low
        # scale_by_tanh's numpy arithmetic, as the reference does it per forward
        self.register_buffer("mu_scale", torch.from_numpy(np.asarray((high - low) / 2))[None],
                             persistent=False)
        self.register_buffer("mu_mean", torch.from_numpy(np.asarray((high + low) / 2))[None],
                             persistent=False)
        self.register_buffer("min_action", torch.as_tensor(low).float(), persistent=False)
        self.register_buffer("max_action", torch.as_tensor(high).float(), persistent=False)

    def forward(self, state):
        h = state
        for layer in self.hidden_layers:
            h = F.relu(layer(h))
        v = self.v(h)
        mu = self.mu(h)
        if self.scale_mu:
            mu = torch.tanh(mu) * self.mu_scale + self.mu_mean
        diag_pre = self.mat_diag(h)
        non_diag = self.mat_non_diag(h) if hasattr(self, "mat_non_diag") else None
        if diag_pre.is_cuda and diag_pre.dtype == torch.float32:
            from pfrl_b200.ops import naf

            mat = naf.head(diag_pre, non_diag)
        else:
            mat_diag = torch.exp(diag_pre)
            if non_diag is not None:
                tril = lower_triangular_matrix(mat_diag, non_diag)
                mat = torch.matmul(tril, torch.transpose(tril, 1, 2))
            else:
                mat = torch.unsqueeze(mat_diag ** 2, dim=2)
        return QuadraticActionValue(mu, mat, v, min_action=self.min_action,
                                    max_action=self.max_action)


class DiscreteActionValueHead(nn.Module):
    def forward(self, q_values):
        return DiscreteActionValue(q_values)
