"""Implicit Quantile Networks (arXiv:1806.06923) on the device replay path.

Reference: pfrl/agents/iqn.py (cosine embedding :14-66, ImplicitQuantileQFunction
:96-136, loss :176-250, IQN :253-433).  The [B, N, N'] quantile-Huber loss,
its per-sample priority error and the weighted reduction are one fused CUDA
kernel pair (csrc/losses.cu) on the GPU.
"""
import numpy as np
import torch
from torch import nn

from pfrl_b200.action_value import QuantileDiscreteActionValue
from pfrl_b200.agents import dqn
from pfrl_b200.ops import losses as fused


def cosine_basis_functions(x, n_basis_functions=64):
    """cos(pi * i * x) for i = 1..n: embedding of quantile thresholds."""
    i_pi = torch.arange(1, n_basis_functions + 1, dtype=torch.float, device=x.device) * np.pi
    return torch.cos(x[..., None] * i_pi)


class CosineBasisLinear(nn.Module):
    def __init__(self, n_basis_functions, out_size):
        super().__init__()
        self.linear = nn.Linear(n_basis_functions, out_size)
        self.n_basis_functions = n_basis_functions
        self.out_size = out_size

    def forward(self, x):
        h = cosine_basis_functions(x, self.n_basis_functions)
        out = self.linear(h.reshape(-1, self.n_basis_functions))
        return out.reshape(*x.shape, self.out_size)


class ImplicitQuantileQFunction(nn.Module):
    """psi: obs -> hidden; phi: taus -> hidden per tau; f: hidden -> actions.
    Calling the module returns a function of the quantile thresholds."""

    def __init__(self, psi, phi, f):
        super().__init__()
        self.psi = psi
        self.phi = phi
        self.f = f

    def forward(self, x):
        psi_x = self.psi(x)
        assert psi_x.ndim == 2

        def evaluate_with_quantile_thresholds(taus):
            batch_size, hidden = psi_x.shape
            n_taus = taus.shape[1]
            h = (psi_x.unsqueeze(1) * self.phi(taus)).reshape(-1, hidden)
            h = self.f(h)
            return QuantileDiscreteActionValue(h.reshape(batch_size, n_taus, h.shape[-1]))

        return evaluate_with_quantile_thresholds


def compute_eltwise_huber_quantile_loss(y, t, taus):
    """|tau - 1[t < y]| * Huber(y, t) broadcast to [B, N, N'] (iqn.py:176-208)."""
    assert y.shape == taus.shape
    y, t, taus = torch.broadcast_tensors(y.unsqueeze(2), t.unsqueeze(1), taus.unsqueeze(2))
    indicator = (t < y).float()
    return torch.abs(taus - indicator) * nn.functional.smooth_l1_loss(y, t, reduction="none")


def compute_value_loss(eltwise_loss, batch_accumulator="mean"):
    assert batch_accumulator in ("mean", "sum") and eltwise_loss.ndim == 3
    if batch_accumulator == "sum":
        return eltwise_loss.mean(2).sum()
    return eltwise_loss.mean((0, 2)).sum()


def compute_weighted_value_loss(eltwise_loss, weights, batch_accumulator="mean"):
    assert batch_accumulator in ("mean", "sum") and eltwise_loss.ndim == 3
    loss_sum = torch.matmul(eltwise_loss.mean(2).sum(1), weights)
    return loss_sum / eltwise_loss.shape[0] if batch_accumulator == "mean" else loss_sum


class IQN(dqn.DQN):
    """DQN over implicit quantile functions; extra keyword arguments
    quantile_thresholds_N / _N_prime / _K and act_deterministically as in the
    reference (iqn.py:280-287)."""

    _recurrent_supported = False

    def __init__(self, *args, **kwargs):
        self.quantile_thresholds_N = kwargs.pop("quantile_thresholds_N", 64)
        self.quantile_thresholds_N_prime = kwargs.pop("quantile_thresholds_N_prime", 64)
        self.quantile_thresholds_K = kwargs.pop("quantile_thresholds_K", 32)
        self.act_deterministically = kwargs.pop("act_deterministically", False)
        super().__init__(*args, **kwargs)

    def _taus(self, batch_size, n):
        return torch.rand(batch_size, n, device=self.device, dtype=torch.float)

    def _compute_target_values(self, exp_batch):
        batch_size = len(exp_batch["reward"])
        taus_tilde = self._taus(batch_size, self.quantile_thresholds_K)
        target_next_tau2av = self.target_model(exp_batch["next_state"])
        greedy_actions = target_next_tau2av(taus_tilde).greedy_actions
        taus_prime = self._taus(batch_size, self.quantile_thresholds_N_prime)
        target_next_maxz = target_next_tau2av(taus_prime).evaluate_actions_as_quantiles(
            greedy_actions)
        return (exp_batch["reward"].unsqueeze(-1)
                + exp_batch["discount"].unsqueeze(-1)
                * (1.0 - exp_batch["is_state_terminal"].unsqueeze(-1)) * target_next_maxz)

    def _compute_y_and_taus(self, exp_batch):
        batch_size = exp_batch["reward"].shape[0]
        tau2av = self.model(exp_batch["state"])
        taus = self._taus(batch_size, self.quantile_thresholds_N)
        av = tau2av(taus)
        y = av.evaluate_actions_as_quantiles(exp_batch["action"])
        self._last_q = av.q_values.detach()
        return y, taus

    def _compute_loss(self, exp_batch, want_errors=False):
        y, taus = self._compute_y_and_taus(exp_batch)
        with torch.no_grad():
            t = self._compute_target_values(exp_batch)
        if self.use_fused_loss and y.is_cuda:
            return fused.quantile_huber_loss(y, t, taus, exp_batch.get("weights"),
                                             mean=self.batch_accumulator == "mean")
        eltwise_loss = compute_eltwise_huber_quantile_loss(y, t, taus)
        delta = eltwise_loss.detach().mean((1, 2)) if want_errors else None
        if "weights" in exp_batch:
            loss = compute_weighted_value_loss(eltwise_loss, exp_batch["weights"],
                                               batch_accumulator=self.batch_accumulator)
        else:
            loss = compute_value_loss(eltwise_loss, batch_accumulator=self.batch_accumulator)
        return loss, delta

    def _evaluate_model(self, batch_obs):
        batch_xs = self.batch_states(batch_obs, self.device, self.phi)
        tau2av = self.model(batch_xs)
        if not self.training and self.act_deterministically:
            taus_tilde = torch.linspace(
                0, 1, self.quantile_thresholds_K, device=self.device,
                dtype=torch.float32).repeat(len(batch_obs), 1)
        else:
            taus_tilde = self._taus(len(batch_obs), self.quantile_thresholds_K)
        return tau2av(taus_tilde)
