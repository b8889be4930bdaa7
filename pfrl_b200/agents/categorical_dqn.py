"""Categorical DQN (C51, arXiv:1707.06887) on the device replay path.

Reference: pfrl/agents/categorical_dqn.py (_apply_categorical_projection
:7-57, CategoricalDQN :100-204).  The projection + cross-entropy + per-sample
priority error + weighted reduction run as one fused CUDA kernel pair
(forward / backward, pfrl_b200/csrc/losses.cu) when the tensors are on the
GPU; the torch formulation below is the CPU path and the numerics reference.
"""
import torch

from pfrl_b200.agents import dqn
from pfrl_b200.ops import losses as fused


def _apply_categorical_projection(y, y_probs, z):
    """Project the distribution (atoms ``y`` [B, n] with probabilities
    ``y_probs`` [B, n]) onto the fixed, evenly spaced support ``z`` [n]
    (Algorithm 1 of the C51 paper; categorical_dqn.py:7-57)."""
    batch_size, n_atoms = y.shape
    assert z.shape == (n_atoms,)
    assert y_probs.shape == (batch_size, n_atoms)
    delta_z = z[1] - z[0]
    v_min, v_max = z[0], z[-1]
    y = torch.clamp(y, v_min, v_max)
    bj = torch.clamp((y - v_min) / delta_z, 0, n_atoms - 1)  # guards inexact delta_z
    lo, up = torch.floor(bj), torch.ceil(bj)
    frac = bj - lo
    z_probs = torch.zeros((batch_size, n_atoms), dtype=torch.float32, device=y.device)
    # mass (1 - frac) to the lower atom, frac to the upper one; "1 - frac"
    # rather than "up - bj" keeps the whole mass when bj is an integer
    z_probs.scatter_add_(1, lo.long(), y_probs * (1 - frac))
    z_probs.scatter_add_(1, up.long(), y_probs * frac)
    return z_probs


def compute_value_loss(eltwise_loss, batch_accumulator="mean"):
    assert batch_accumulator in ("mean", "sum")
    if batch_accumulator == "sum":
        return eltwise_loss.sum()
    return eltwise_loss.sum(dim=1).mean()


def compute_weighted_value_loss(eltwise_loss, batch_size, weights, batch_accumulator="mean"):
    assert batch_accumulator in ("mean", "sum")
    loss_sum = torch.matmul(eltwise_loss.sum(dim=1), weights.to(eltwise_loss.device))
    return loss_sum / batch_size if batch_accumulator == "mean" else loss_sum


class CategoricalDQN(dqn.DQN):
    """DQN over return distributions; ``q_function`` must return a
    DistributionalDiscreteActionValue, ``clip_delta`` is ignored."""

    _recurrent_supported = False

    use_fused_loss = True

    def _next_distribution(self, exp_batch):
        """(p(s', a*) [B, n_atoms], z_values) with a* greedy under the target net."""
        target_next_qout = self.target_model(exp_batch["next_state"])
        return target_next_qout.max_as_distribution.detach(), target_next_qout.z_values

    def _compute_target_values(self, exp_batch):
        next_q_max, z_values = self._next_distribution(exp_batch)
        rewards = exp_batch["reward"]
        Tz = (rewards[..., None]
              + (1.0 - exp_batch["is_state_terminal"][..., None])
              * exp_batch["discount"][..., None] * z_values[None])
        return _apply_categorical_projection(Tz, next_q_max, z_values)

    def _compute_y_and_t(self, exp_batch):
        qout = self.model(exp_batch["state"])
        actions = exp_batch["action"]
        batch_q = qout.evaluate_actions_as_distribution(actions)
        with torch.no_grad():
            batch_q_target = self._compute_target_values(exp_batch)
            self._last_q = qout.evaluate_actions(actions).detach()
        return batch_q, batch_q_target

    def _compute_loss(self, exp_batch, want_errors=False):
        """Cross entropy between the projected target and the prediction
        (categorical_dqn.py:178-204); per-sample sums are the priorities."""
        if self.use_fused_loss and exp_batch["reward"].is_cuda:
            return self._compute_loss_fused(exp_batch)
        y, t = self._compute_y_and_t(exp_batch)
        eltwise_loss = -t * torch.log(torch.clamp(y, 1e-10, 1.0))
        delta = eltwise_loss.detach().sum(dim=1) if want_errors else None
        if "weights" in exp_batch:
            loss = compute_weighted_value_loss(
                eltwise_loss, y.shape[0], exp_batch["weights"],
                batch_accumulator=self.batch_accumulator)
        else:
            loss = compute_value_loss(eltwise_loss, batch_accumulator=self.batch_accumulator)
        return loss, delta

    def _compute_loss_fused(self, exp_batch):
        qout = self.model(exp_batch["state"])
        actions = exp_batch["action"]
        y = qout.evaluate_actions_as_distribution(actions)
        with torch.no_grad():
            next_p, z_values = self._next_distribution(exp_batch)
            self._last_q = qout.evaluate_actions(actions).detach()
        # the model's own atoms, as the torch path uses them: a linspace rebuilt on the
        # device differs from them in the last bit for some atoms
        loss, delta = fused.c51_loss(
            y, next_p, exp_batch["reward"], exp_batch["discount"],
            exp_batch["is_state_terminal"], exp_batch.get("weights"),
            mean=self.batch_accumulator == "mean", z=z_values)
        return loss, delta
