"""Action-value containers returned by Q-functions.

Same attribute surface as pfrl/action_value.py (ActionValue :9-42,
DiscreteActionValue :44-94, DistributionalDiscreteActionValue :97-180,
QuantileDiscreteActionValue :183-229): ``greedy_actions``, ``max``,
``evaluate_actions``, ``params`` and slicing.
"""
from abc import ABCMeta, abstractmethod

import torch
import torch.nn.functional as F


class ActionValue(object, metaclass=ABCMeta):
    @property
    @abstractmethod
    def greedy_actions(self):
        raise NotImplementedError()

    @property
    @abstractmethod
    def max(self):
        raise NotImplementedError()

    @abstractmethod
    def evaluate_actions(self, actions):
        raise NotImplementedError()

    @property
    @abstractmethod
    def params(self):
        raise NotImplementedError()

    def __getitem__(self, i):
        raise NotImplementedError()


def _row_gather(table, actions):
    """table[b, actions[b]] (keeps trailing dims)."""
    idx = actions.long().to(table.device)
    return table[torch.arange(table.shape[0], device=table.device), idx]


class DiscreteActionValue(ActionValue):
    """Q(s, .) for a finite action set; ``q_values`` is [batch, n_actions]."""

    def __init__(self, q_values, q_values_formatter=lambda x: x):
        assert isinstance(q_values, torch.Tensor)
        self.device = q_values.device
        self.q_values = q_values
        self.n_actions = q_values.shape[1]
        self.q_values_formatter = q_values_formatter

    @property
    def greedy_actions(self):
        return self.q_values.detach().argmax(dim=1).int()

    @property
    def max(self):
        return _row_gather(self.q_values, self.greedy_actions)

    def evaluate_actions(self, actions):
        return _row_gather(self.q_values, actions)

    def compute_advantage(self, actions):
        return self.evaluate_actions(actions) - self.max

    def compute_double_advantage(self, actions, argmax_actions):
        return self.evaluate_actions(actions) - self.evaluate_actions(argmax_actions)

    def compute_expectation(self, beta):
        return torch.sum(F.softmax(beta * self.q_values) * self.q_values, dim=1)

    def __repr__(self):
        return "DiscreteActionValue greedy_actions:{} q_values:{}".format(
            self.greedy_actions.detach().cpu().numpy(),
            self.q_values_formatter(self.q_values.detach().cpu().numpy()))

    @property
    def params(self):
        return (self.q_values,)

    def __getitem__(self, i):
        return DiscreteActionValue(self.q_values[i], q_values_formatter=self.q_values_formatter)


class DistributionalDiscreteActionValue(ActionValue):
    """Return distributions over fixed atoms: ``q_dist`` [batch, n_actions,
    n_atoms] probabilities, ``z_values`` [n_atoms] (C51 / Rainbow)."""

    def __init__(self, q_dist, z_values, q_values_formatter=lambda x: x):
        assert isinstance(q_dist, torch.Tensor) and isinstance(z_values, torch.Tensor)
        assert q_dist.ndim == 3 and z_values.ndim == 1
        assert q_dist.shape[2] == z_values.shape[0]
        self.device = q_dist.device
        self.z_values = z_values
        self.q_values = torch.matmul(q_dist, z_values)  # expectation per action
        self.q_dist = q_dist
        self.n_actions = q_dist.shape[1]
        self.q_values_formatter = q_values_formatter

    @property
    def greedy_actions(self):
        return self.q_values.argmax(dim=1).detach()

    @property
    def max(self):
        return _row_gather(self.q_values, self.greedy_actions)

    @property
    def max_as_distribution(self):
        """Distribution of the greedy action, [batch, n_atoms]."""
        return _row_gather(self.q_dist, self.greedy_actions)

    def evaluate_actions(self, actions):
        return _row_gather(self.q_values, actions)

    def evaluate_actions_as_distribution(self, actions):
        return _row_gather(self.q_dist, actions)

    # expectations-based helpers, as for plain Q-values
    def compute_advantage(self, actions):
        return self.evaluate_actions(actions) - self.max

    def compute_double_advantage(self, actions, argmax_actions):
        return self.evaluate_actions(actions) - self.evaluate_actions(argmax_actions)

    def compute_expectation(self, beta):
        return (torch.softmax(beta * self.q_values, dim=-1) * self.q_values).sum(dim=1)

    def __repr__(self):
        return "DistributionalDiscreteActionValue greedy_actions:{} q_values:{}".format(
            self.greedy_actions.detach().cpu().numpy(),
            self.q_values_formatter(self.q_values.detach().cpu().numpy()))

    @property
    def params(self):
        return (self.q_dist,)

    def __getitem__(self, i):
        return DistributionalDiscreteActionValue(
            self.q_dist[i], self.z_values, q_values_formatter=self.q_values_formatter)


class QuantileDiscreteActionValue(DiscreteActionValue):
    """Quantile estimates [batch, N, n_actions]; Q = mean over quantiles (IQN)."""

    def __init__(self, quantiles, q_values_formatter=lambda x: x):
        assert quantiles.ndim == 3
        self.quantiles = quantiles
        self.n_actions = quantiles.shape[2]
        self.q_values_formatter = q_values_formatter
        self.device = quantiles.device

    @property
    def q_values(self):
        return self.quantiles.mean(1)

    @q_values.setter
    def q_values(self, value):  # DiscreteActionValue.__init__ is bypassed
        raise AttributeError("q_values is derived from quantiles")

    def evaluate_actions_as_quantiles(self, actions):
        """[batch, N] quantiles of the given actions."""
        idx = actions.long().to(self.quantiles.device)
        return self.quantiles[torch.arange(self.quantiles.shape[0], device=idx.device), :, idx]

    def __repr__(self):
        return "QuantileDiscreteActionValue greedy_actions:{} q_values:{}".format(
            self.greedy_actions.detach().cpu().numpy(),
            self.q_values_formatter(self.q_values.detach().cpu().numpy()))

    @property
    def params(self):
        return (self.quantiles,)

    def __getitem__(self, i):
        return QuantileDiscreteActionValue(self.quantiles[i], self.q_values_formatter)


def _as_bound(b, device):
    """A bound as an fp32 tensor on ``device``: a scalar becomes [b]; a tensor already there
    in fp32 is used as it is, so no copy is made per forward (and the Q-function can be
    captured in a CUDA graph)."""
    if b is None:
        return None
    if isinstance(b, torch.Tensor) and b.device == device and b.dtype == torch.float32:
        return b
    if isinstance(b, (int, float)):
        b = [b]
    return torch.as_tensor(b).to(device).float()


class QuadraticActionValue(ActionValue):
    """Q(s, u) = V(s) - 1/2 (u - mu(s))^T P(s) (u - mu(s)) for continuous actions (NAF,
    arXiv:1603.00748; pfrl/action_value.py QuadraticActionValue).

    ``mu`` [batch, n] maximises the advantage, ``mat`` [batch, n, n] is P (positive definite
    when it comes from a NAF head), ``v`` [batch, 1] or [batch].  ``min_action`` and
    ``max_action`` (scalar, sequence, ndarray or tensor; not batched) clamp the greedy
    action; ``max`` is ``v`` without bounds and Q at the greedy action with them."""

    def __init__(self, mu, mat, v, min_action=None, max_action=None):
        self.mu = mu
        self.mat = mat
        self.v = v
        self.device = mu.device
        self.min_action = _as_bound(min_action, self.device)
        self.max_action = _as_bound(max_action, self.device)
        self.batch_size = self.mu.shape[0]
        self._greedy = self._max = None

    @property
    def greedy_actions(self):
        if self._greedy is None:
            a = self.mu
            if self.min_action is not None:
                a = torch.max(self.min_action.unsqueeze(0).expand_as(a), a)
            if self.max_action is not None:
                a = torch.min(self.max_action.unsqueeze(0).expand_as(a), a)
            self._greedy = a
        return self._greedy

    @property
    def max(self):
        if self._max is None:
            if self.min_action is None and self.max_action is None:
                self._max = self.v.reshape(self.batch_size)
            else:
                self._max = self.evaluate_actions(self.greedy_actions)
        return self._max

    def evaluate_actions(self, actions):
        u_minus_mu = actions - self.mu
        a = -0.5 * torch.matmul(torch.matmul(u_minus_mu[:, None, :], self.mat),
                                u_minus_mu[:, :, None])[:, 0, 0]
        return a + self.v.reshape(self.batch_size)

    def compute_advantage(self, actions):
        return self.evaluate_actions(actions) - self.max

    def compute_double_advantage(self, actions, argmax_actions):
        return self.evaluate_actions(actions) - self.evaluate_actions(argmax_actions)

    def __repr__(self):
        return "QuadraticActionValue greedy_actions:{} v:{}".format(
            self.greedy_actions.detach().cpu().numpy(), self.v.detach().cpu().numpy())

    @property
    def params(self):
        return (self.mu, self.mat, self.v)

    def __getitem__(self, i):
        return QuadraticActionValue(self.mu[i], self.mat[i], self.v[i],
                                    min_action=self.min_action, max_action=self.max_action)


class SingleActionValue(ActionValue):
    """Action value known only through callables: ``evaluator(actions)`` scores
    given actions, ``maximizer()`` returns the greedy ones (continuous-action
    critics; reference: pfrl/action_value.py:327-365).  Both results are computed
    at most once."""

    def __init__(self, evaluator, maximizer=None):
        self.evaluator = evaluator
        self.maximizer = maximizer
        self._greedy = None
        self._max = None

    @property
    def greedy_actions(self):
        if self._greedy is None:
            self._greedy = self.maximizer()
        return self._greedy

    @property
    def max(self):
        if self._max is None:
            self._max = self.evaluator(self.greedy_actions)
        return self._max

    def evaluate_actions(self, actions):
        return self.evaluator(actions)

    def compute_advantage(self, actions):
        return self.evaluator(actions) - self.max

    def compute_double_advantage(self, actions, argmax_actions):
        return self.evaluate_actions(actions) - self.evaluate_actions(argmax_actions)

    def __repr__(self):
        return "SingleActionValue"

    @property
    def params(self):
        return ()

    def __getitem__(self, i):
        raise NotImplementedError
