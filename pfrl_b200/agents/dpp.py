from abc import ABCMeta, abstractmethod

import torch

from pfrl_b200.agents import _advantage
from pfrl_b200.agents.dqn import DQN


class AbstractDPP(DQN, metaclass=ABCMeta):
    """Dynamic policy programming (arXiv:1004.2027; pfrl/agents/dpp.py).

    With L an operator that maps a row of action values to one value, the
    target is Q'(s, a) + r + discount (1 - terminal) L Q'(s') - L Q'(s): the
    target network's value of the stored action, moved by the Bellman backup of
    L and re-centred by L at s.  Subclasses define L in ``_l_operator``
    (an action value -> a [B] tensor); DPP, DPPL and DPPGreedy run it fused on
    CUDA, any other subclass in torch."""

    _recurrent_supported = False

    _fused_mode = None

    @abstractmethod
    def _l_operator(self, qout):
        raise NotImplementedError()

    def _compute_target_values(self, exp_batch):
        """r + discount (1 - terminal) L Q'(s')."""
        next_l = self._l_operator(self.target_model(exp_batch["next_state"]))
        return exp_batch["reward"] + exp_batch["discount"] * (
            1.0 - exp_batch["is_state_terminal"]) * next_l

    def _compute_y_and_t(self, exp_batch, qout=None):
        batch_size = exp_batch["reward"].shape[0]
        action = exp_batch["action"]
        # forwards in the reference's order: online(s), target(s), then target(s') in
        # _compute_target_values
        if qout is None:  # the fused path hands in its own forward at s
            qout = self.model(exp_batch["state"])
        y = qout.evaluate_actions(action).reshape(batch_size, 1)
        with torch.no_grad():
            target_qout = self.target_model(exp_batch["state"])
            l_here = self._l_operator(target_qout).reshape(batch_size, 1)
            backup = self._compute_target_values(exp_batch).reshape(batch_size, 1)
            t = target_qout.evaluate_actions(action).reshape(batch_size, 1) + backup - l_here
        return y, t

    def _compute_loss(self, exp_batch, want_errors=False):
        return _advantage.compute_loss(self, exp_batch, want_errors,
                                       eta=getattr(self, "eta", 1.0))


class DPP(AbstractDPP):
    """DPP whose L is the softmax-weighted mean of the action values,
    sum_b softmax(eta Q)_b Q_b.  ``eta`` > 0 is the inverse temperature, a
    keyword argument (default 1.0)."""

    _fused_mode = "dpp"

    def __init__(self, *args, **kwargs):
        self.eta = kwargs.pop("eta", 1.0)
        super().__init__(*args, **kwargs)

    def _l_operator(self, qout):
        return qout.compute_expectation(self.eta)


class DPPL(AbstractDPP):
    """DPP whose L is the soft maximum logsumexp(eta Q) / eta; ``eta`` > 0 as
    for DPP (default 1.0)."""

    _fused_mode = "dppl"

    def __init__(self, *args, **kwargs):
        self.eta = kwargs.pop("eta", 1.0)
        super().__init__(*args, **kwargs)

    def _l_operator(self, qout):
        return torch.logsumexp(self.eta * qout.q_values, dim=1) / self.eta


class DPPGreedy(AbstractDPP):
    """DPP whose L is the hard maximum max_b Q_b: the limit of DPP and DPPL as
    eta grows without bound."""

    _fused_mode = "dpp_greedy"

    def _l_operator(self, qout):
        return qout.max
