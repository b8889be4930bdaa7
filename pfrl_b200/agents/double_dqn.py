from pfrl_b200.agents import dqn
from pfrl_b200.utils.modes import evaluating


class DoubleDQN(dqn.DQN):
    """Double DQN (arXiv:1509.06461): the online network picks the next
    action, the target network evaluates it (pfrl/agents/double_dqn.py:12-40)."""

    _fused_mode = "double_dqn"

    def _next_q(self, exp_batch):
        # recurrent: both forwards run over the packed next states from the
        # batch's next_recurrent_state (double_dqn.py:15-32)
        with evaluating(self.model):
            next_qout = self._forward(self.model, exp_batch, "next_state")
        target_next_qout = self._forward(self.target_model, exp_batch, "next_state")
        return target_next_qout.evaluate_actions(next_qout.greedy_actions)
