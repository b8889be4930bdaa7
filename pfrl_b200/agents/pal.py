import torch

from pfrl_b200.agents import _advantage, dqn


class PAL(dqn.DQN):
    """Persistent advantage learning (arXiv:1512.04860; pfrl/agents/pal.py).

    Like AL, but the correction added to the Bellman target is ``alpha`` times
    the larger of two advantages of the stored action a: the target network's
    at s and at s'.  Using a at s' too is what makes the operator "persistent":
    an action that stays good in the next state keeps its value.  ``alpha`` is a
    keyword argument (default 0.9).
    """

    _recurrent_supported = False

    _fused_mode = "pal"

    def __init__(self, *args, **kwargs):
        self.alpha = kwargs.pop("alpha", 0.9)
        super().__init__(*args, **kwargs)

    def _persistent_target(self, exp_batch, target_qout, target_next_qout, next_v):
        """r + discount (1 - terminal) next_v + alpha max(A'(s, a), A'(s', a))."""
        action = exp_batch["action"]
        bellman = exp_batch["reward"] + exp_batch["discount"] * (
            1.0 - exp_batch["is_state_terminal"]) * next_v
        advantage = torch.max(target_qout.compute_advantage(action),
                              target_next_qout.compute_advantage(action))
        return bellman + self.alpha * advantage

    def _compute_y_and_t(self, exp_batch, qout=None):
        # forwards in the reference's order: online(s), target(s), target(s')
        if qout is None:  # the fused path hands in its own forward at s
            qout = self.model(exp_batch["state"])
        y = qout.evaluate_actions(exp_batch["action"])
        with torch.no_grad():
            target_qout = self.target_model(exp_batch["state"])
            target_next_qout = self.target_model(exp_batch["next_state"])
            t = self._persistent_target(exp_batch, target_qout, target_next_qout,
                                        target_next_qout.max)
        return y, t

    def _compute_loss(self, exp_batch, want_errors=False):
        return _advantage.compute_loss(self, exp_batch, want_errors, alpha=self.alpha)
