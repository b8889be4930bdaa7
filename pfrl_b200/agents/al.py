import torch

from pfrl_b200.agents import _advantage, dqn


class AL(dqn.DQN):
    """Advantage learning (arXiv:1512.04860; pfrl/agents/al.py).

    The regression target is the one-step Bellman target plus ``alpha`` times
    the target network's advantage of the stored action, Q'(s, a) - max_b Q'(s, b).
    The advantage is never positive, so non-greedy actions are pushed down and
    the gap to the greedy action grows.  ``alpha`` is a keyword argument
    (default 0.9); everything else is DQN's.
    """

    _recurrent_supported = False

    _fused_mode = "al"

    def __init__(self, *args, **kwargs):
        self.alpha = kwargs.pop("alpha", 0.9)
        super().__init__(*args, **kwargs)

    def _compute_y_and_t(self, exp_batch, qout=None):
        # forwards in the reference's order: online(s), target(s), target(s')
        if qout is None:  # the fused path hands in its own forward at s
            qout = self.model(exp_batch["state"])
        y = qout.evaluate_actions(exp_batch["action"])
        with torch.no_grad():
            target_qout = self.target_model(exp_batch["state"])
            target_next_qout = self.target_model(exp_batch["next_state"])
            bellman = exp_batch["reward"] + exp_batch["discount"] * (
                1.0 - exp_batch["is_state_terminal"]) * target_next_qout.max
            t = bellman + self.alpha * target_qout.compute_advantage(exp_batch["action"])
        return y, t

    def _compute_loss(self, exp_batch, want_errors=False):
        return _advantage.compute_loss(self, exp_batch, want_errors, alpha=self.alpha)
