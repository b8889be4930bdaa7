import torch

from pfrl_b200.agents import pal


class DoublePAL(pal.PAL):
    """PAL with a double-Q next-state value (pfrl/agents/double_pal.py): the
    online network picks the greedy action at s', the target network values it.

    Unlike DoubleDQN, the online network's forward at s' runs in whatever
    train / eval mode the model is in, as the reference does; with noisy layers
    this matters for the noise stream."""

    _fused_mode = "double_pal"

    def _compute_y_and_t(self, exp_batch, qout=None):
        # forwards in the reference's order: online(s), online(s'), target(s), target(s')
        if qout is None:  # the fused path hands in its own forward at s
            qout = self.model(exp_batch["state"])
        y = qout.evaluate_actions(exp_batch["action"])
        with torch.no_grad():
            next_qout = self.model(exp_batch["next_state"])
            target_qout = self.target_model(exp_batch["state"])
            target_next_qout = self.target_model(exp_batch["next_state"])
            next_v = target_next_qout.evaluate_actions(next_qout.greedy_actions)
            t = self._persistent_target(exp_batch, target_qout, target_next_qout, next_v)
        return y, t
