"""A3C: Asynchronous Advantage Actor-Critic (arXiv:1602.01783).

Public surface = pfrl/agents/a3c.py: the reference's constructor, ``shared_model`` /
``model``, ``sync_parameters``, ``assert_shared_memory``, ``shared_attributes``,
``saved_attributes``, ``process_idx``, ``load`` and statistics.  Training is single-process
through ``train_agent`` / ``train_agent_with_evaluation``, on the device of ``model``.

An fp32 ``Categorical`` (built from logits) or ``Independent(Normal, 1)`` policy on CUDA
takes the fused path (``use_fused``, on by default):
  * acting runs under ``no_grad`` and keeps each step's batched observation and sampled
    action on the device; ``average_value`` and ``average_entropy`` are fp64 device
    averages, read back in ``get_statistics``.  The action's copy to the host, which
    ``act`` returns, is the step's only synchronisation after the observation's upload;
  * an update takes the bootstrap value from the reference's separate eval-mode forward
    and leaves it on the device, forwards the model once over the recorded observations
    (one packed sequence from the segment's starting state for a recurrent model), uploads
    the rewards, and runs the returns scan and the loss gradient of every row in one
    kernel (csrc/a3c.cu).  One backward applies the gradient, then the reference's
    clipping, the copy of the gradients to ``shared_model``, the optimizer step and
    ``sync_parameters``.  Nothing in the update synchronises with the host.
Recomputing the forward is the reference's own algorithm here, so any model may take it.
CPU models, ``use_fused = False``, and other distributions or dtypes (a ``Categorical``
built from ``probs`` among them) run the reference's formulation in its order.
"""
import contextlib
import copy
import logging
from logging import getLogger

import numpy as np
import torch
import torch.nn.functional as F

from pfrl_b200 import agent
from pfrl_b200.agents.acer import _pinned_to
from pfrl_b200.agents.reinforce import _cat, fused_distribution
from pfrl_b200.ops import a3c as fused
from pfrl_b200.utils import copy_param
from pfrl_b200.utils.batch_states import batch_states
from pfrl_b200.utils.clip_l2_grad_norm import clip_l2_grad_norm_
from pfrl_b200.utils.mode_of_distribution import mode_of_distribution
from pfrl_b200.utils.modes import evaluating, no_distribution_validation
from pfrl_b200.utils.recurrent import one_step_forward, pack_and_forward

logger = getLogger(__name__)


class A3C(agent.AttributeSavingMixin, agent.AsyncAgent):
    """A3C: Asynchronous Advantage Actor-Critic.

    Arguments as the reference's ``pfrl.agents.A3C``.  The models stay on the device of
    ``model``.  Statistics: average_value, average_entropy.
    """

    process_idx = None
    saved_attributes = ("model", "optimizer")

    def __init__(self, model, optimizer, t_max, gamma, beta=1e-2, process_idx=0,
                 phi=lambda x: x, pi_loss_coef=1.0, v_loss_coef=0.5,
                 keep_loss_scale_same=False, normalize_grad_by_t_max=False,
                 use_average_reward=False, act_deterministically=False, max_grad_norm=None,
                 recurrent=False, average_entropy_decay=0.999, average_value_decay=0.999,
                 batch_states=batch_states):
        # Globally shared model
        self.shared_model = model
        # Thread specific model
        self.model = copy.deepcopy(self.shared_model)
        self.optimizer = optimizer

        self.t_max = t_max
        self.gamma = gamma
        self.beta = beta
        self.phi = phi
        self.pi_loss_coef = pi_loss_coef
        self.v_loss_coef = v_loss_coef
        self.keep_loss_scale_same = keep_loss_scale_same
        self.normalize_grad_by_t_max = normalize_grad_by_t_max
        self.use_average_reward = use_average_reward
        self.act_deterministically = act_deterministically
        self.max_grad_norm = max_grad_norm
        self.recurrent = recurrent
        self.average_value_decay = average_value_decay
        self.average_entropy_decay = average_entropy_decay
        self.batch_states = batch_states

        param = next(iter(model.parameters()), None)
        self.device = param.device if param is not None else torch.device("cpu")
        self.use_fused = True
        self.t = 0
        self.t_start = 0
        self.past_obs = {}
        self.past_action = {}
        self.past_rewards = {}
        self.past_recurrent_state = {}
        # the fused path's record: each step's batched observation, on the device
        self.past_statevar = {}
        self.average_reward = 0

        # Recurrent states of the model
        self.train_recurrent_states = None
        self.test_recurrent_states = None

        # Stats
        self.average_value = 0
        self.average_entropy = 0
        # the fused path's statistics: fp64 device averages of value and entropy (None while
        # the host attributes hold the values)
        self._stats = None
        self._stat_rates = None

    def sync_parameters(self):
        copy_param.copy_param(target_link=self.model, source_link=self.shared_model)

    def assert_shared_memory(self):
        agent.assert_shared_memory(self, ("model", "shared_model"))

    @property
    def shared_attributes(self):
        return ("shared_model", "optimizer")

    def _fused_ok(self):
        return self.use_fused and self.device.type == "cuda"

    def _validation(self, fused_step):
        # argument validation of the distributions would read the device
        return no_distribution_validation() if fused_step else contextlib.nullcontext()

    # ----------------------------------------------------------------- updates
    def _loss_factors(self):
        """pi_loss_factor and v_loss_factor, as the reference computes them."""
        pi_loss_factor = self.pi_loss_coef
        v_loss_factor = self.v_loss_coef

        # Normalize the loss of sequences truncated by terminal states
        if self.keep_loss_scale_same and self.t - self.t_start < self.t_max:
            factor = self.t_max / (self.t - self.t_start)
            pi_loss_factor *= factor
            v_loss_factor *= factor

        if self.normalize_grad_by_t_max:
            pi_loss_factor /= self.t - self.t_start
            v_loss_factor /= self.t - self.t_start
        return pi_loss_factor, v_loss_factor

    def update(self, statevar):
        assert self.t_start < self.t

        n = self.t - self.t_start

        self.assert_shared_memory()

        steps = range(self.t_start, self.t)
        # the segment was recorded on the device, every step of it
        fused_step = self._fused_ok() and all(i in self.past_statevar for i in steps)
        with self._validation(fused_step):
            if statevar is None:
                vout = None
            else:
                with torch.no_grad(), evaluating(self.model):
                    if self.recurrent:
                        (_, vout), _ = one_step_forward(
                            self.model, statevar, self.train_recurrent_states)
                    else:
                        _, vout = self.model(statevar)

            pi_loss_factor, v_loss_factor = self._loss_factors()

            # Batch re-compute for efficient backprop
            if fused_step:
                batch_obs = _cat([self.past_statevar[i] for i in steps])
            else:
                batch_obs = self.batch_states([self.past_obs[i] for i in steps], self.device,
                                              self.phi)
            if self.recurrent:
                (batch_distrib, batch_v), _ = pack_and_forward(
                    self.model, [batch_obs], self.past_recurrent_state[self.t_start])
            else:
                batch_distrib, batch_v = self.model(batch_obs)
            batch_action = torch.stack([self.past_action[i] for i in steps])

            self.model.zero_grad()
            if (fused_step and fused_distribution(batch_distrib)
                    and batch_v.dtype == torch.float32
                    and (vout is None or vout.dtype == torch.float32)):
                self._fused_backward(batch_distrib, batch_v, batch_action, vout,
                                     pi_loss_factor, v_loss_factor)
            else:
                self._reference_backward(n, batch_distrib, batch_v, batch_action, vout,
                                         pi_loss_factor, v_loss_factor)

        if self.max_grad_norm is not None:
            clip_l2_grad_norm_(self.model.parameters(), self.max_grad_norm)
        # Copy the gradients to the globally shared model
        if fused_step:
            copy_param.copy_grad_into(target_link=self.shared_model, source_link=self.model)
        else:
            copy_param.copy_grad(target_link=self.shared_model, source_link=self.model)
        # Update the globally shared model
        self.optimizer.step()
        if self.process_idx == 0:
            logger.debug("update")

        self.sync_parameters()

        self.past_obs = {}
        self.past_action = {}
        self.past_rewards = {}
        self.past_recurrent_state = {}
        self.past_statevar = {}

        self.t_start = self.t

    def _reference_backward(self, n, batch_distrib, batch_v, batch_action, vout,
                            pi_loss_factor, v_loss_factor):
        """pfrl/agents/a3c.py:177-214, from the loss on."""
        R = 0 if vout is None else float(vout)
        batch_log_prob = batch_distrib.log_prob(batch_action)
        batch_entropy = batch_distrib.entropy()
        rev_returns = []
        for i in reversed(range(self.t_start, self.t)):
            R *= self.gamma
            R += self.past_rewards[i]
            rev_returns.append(R)
        batch_return = torch.as_tensor(list(reversed(rev_returns)), dtype=torch.float,
                                       device=self.device)
        batch_adv = batch_return - batch_v.detach().squeeze(-1)
        assert batch_log_prob.shape == (n,)
        assert batch_adv.shape == (n,)
        assert batch_entropy.shape == (n,)
        pi_loss = torch.sum(-batch_adv * batch_log_prob - self.beta * batch_entropy, dim=0)
        assert batch_v.shape == (n, 1)
        assert batch_return.shape == (n,)
        v_loss = F.mse_loss(batch_v, batch_return[..., None], reduction="sum") / 2

        if pi_loss_factor != 1.0:
            pi_loss *= pi_loss_factor

        if v_loss_factor != 1.0:
            v_loss *= v_loss_factor

        if self.process_idx == 0:
            logger.debug("pi_loss:%s v_loss:%s", pi_loss, v_loss)

        total_loss = torch.squeeze(pi_loss) + torch.squeeze(v_loss)

        # Compute gradients using thread-specific model
        total_loss.backward()

    def _fused_backward(self, batch_distrib, batch_v, batch_action, vout, pi_loss_factor,
                        v_loss_factor):
        """The loss gradient of every row in one launch, applied with one backward."""
        n = batch_v.shape[0]
        assert batch_v.shape == (n, 1)
        # the update's one upload
        rewards = _pinned_to(np.asarray([self.past_rewards[i]
                                         for i in range(self.t_start, self.t)],
                                        dtype=np.float64), self.device)
        bootstrap = None if vout is None else vout.detach().reshape(1)
        want_loss = self.process_idx == 0 and logger.isEnabledFor(logging.DEBUG)
        args = (batch_v, rewards, bootstrap, self.gamma, self.beta, pi_loss_factor,
                v_loss_factor)
        if type(batch_distrib) is torch.distributions.Categorical:
            tensors = [batch_distrib._param]
            grads, g_v, _, pi_loss, v_loss = fused.loss_grads(
                *args, z=batch_distrib._param, actions=batch_action.reshape(-1),
                want_loss=want_loss)
        else:
            loc, scale = batch_distrib.base_dist.loc, batch_distrib.base_dist.scale
            tensors = [loc, scale]
            grads, g_v, _, pi_loss, v_loss = fused.loss_grads(
                *args, loc=loc, scale=scale, action_values=batch_action.reshape(loc.shape),
                scale_grad=scale.requires_grad, want_loss=want_loss)
        if self.process_idx == 0:
            logger.debug("pi_loss:%s v_loss:%s", pi_loss, v_loss)
        pairs = [(t, g) for t, g in zip(tensors + [batch_v], list(grads) + [g_v.reshape(n, 1)])
                 if t.requires_grad]
        torch.autograd.backward([t for t, _ in pairs], [g for _, g in pairs])

    # ------------------------------------------------------------------ acting
    def act(self, obs):
        if self.training:
            return self._act_train(obs)
        else:
            return self._act_eval(obs)

    def observe(self, obs, reward, done, reset):
        if self.training:
            self._observe_train(obs, reward, done, reset)
        else:
            self._observe_eval(obs, reward, done, reset)

    def _act_train(self, obs):
        self.past_obs[self.t] = obs

        fused_step = self._fused_ok()
        with torch.no_grad(), self._validation(fused_step):
            statevar = self.batch_states([obs], self.device, self.phi)
            if self.recurrent:
                self.past_recurrent_state[self.t] = self.train_recurrent_states
                (pout, vout), self.train_recurrent_states = one_step_forward(
                    self.model, statevar, self.train_recurrent_states
                )
            else:
                pout, vout = self.model(statevar)
            # Do not backprop through sampled actions
            action = pout.sample()
            self.past_action[self.t] = action[0].detach()
            if fused_step:
                self.past_statevar[self.t] = statevar
            action = action.cpu().numpy()[0]

            # Update stats
            self._update_stats(vout, pout, fused_step)

        return action

    def _update_stats(self, vout, pout, fused_step):
        if (fused_step and fused_distribution(pout) and vout.dtype == torch.float32):
            if self._stats is None:
                self._stats = _pinned_to(
                    np.array([self.average_value, self.average_entropy], np.float64),
                    self.device)
                self._stat_rates = _pinned_to(
                    np.array([1 - self.average_value_decay, 1 - self.average_entropy_decay],
                             np.float64), self.device)
            x = torch.stack([vout.reshape(()), pout.entropy().reshape(())]).double()
            self._stats += self._stat_rates * (x - self._stats)
            return
        self._sync_stats()
        self.average_value += (1 - self.average_value_decay) * (
            float(vout) - self.average_value
        )
        self.average_entropy += (1 - self.average_entropy_decay) * (
            float(pout.entropy()) - self.average_entropy
        )

    def _sync_stats(self):
        """Bring the fused path's device averages back to the host attributes."""
        if self._stats is not None:
            self.average_value, self.average_entropy = self._stats.tolist()
            self._stats = None

    def _observe_train(self, obs, reward, done, reset):
        self.t += 1
        self.past_rewards[self.t - 1] = reward
        if self.process_idx == 0:
            logger.debug(
                "t:%s action:%s reward:%s", self.t, self.past_action[self.t - 1], reward
            )
        if self.t - self.t_start == self.t_max or done or reset:
            if done:
                statevar = None
            else:
                statevar = self.batch_states([obs], self.device, self.phi)
            self.update(statevar)
        if done or reset:
            self.train_recurrent_states = None

    def _act_eval(self, obs):
        # Use the process-local model for acting
        with torch.no_grad(), evaluating(self.model):
            statevar = self.batch_states([obs], self.device, self.phi)
            if self.recurrent:
                (pout, _), self.test_recurrent_states = one_step_forward(
                    self.model, statevar, self.test_recurrent_states
                )
            else:
                pout, _ = self.model(statevar)
            if self.act_deterministically:
                return mode_of_distribution(pout).cpu().numpy()[0]
            else:
                return pout.sample().cpu().numpy()[0]

    def _observe_eval(self, obs, reward, done, reset):
        if done or reset:
            self.test_recurrent_states = None

    def load(self, dirname):
        super().load(dirname)
        copy_param.copy_param(target_link=self.shared_model, source_link=self.model)

    def get_statistics(self):
        self._sync_stats()
        return [
            ("average_value", self.average_value),
            ("average_entropy", self.average_entropy),
        ]
