"""William's episodic REINFORCE.

Public surface = pfrl/agents/reinforce.py: the reference's constructor, attributes,
``saved_attributes`` and statistics.  Returns are the reference's own per-episode
expression ``np.cumsum(list(reversed(r_seq[1:])))[::-1]`` on the host rewards, with its
quirks: ``_observe_train`` appends the terminal reward twice and ``r_seq[1:]`` drops the
first one.

An fp32 ``Categorical`` or ``Independent(Normal, 1)`` policy on CUDA takes the fused path
(``use_fused``, on by default):
  * acting runs under ``no_grad`` and records the batched observation (it stays on the
    device) and the sampled action (also kept on the device); ``average_entropy`` is an
    fp64 device average, read back in ``get_statistics``.  A step synchronises with the
    host where the reference's does too: the observation's upload in ``batch_states`` and
    the action's copy to the host, which ``act`` returns;
  * an update forwards the model once over every recorded step (one batch, or one packed
    sequence of the episodes from a ``None`` state for a recurrent model), uploads the
    returns, and runs the loss gradient of all rows in one kernel
    (csrc/reinforce.cu) that writes d loss / d(distribution parameters); one backward
    applies it, then the reference's clipping and optimizer step.  Nothing in the update
    synchronises with the host.
Recomputing the forward equals the graph acting would have kept because the parameters
do not change within a batch of episodes; so a model holding Dropout or BatchNorm in
train mode, or noisy layers (which draw fresh noise on every forward in either mode),
does not take the fused path.  Such models, CPU models, ``use_fused = False`` and other
distributions (a ``Categorical`` built from ``probs`` among them: its ``_param`` is not
the normalised logits the kernel differentiates) run the reference's formulation,
keeping each step's graph from acting.
"""
import warnings
from logging import getLogger

import numpy as np
import torch
from torch import nn

from pfrl_b200 import agent
from pfrl_b200.agents.acer import _pinned_to
from pfrl_b200.nn.noisy_linear import FactorizedNoisyLinear
from pfrl_b200.ops import reinforce as fused
from pfrl_b200.utils.batch_states import batch_states as default_batch_states
from pfrl_b200.utils.clip_l2_grad_norm import clip_l2_grad_norm_
from pfrl_b200.utils.mode_of_distribution import mode_of_distribution
from pfrl_b200.utils.modes import no_distribution_validation
from pfrl_b200.utils.recurrent import flatten_sequences_time_first, one_step_forward, \
    pack_and_forward

# layers whose train-mode forward is not a function of the parameters and the input alone
_TRAIN_MODE_STOCHASTIC = (nn.modules.dropout._DropoutNd, nn.modules.batchnorm._BatchNorm)


def recompute_equals_acting(model):
    """Whether a second forward of ``model`` on the same input gives what acting got: no
    Dropout or BatchNorm in train mode, and no noisy layer (whose forward draws fresh
    noise in either mode)."""
    return not any(isinstance(m, FactorizedNoisyLinear)
                   or (isinstance(m, _TRAIN_MODE_STOCHASTIC) and m.training)
                   for m in model.modules())


def fused_distribution(distrib):
    """The kernel's case: an fp32 ``Categorical`` over [N, K] built from logits (so that
    ``_param`` holds the normalised logits) or an fp32 ``Independent(Normal, 1)`` over
    [N, A]."""
    D = torch.distributions
    if type(distrib) is D.Categorical:
        return (distrib._param is vars(distrib).get("logits")
                and distrib._param.dtype == torch.float32 and distrib._param.dim() == 2)
    if type(distrib) is D.Independent and type(distrib.base_dist) is D.Normal:
        base = distrib.base_dist
        return (distrib.reinterpreted_batch_ndims == 1 and base.loc.dim() == 2
                and base.loc.dtype == torch.float32 and base.scale.dtype == torch.float32)
    return False


def _cat(xs):
    """Concatenate batched observations (tensors, or tuples of them) along axis 0."""
    if isinstance(xs[0], tuple):
        return tuple(_cat([x[i] for x in xs]) for i in range(len(xs[0])))
    return torch.cat(xs)


class REINFORCE(agent.AttributeSavingMixin, agent.Agent):
    """William's episodic REINFORCE.

    Arguments as the reference's ``pfrl.agents.REINFORCE``.  Statistics: average_entropy.
    """

    saved_attributes = ("model", "optimizer")

    def __init__(self, model, optimizer, gpu=None, beta=0, phi=lambda x: x, batchsize=1,
                 act_deterministically=False, average_entropy_decay=0.999,
                 backward_separately=False, batch_states=default_batch_states, recurrent=False,
                 max_grad_norm=None, logger=None):
        self.model = model
        if gpu is not None and gpu >= 0:
            assert torch.cuda.is_available()
            self.device = torch.device("cuda:{}".format(gpu))
            self.model.to(self.device)
        else:
            self.device = torch.device("cpu")
        self.optimizer = optimizer
        self.beta = beta
        self.phi = phi
        self.batchsize = batchsize
        self.backward_separately = backward_separately
        self.act_deterministically = act_deterministically
        self.average_entropy_decay = average_entropy_decay
        self.batch_states = batch_states
        self.recurrent = recurrent
        self.max_grad_norm = max_grad_norm
        self.logger = logger or getLogger(__name__)

        # Recurrent states of the model
        self.train_recurrent_states = None
        self.test_recurrent_states = None

        # Statistics
        self.average_entropy = 0

        self.t = 0
        self.n_backward = 0
        self.use_fused = True
        # the fused path's average_entropy: an fp64 device scalar (None while the host
        # attribute holds the value)
        self._entropy_stat = None
        # whether the steps recorded since the last update are fused (observations and
        # sampled actions, on the device) or the reference's (graphs); decided at the
        # first step of a record
        self._fused_record = False
        # False once a policy's distribution turned out not to be the kernel's case
        self._fused_distribution = True
        self._clear_record()

    # ---------------------------------------------------------------- records
    def _clear_record(self):
        self.reward_sequences = [[]]
        self.log_prob_sequences = [[]]
        self.entropy_sequences = [[]]
        self.obs_sequences = [[]]
        self.action_sequences = [[]]

    def _record_is_empty(self):
        return len(self.reward_sequences) == 1 and not self.reward_sequences[0] \
            and not self.log_prob_sequences[0] and not self.obs_sequences[0]

    def _fused_ok(self):
        return (self.use_fused and self._fused_distribution and self.device.type == "cuda"
                and recompute_equals_acting(self.model))

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

    def _forward(self, batch_obs, recurrent_states):
        if self.recurrent:
            return one_step_forward(self.model, batch_obs, recurrent_states)
        return self.model(batch_obs), None

    def _act_train(self, obs):
        batch_obs = self.batch_states([obs], self.device, self.phi)
        if self._record_is_empty():
            self._fused_record = self._fused_ok()
        if self._fused_record:
            action = self._act_train_fused(batch_obs)
            if action is not None:
                return action
        action_distrib, self.train_recurrent_states = self._forward(
            batch_obs, self.train_recurrent_states)
        batch_action = action_distrib.sample()

        # Save values used to compute losses
        self.log_prob_sequences[-1].append(action_distrib.log_prob(batch_action))
        self.entropy_sequences[-1].append(action_distrib.entropy())

        action = batch_action.cpu().numpy()[0]

        self.logger.debug("t:%s a:%s", self.t, action)

        # Update stats
        self._sync_stats()
        self.average_entropy += (1 - self.average_entropy_decay) * (
            float(action_distrib.entropy()) - self.average_entropy
        )

        return action

    def _act_train_fused(self, batch_obs):
        """One step of the fused record; None (nothing recorded, the recurrent state as it
        was) when the policy's distribution is not the kernel's case."""
        with torch.no_grad(), no_distribution_validation():
            action_distrib, states = self._forward(batch_obs, self.train_recurrent_states)
            if not fused_distribution(action_distrib):
                if not self._record_is_empty():
                    raise NotImplementedError(
                        "the policy's distribution changed type within a batch of episodes")
                self._fused_distribution = False
                self._fused_record = False
                return None
            self.train_recurrent_states = states
            batch_action = action_distrib.sample()
            if self._entropy_stat is None:
                self._entropy_stat = _pinned_to(np.array(self.average_entropy, np.float64),
                                                self.device)
            entropy = action_distrib.entropy().reshape(()).double()
            self._entropy_stat += (1 - self.average_entropy_decay) * (
                entropy - self._entropy_stat)
        self.obs_sequences[-1].append(batch_obs)
        self.action_sequences[-1].append(batch_action)
        action = batch_action.cpu().numpy()[0]
        self.logger.debug("t:%s a:%s", self.t, action)
        return action

    def _sync_stats(self):
        """Bring the fused path's device average back to the host attribute."""
        if self._entropy_stat is not None:
            self.average_entropy = self._entropy_stat.item()
            self._entropy_stat = None

    def _observe_train(self, obs, reward, done, reset):
        self.reward_sequences[-1].append(reward)
        self.t += 1

        if done or reset:
            if not done:
                warnings.warn(
                    "Since REINFORCE supports episodic environments only, "
                    "reset=True with done=False will throw away the last episode."
                )
                self.reward_sequences[-1] = []
                self.log_prob_sequences[-1] = []
                self.entropy_sequences[-1] = []
                self.obs_sequences[-1] = []
                self.action_sequences[-1] = []
            elif done:
                self.reward_sequences[-1].append(reward)
                if self.backward_separately:
                    self.accumulate_grad()
                    if self.n_backward == self.batchsize:
                        self.update_with_accumulated_grad()
                else:
                    if len(self.reward_sequences) == self.batchsize:
                        self.batch_update()
                    else:
                        # Prepare for the next episode
                        self.reward_sequences.append([])
                        self.log_prob_sequences.append([])
                        self.entropy_sequences.append([])
                        self.obs_sequences.append([])
                        self.action_sequences.append([])
            self.train_recurrent_states = None

    def _act_eval(self, obs):
        with torch.no_grad():
            batch_obs = self.batch_states([obs], self.device, self.phi)
            if self.recurrent:
                action_distrib, self.test_recurrent_states = one_step_forward(
                    self.model, batch_obs, self.test_recurrent_states
                )
            else:
                action_distrib = self.model(batch_obs)
            if self.act_deterministically:
                return mode_of_distribution(action_distrib).cpu().numpy()[0]
            else:
                return action_distrib.sample().cpu().numpy()[0]

    def _observe_eval(self, obs, reward, done, reset):
        if done or reset:
            self.test_recurrent_states = None

    # ----------------------------------------------------------------- updates
    def accumulate_grad(self):
        if self.n_backward == 0:
            self.optimizer.zero_grad()
        if self._fused_record:
            with no_distribution_validation():
                self._accumulate_grad_fused()
        else:
            # Compute losses
            losses = []
            for r_seq, log_prob_seq, ent_seq in zip(
                self.reward_sequences, self.log_prob_sequences, self.entropy_sequences
            ):
                assert len(r_seq) - 1 == len(log_prob_seq) == len(ent_seq)
                # Convert rewards into returns (=sum of future rewards)
                R_seq = np.cumsum(list(reversed(r_seq[1:])))[::-1]
                for R, log_prob, entropy in zip(R_seq, log_prob_seq, ent_seq):
                    loss = -R * log_prob - self.beta * entropy
                    losses.append(loss)
            total_loss = torch.stack(losses).sum() / self.batchsize
            total_loss.backward()
        self._clear_record()
        self.n_backward += 1

    def _fused_inputs(self):
        """(distribution over every recorded row, returns [N] on the host and the sampled
        actions [N(, A)] on the device, both in the distribution's row order)."""
        returns = []
        for r_seq, obs_seq, act_seq in zip(self.reward_sequences, self.obs_sequences,
                                           self.action_sequences):
            assert len(r_seq) - 1 == len(obs_seq) == len(act_seq)
            # the reference's returns, in the dtype numpy picks for them
            returns.append(np.asarray(np.cumsum(list(reversed(r_seq[1:])))[::-1]))
        actions = [a for seq in self.action_sequences for a in seq]
        if not self.recurrent:
            distrib = self.model(_cat([o for seq in self.obs_sequences for o in seq]))
            return distrib, np.concatenate(returns), torch.cat(actions)
        # the episodes longest first as one packed sequence, from the state acting began
        # each episode with; the output rows are time-major, and the returns and actions
        # are put in that order on the host (a list reordering, no device work)
        order = sorted(range(len(returns)), key=lambda i: -len(returns[i]))
        starts = np.cumsum([0] + [len(r) for r in returns])
        rows = flatten_sequences_time_first(
            [list(range(starts[i], starts[i + 1])) for i in order])
        distrib, _ = pack_and_forward(self.model, [_cat(self.obs_sequences[i]) for i in order],
                                      None)
        return (distrib, np.concatenate(returns)[np.asarray(rows, dtype=np.int64)],
                torch.cat([actions[r] for r in rows]))

    def _accumulate_grad_fused(self):
        distrib, returns, actions = self._fused_inputs()
        if not fused_distribution(distrib):
            raise NotImplementedError(
                "the policy's distribution changed type within a batch of episodes")
        # the update's one upload
        R = _pinned_to(returns.astype(np.float32), self.device)
        if type(distrib) is torch.distributions.Categorical:
            tensors = [distrib._param]
            grads = list(fused.loss_grads(R, self.batchsize, self.beta, z=distrib._param,
                                          actions=actions.reshape(-1)))
        else:
            loc, scale = distrib.base_dist.loc, distrib.base_dist.scale
            a = actions.reshape(loc.shape)
            g_loc, g_scale = fused.loss_grads(R, self.batchsize, self.beta, loc=loc,
                                              scale=scale, action_values=a,
                                              scale_grad=scale.requires_grad)
            tensors, grads = [loc], [g_loc]
            if scale.requires_grad:
                tensors.append(scale)
                grads.append(g_scale)
        torch.autograd.backward(tensors, grads)

    def batch_update(self):
        assert len(self.reward_sequences) == self.batchsize
        assert len(self.log_prob_sequences) == self.batchsize
        assert len(self.entropy_sequences) == self.batchsize
        # Update the model
        assert self.n_backward == 0
        self.accumulate_grad()
        if self.max_grad_norm is not None:
            clip_l2_grad_norm_(self.model.parameters(), self.max_grad_norm)
        self.optimizer.step()
        self.n_backward = 0

    def update_with_accumulated_grad(self):
        assert self.n_backward == self.batchsize
        if self.max_grad_norm is not None:
            clip_l2_grad_norm_(self.model.parameters(), self.max_grad_norm)
        self.optimizer.step()
        self.n_backward = 0

    def get_statistics(self):
        self._sync_stats()
        return [
            ("average_entropy", self.average_entropy),
        ]
