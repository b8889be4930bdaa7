"""ACER (Actor-Critic with Experience Replay, https://arxiv.org/abs/1611.01224).

Public surface = pfrl/agents/acer.py: the module functions, the two action heads, and
``ACER`` with the reference's constructor, ``saved_attributes``, ``shared_attributes``,
``process_idx`` and statistics.  Training is single-process (``experiments.train_agent``
/ ``train_agent_with_evaluation``); the models live on the device of the model passed in.

An fp32 ``Categorical`` policy on CUDA takes the fused path (``use_fused``, on by
default):
  * the replay update gathers the sampled subsequence's states (and the bootstrap
    state when its last transition is not terminal) in one launch, forwards ``model``
    once over them (one packed sequence from a ``None`` state for a recurrent model)
    and ``shared_average_model`` once, reads the behaviour policy's rows from the
    buffer's mu ring, and runs the whole loss in one kernel (csrc/acer.cu) that
    writes d loss / d logits and d loss / d Q; one backward applies them;
  * the online update stacks the outputs kept from acting and runs the same kernel
    on-policy;
  * acting keeps the statistics as fp64 device averages; the action is its only copy
    to the host.
Neither update copies anything to the host or synchronises with it.  Everything else
(CPU models, ``use_fused = False``, other distributions such as the Gaussian head) runs
the reference's formulation in its operation order on the model's device.
"""
import copy
from logging import getLogger

import numpy as np
import torch
from torch import nn

from pfrl_b200 import agent
from pfrl_b200.action_value import SingleActionValue
from pfrl_b200.ops import acer as fused
from pfrl_b200.utils import copy_param
from pfrl_b200.utils.batch_states import batch_states
from pfrl_b200.utils.clip_l2_grad_norm import clip_l2_grad_norm_
from pfrl_b200.utils.mode_of_distribution import mode_of_distribution
from pfrl_b200.utils.modes import no_distribution_validation
from pfrl_b200.utils.recurrent import detach_recurrent_state, one_step_forward, pack_and_forward


def compute_importance(pi, mu, x):
    """pi(x) / mu(x) as a Python float."""
    with torch.no_grad():
        return float(torch.exp(pi.log_prob(x) - mu.log_prob(x)))


def compute_full_importance(pi, mu):
    """pi / mu for every category (both Categorical; their logits are normalised)."""
    assert isinstance(pi, torch.distributions.Categorical)
    assert isinstance(mu, torch.distributions.Categorical)
    with torch.no_grad():
        return torch.exp(pi.logits - mu.logits)


def compute_policy_gradient_full_correction(action_distrib, action_distrib_mu, action_value,
                                            v, truncation_threshold):
    """Off-policy bias correction summed over all actions (categorical policies)."""
    assert isinstance(action_distrib, torch.distributions.Categorical)
    assert isinstance(action_distrib_mu, torch.distributions.Categorical)
    assert truncation_threshold is not None
    assert np.isscalar(v)
    with torch.no_grad():
        rho_all_inv = compute_full_importance(action_distrib_mu, action_distrib)
        weight = torch.nn.functional.relu(1 - truncation_threshold * rho_all_inv) \
            * action_distrib.probs[0]
        adv = action_value.q_values[0] - v
    return -(weight * action_distrib.logits * adv).sum(1)


def compute_policy_gradient_sample_correction(action_distrib, action_distrib_mu, action_value,
                                              v, truncation_threshold):
    """Off-policy bias correction on one action sampled from the policy."""
    assert np.isscalar(v)
    assert truncation_threshold is not None
    with torch.no_grad():
        sample_action = action_distrib.sample()
        rho_dash_inv = compute_importance(action_distrib_mu, action_distrib, sample_action)
        if truncation_threshold > 0 and rho_dash_inv >= 1 / truncation_threshold:
            return torch.as_tensor(0, dtype=torch.float)
        weight = max(0, 1 - truncation_threshold * rho_dash_inv)
        assert weight <= 1
        adv = float(action_value.evaluate_actions(sample_action)) - v
    return -(weight * action_distrib.log_prob(sample_action) * adv)


def compute_policy_gradient_loss(action, advantage, action_distrib, action_distrib_mu,
                                 action_value, v, truncation_threshold):
    """Policy-gradient loss with truncated importance weights and bias correction
    (on-policy when ``action_distrib_mu`` is None)."""
    assert np.isscalar(advantage)
    assert np.isscalar(v)
    log_prob = action_distrib.log_prob(action)
    if action_distrib_mu is None:
        return -log_prob * advantage
    rho = compute_importance(action_distrib, action_distrib_mu, action)
    g_loss = 0
    if truncation_threshold is None:
        g_loss -= rho * log_prob * advantage
        return g_loss
    g_loss -= min(truncation_threshold, rho) * log_prob * advantage
    correction = (compute_policy_gradient_full_correction
                  if isinstance(action_distrib, torch.distributions.Categorical)
                  else compute_policy_gradient_sample_correction)
    g_loss += correction(action_distrib=action_distrib, action_distrib_mu=action_distrib_mu,
                         action_value=action_value, v=v,
                         truncation_threshold=truncation_threshold)
    return g_loss


class ACERDiscreteActionHead(nn.Module):
    """A policy ``pi`` and a Q-function ``q`` over the same input; returns the action
    distribution, the Q values and v = sum_a pi(a) Q(a)."""

    def __init__(self, pi, q):
        super().__init__()
        self.pi = pi
        self.q = q

    def forward(self, obs):
        action_distrib = self.pi(obs)
        action_value = self.q(obs)
        v = (action_distrib.probs * action_value.q_values).sum(1)
        return action_distrib, action_value, v


class ACERContinuousActionHead(nn.Module):
    """A policy ``pi``, a V-function ``v`` and an advantage function ``adv``; Q(a) is
    v + adv(a) minus the mean advantage of ``n`` actions sampled from the policy."""

    def __init__(self, pi, v, adv, n=5):
        super().__init__()
        self.pi = pi
        self.v = v
        self.adv = adv
        self.n = n

    def forward(self, obs):
        action_distrib = self.pi(obs)
        v = self.v(obs)

        def evaluator(action):
            adv_mean = sum(self.adv((obs, action_distrib.sample()))
                           for _ in range(self.n)) / self.n
            return v + self.adv((obs, action)) - adv_mean

        return action_distrib, SingleActionValue(evaluator), v


def get_params_of_distribution(distrib):
    if isinstance(distrib, torch.distributions.Independent):
        return get_params_of_distribution(distrib.base_dist)
    if isinstance(distrib, torch.distributions.Categorical):
        return (distrib._param,)
    if isinstance(distrib, torch.distributions.Normal):
        return distrib.loc, distrib.scale
    raise NotImplementedError("{} is not supported by ACER".format(type(distrib)))


def deepcopy_distribution(distrib):
    """A copy of ``distrib`` whose tensors are detached leaves (a distribution whose
    tensors carry a graph cannot be deep-copied)."""
    D = torch.distributions
    if isinstance(distrib, D.Independent):
        return D.Independent(deepcopy_distribution(distrib.base_dist),
                             distrib.reinterpreted_batch_ndims)
    if isinstance(distrib, D.Categorical):
        return D.Categorical(logits=distrib.logits.clone().detach())
    if isinstance(distrib, D.Normal):
        return D.Normal(loc=distrib.loc.clone().detach(), scale=distrib.scale.clone().detach())
    raise NotImplementedError("{} is not supported by ACER".format(type(distrib)))


def compute_loss_with_kl_constraint(distrib, another_distrib, original_loss, delta):
    """Efficient TRPO: the loss whose gradient in the distribution's parameters is
    g - max(0, (k.g - delta) / k.k) k, with g = d original_loss and k = d(-KL).

    Returns (loss, KL(another_distrib || distrib) as a float)."""
    distrib_params = get_params_of_distribution(distrib)
    for param in distrib_params:
        assert param.shape[0] == 1
        assert param.requires_grad
    g = [grad[0] for grad in torch.autograd.grad([original_loss], distrib_params,
                                                 retain_graph=True)]
    kl = torch.distributions.kl_divergence(another_distrib, distrib)
    k = [grad[0] for grad in torch.autograd.grad([-kl], distrib_params, retain_graph=True)]
    kg_dot = sum(torch.dot(kp.flatten(), gp.flatten()) for kp, gp in zip(k, g))
    kk_dot = sum(torch.dot(kp.flatten(), kp.flatten()) for kp in k)
    k_factor = max(0, (kg_dot - delta) / kk_dot) if kk_dot > 0 else 0
    z = [gp - k_factor * kp for kp, gp in zip(k, g)]
    loss = 0
    for p, zp in zip(distrib_params, z):
        loss += (p * zp).sum()
    return loss.reshape(original_loss.shape), float(kl)


def _pinned_to(x, device):
    """Host array -> ``device`` without a synchronisation (a page-locked staging copy)."""
    t = torch.as_tensor(x)
    if device.type != "cuda":
        return t.to(device)
    return t.pin_memory().to(device, non_blocking=True)


class ACER(agent.AttributeSavingMixin, agent.AsyncAgent):
    """ACER (Actor-Critic with Experience Replay).

    Arguments as the reference's ``pfrl.agents.ACER``.  The models stay on the device
    of ``model``.  Statistics: average_value, average_entropy, average_kl.
    """

    process_idx = None
    saved_attributes = ("model", "optimizer")

    def __init__(self, model, optimizer, t_max, gamma, replay_buffer, beta=1e-2,
                 phi=lambda x: x, pi_loss_coef=1.0, Q_loss_coef=0.5, use_trust_region=True,
                 trust_region_alpha=0.99, trust_region_delta=1, truncation_threshold=10,
                 disable_online_update=False, n_times_replay=8, replay_start_size=10**4,
                 normalize_loss_by_steps=True, act_deterministically=False,
                 max_grad_norm=None, recurrent=False, use_Q_opc=False,
                 average_entropy_decay=0.999, average_value_decay=0.999,
                 average_kl_decay=0.999, logger=None):
        self.shared_model = model
        self.shared_average_model = copy.deepcopy(self.shared_model)
        self.model = copy.deepcopy(self.shared_model)
        self.optimizer = optimizer
        self.replay_buffer = replay_buffer
        self.t_max = t_max
        self.gamma = gamma
        self.beta = beta
        self.phi = phi
        self.pi_loss_coef = pi_loss_coef
        self.Q_loss_coef = Q_loss_coef
        self.normalize_loss_by_steps = normalize_loss_by_steps
        self.act_deterministically = act_deterministically
        self.max_grad_norm = max_grad_norm
        self.recurrent = recurrent
        self.use_trust_region = use_trust_region
        self.trust_region_alpha = trust_region_alpha
        self.truncation_threshold = truncation_threshold
        self.trust_region_delta = trust_region_delta
        self.disable_online_update = disable_online_update
        self.n_times_replay = n_times_replay
        self.use_Q_opc = use_Q_opc
        self.replay_start_size = replay_start_size
        self.average_value_decay = average_value_decay
        self.average_entropy_decay = average_entropy_decay
        self.average_kl_decay = average_kl_decay
        self.logger = logger if logger else getLogger(__name__)

        param = next(iter(model.parameters()), None)
        self.device = param.device if param is not None else torch.device("cpu")
        self.use_fused = True
        self.t = 0
        self.last_state = None
        self.last_action = None

        self.train_recurrent_states = None
        self.shared_recurrent_states = None
        self.test_recurrent_states = None

        self.average_value = 0
        self.average_entropy = 0
        self.average_kl = 0
        # the fused path's statistics: fp64 device averages of value, entropy and KL
        self._stats = None
        self._stat_rates = None

        self.init_history_data_for_online_update()

    def init_history_data_for_online_update(self):
        self.past_actions = {}
        self.past_rewards = {}
        self.past_values = {}
        self.past_action_distrib = {}
        self.past_action_values = {}
        self.past_avg_action_distrib = {}
        self.t_start = self.t

    def sync_parameters(self):
        copy_param.copy_param(target_link=self.model, source_link=self.shared_model)
        copy_param.soft_copy_param(target_link=self.shared_average_model,
                                   source_link=self.model, tau=1 - self.trust_region_alpha)

    def assert_shared_memory(self):
        agent.assert_shared_memory(self, ("model", "shared_model", "shared_average_model"))

    @property
    def shared_attributes(self):
        return ("shared_model", "shared_average_model", "optimizer")

    # ------------------------------------------------- reference formulation
    def compute_one_step_pi_loss(self, action, advantage, action_distrib, action_distrib_mu,
                                 action_value, v, avg_action_distrib):
        assert np.isscalar(advantage)
        assert np.isscalar(v)
        g_loss = compute_policy_gradient_loss(
            action=action, advantage=advantage, action_distrib=action_distrib,
            action_distrib_mu=action_distrib_mu, action_value=action_value, v=v,
            truncation_threshold=self.truncation_threshold)
        if self.use_trust_region:
            pi_loss, kl = compute_loss_with_kl_constraint(
                action_distrib, avg_action_distrib, g_loss, delta=self.trust_region_delta)
            self.average_kl += (1 - self.average_kl_decay) * (kl - self.average_kl)
        else:
            pi_loss = g_loss
        pi_loss -= self.beta * action_distrib.entropy()
        return pi_loss

    def compute_loss(self, t_start, t_stop, R, actions, rewards, values, action_values,
                     action_distribs, action_distribs_mu, avg_action_distribs):
        assert np.isscalar(R)
        pi_loss = 0
        Q_loss = 0
        Q_ret = R
        Q_opc = R
        discrete = isinstance(action_distribs[t_start], torch.distributions.Categorical)
        del R
        for i in reversed(range(t_start, t_stop)):
            r = rewards[i]
            v = values[i]
            action_distrib = action_distribs[i]
            action_distrib_mu = action_distribs_mu[i] if action_distribs_mu else None
            avg_action_distrib = avg_action_distribs[i]
            action_value = action_values[i]
            ba = torch.as_tensor(actions[i], device=self.device).unsqueeze(0)
            if action_distrib_mu is not None:
                rho = compute_importance(action_distrib, action_distrib_mu, ba)
            else:
                rho = 1
            Q_ret = r + self.gamma * Q_ret
            Q_opc = r + self.gamma * Q_opc
            assert np.isscalar(Q_ret)
            assert np.isscalar(Q_opc)
            advantage = (Q_opc if self.use_Q_opc else Q_ret) - float(v)
            pi_loss += self.compute_one_step_pi_loss(
                action=ba, advantage=advantage, action_distrib=action_distrib,
                action_distrib_mu=action_distrib_mu, action_value=action_value, v=float(v),
                avg_action_distrib=avg_action_distrib)
            Q = action_value.evaluate_actions(ba)
            assert Q.requires_grad, "Q must be backprop-able"
            Q_loss += nn.functional.mse_loss(torch.tensor(Q_ret, device=self.device), Q) / 2
            if not discrete:
                assert v.requires_grad, "v must be backprop-able"
                v_target = min(1, rho) * (Q_ret - float(Q)) + float(v)
                Q_loss += nn.functional.mse_loss(torch.tensor(v_target, device=self.device),
                                                 v) / 2
            if self.process_idx == 0:
                self.logger.debug("t:%s v:%s Q:%s Q_ret:%s Q_opc:%s", i, float(v), float(Q),
                                  Q_ret, Q_opc)
            c = min(1, rho) if discrete else min(1, rho ** (1 / ba.numel()))
            Q_ret = c * (Q_ret - float(Q)) + float(v)
            Q_opc = Q_opc - float(Q) + float(v)
        pi_loss *= self.pi_loss_coef
        Q_loss *= self.Q_loss_coef
        if self.normalize_loss_by_steps:
            pi_loss /= t_stop - t_start
            Q_loss /= t_stop - t_start
        if self.process_idx == 0:
            self.logger.debug("pi_loss:%s Q_loss:%s", float(pi_loss), float(Q_loss))
        return pi_loss + Q_loss.reshape(*pi_loss.shape)

    def update(self, t_start, t_stop, R, actions, rewards, values, action_values,
               action_distribs, action_distribs_mu, avg_action_distribs):
        assert np.isscalar(R)
        self.assert_shared_memory()
        total_loss = self.compute_loss(
            t_start=t_start, t_stop=t_stop, R=R, actions=actions, rewards=rewards,
            values=values, action_values=action_values, action_distribs=action_distribs,
            action_distribs_mu=action_distribs_mu, avg_action_distribs=avg_action_distribs)
        self.model.zero_grad()
        total_loss.squeeze().backward()
        self._apply_gradients()

    def _apply_gradients(self):
        if self.max_grad_norm is not None:
            clip_l2_grad_norm_(self.model.parameters(), self.max_grad_norm)
        copy_param.copy_grad(target_link=self.shared_model, source_link=self.model)
        self.optimizer.step()
        self.sync_parameters()

    def _forward(self, model, states, recurrent_state):
        if self.recurrent:
            return one_step_forward(model, states, recurrent_state)
        return model(states), None

    def update_from_replay(self):
        if self.replay_buffer is None:
            return
        if len(self.replay_buffer) < self.replay_start_size:
            return
        episodes = self.replay_buffer.sample_episodes(1, self.t_max)
        if self._fused_ok():
            # argument validation of the distributions would read the device
            with no_distribution_validation():
                done = self._update_from_replay_fused(episodes)
            if done:
                return
        episode = episodes[0]
        model_rs = shared_rs = None
        rewards, actions, action_distribs, action_distribs_mu = {}, {}, {}, {}
        avg_action_distribs, action_values, values = {}, {}, {}
        for t, transition in enumerate(episode):
            bs = batch_states([transition["state"]], self.device, self.phi)
            (action_distrib, action_value, v), model_rs = self._forward(self.model, bs,
                                                                        model_rs)
            with torch.no_grad():
                (avg_action_distrib, _, _), shared_rs = self._forward(
                    self.shared_average_model, bs, shared_rs)
            actions[t] = transition["action"]
            values[t] = v
            action_distribs[t] = action_distrib
            avg_action_distribs[t] = avg_action_distrib
            rewards[t] = transition["reward"]
            action_distribs_mu[t] = transition["mu"]
            action_values[t] = action_value
        last_transition = episode[-1]
        if last_transition["is_state_terminal"]:
            R = 0
        else:
            with torch.no_grad():
                last_s = batch_states([last_transition["next_state"]], self.device, self.phi)
                (_, _, last_v), _ = self._forward(self.model, last_s, model_rs)
            R = float(last_v)
        return self.update(R=R, t_start=0, t_stop=len(episode), rewards=rewards,
                           actions=actions, values=values, action_distribs=action_distribs,
                           action_distribs_mu=action_distribs_mu,
                           avg_action_distribs=avg_action_distribs, action_values=action_values)

    def update_on_policy(self, statevar):
        assert self.t_start < self.t
        if not self.disable_online_update:
            if self._fused_ok() and self._fused_distribs(
                    [self.past_action_distrib[i] for i in range(self.t_start, self.t)]):
                with no_distribution_validation():
                    self._update_on_policy_fused(statevar)
            else:
                if statevar is None:
                    R = 0
                else:
                    with torch.no_grad():
                        (_, _, v), _ = self._forward(self.model, statevar,
                                                     self.train_recurrent_states)
                    R = float(v)
                self.update(t_start=self.t_start, t_stop=self.t, R=R,
                            actions=self.past_actions, rewards=self.past_rewards,
                            values=self.past_values, action_values=self.past_action_values,
                            action_distribs=self.past_action_distrib, action_distribs_mu=None,
                            avg_action_distribs=self.past_avg_action_distrib)
        self.init_history_data_for_online_update()
        self.train_recurrent_states = detach_recurrent_state(self.train_recurrent_states)

    # ------------------------------------------------------------ the fused path
    def _fused_ok(self):
        return self.use_fused and self.device.type == "cuda"

    @staticmethod
    def _fused_distribs(distribs):
        """The kernel's case: fp32 Categorical policies on CUDA."""
        return all(type(d) is torch.distributions.Categorical and d._param.dtype == torch.float32
                   and d._param.is_cuda and d._param.dim() == 2 for d in distribs)

    def _kernel(self, z, q, avg_z, mu_z, actions, rewards, bootstrap, on_policy):
        if self.use_trust_region and self._stats is None:
            self._init_stats()
        return fused.loss_grads(
            z, q, actions, rewards, avg_z=avg_z, mu_z=None if on_policy else mu_z,
            bootstrap=bootstrap, gamma=self.gamma, truncation_threshold=self.truncation_threshold,
            use_trust_region=self.use_trust_region, delta=self.trust_region_delta,
            beta=self.beta, pi_loss_coef=self.pi_loss_coef, Q_loss_coef=self.Q_loss_coef,
            normalize_loss_by_steps=self.normalize_loss_by_steps, use_Q_opc=self.use_Q_opc,
            average_kl=self._stats[2:3] if self.use_trust_region else None,
            average_kl_decay=self.average_kl_decay)

    def _fused_backward(self, z, q, g_z, g_q):
        self.assert_shared_memory()
        self.model.zero_grad()
        torch.autograd.backward([z, q], [g_z, g_q])
        self._apply_gradients()

    def _replay_inputs(self, episodes):
        """(states [T(+1), ...], actions [T], rewards fp64 [T], mu logits [T, K], terminal)
        of the one sampled subsequence, on the device; None where the buffer cannot give
        them (a mu that is not an fp32 Categorical)."""
        from pfrl_b200.replay_buffers.episodic import DeviceEpisodes

        dev = self.device
        if isinstance(episodes, DeviceEpisodes):
            rbuf = episodes.buffer
            if (rbuf._mu_layout is None or rbuf._mu_layout[0] is not torch.distributions.Categorical
                    or rbuf._mu_layout[2] != torch.float32):
                return None
            terminal = bool(episodes.last_terminal[0])
            batch = rbuf._gather_sequences(episodes, 1.0, self.phi)
            states = batch["state"].data
            if not terminal:
                states = torch.cat([states, batch["next_state"].data[-1:]])
            actions = batch["action"].reshape(-1)
            rewards = rbuf._rewards_f64_device(episodes)
            mu = rbuf.mu_rows(episodes)
            return states, actions, rewards, mu, terminal
        episode = episodes[0]
        if not all(type(t["mu"]) is torch.distributions.Categorical for t in episode):
            return None
        terminal = bool(episode[-1]["is_state_terminal"])
        obs = [t["state"] for t in episode]
        if not terminal:
            obs.append(episode[-1]["next_state"])
        states = batch_states(obs, dev, self.phi)
        actions = _pinned_to(np.asarray([t["action"] for t in episode], dtype=np.int64), dev)
        rewards = _pinned_to(np.asarray([t["reward"] for t in episode], dtype=np.float64), dev)
        mu = torch.cat([t["mu"].logits.to(dev) for t in episode])
        return states, actions, rewards, mu, terminal

    def _update_from_replay_fused(self, episodes):
        """One replay update with no host synchronisation; False when the kernel does not
        cover the case (nothing done then)."""
        inputs = self._replay_inputs(episodes)
        if inputs is None:
            return False
        states, actions, rewards, mu, terminal = inputs
        T = rewards.shape[0]
        if self.recurrent:
            (distrib, action_value, v), _ = pack_and_forward(self.model, [states], None)
        else:
            distrib, action_value, v = self.model(states)
        if not self._fused_distribs([distrib]):
            return False
        with torch.no_grad():
            if self.recurrent:
                (avg, _, _), _ = pack_and_forward(self.shared_average_model, [states[:T]], None)
            else:
                avg, _, _ = self.shared_average_model(states[:T])
        z, q = distrib._param, action_value.q_values
        bootstrap = None if terminal else v[T:T + 1].detach()
        g_z, g_q = self._kernel(z[:T], q[:T], avg._param, mu, actions, rewards, bootstrap,
                                on_policy=False)
        self._fused_backward(z[:T], q[:T], g_z, g_q)
        return True

    def _update_on_policy_fused(self, statevar):
        steps = range(self.t_start, self.t)
        if statevar is None:
            bootstrap = None
        else:
            with torch.no_grad():
                (_, _, v), _ = self._forward(self.model, statevar, self.train_recurrent_states)
            bootstrap = v.reshape(1)
        z = torch.cat([self.past_action_distrib[i]._param for i in steps])
        q = torch.cat([self.past_action_values[i].q_values for i in steps])
        avg = torch.cat([self.past_avg_action_distrib[i]._param for i in steps])
        actions = torch.stack([torch.as_tensor(self.past_actions[i]).reshape(())
                               for i in steps])
        rewards = _pinned_to(np.asarray([self.past_rewards[i] for i in steps],
                                        dtype=np.float64), self.device)
        g_z, g_q = self._kernel(z, q, avg, None, actions, rewards, bootstrap, on_policy=True)
        self._fused_backward(z, q, g_z, g_q)

    def _init_stats(self):
        self._stats = _pinned_to(np.array([self.average_value, self.average_entropy,
                                           self.average_kl], dtype=np.float64), self.device)
        self._stat_rates = _pinned_to(np.array([1 - self.average_value_decay,
                                                1 - self.average_entropy_decay]), self.device)

    def _update_stats(self, v, action_distrib):
        if self._fused_ok() and self._fused_distribs([action_distrib]):
            if self._stats is None:
                self._init_stats()
            with torch.no_grad():
                x = torch.stack([v.reshape(()), action_distrib.entropy().reshape(())]).double()
                self._stats[:2] += self._stat_rates * (x - self._stats[:2])
            return
        self._sync_stats()
        self.average_value += (1 - self.average_value_decay) * (float(v) - self.average_value)
        self.average_entropy += (1 - self.average_entropy_decay) * (
            float(action_distrib.entropy()) - self.average_entropy)

    def _sync_stats(self):
        """Bring the fused path's device averages back to the host attributes."""
        if self._stats is not None:
            self.average_value, self.average_entropy, self.average_kl = self._stats.tolist()
            self._stats = None

    # ------------------------------------------------------------------ acting
    def act(self, obs):
        if self.training:
            return self._act_train(obs)
        return self._act_eval(obs)

    def observe(self, obs, reward, done, reset):
        if self.training:
            self._observe_train(obs, reward, done, reset)
        else:
            self._observe_eval(obs, reward, done, reset)

    def _act_train(self, obs):
        statevar = batch_states([obs], self.device, self.phi)
        (action_distrib, action_value, v), self.train_recurrent_states = self._forward(
            self.model, statevar, self.train_recurrent_states)
        self.past_action_values[self.t] = action_value
        action = action_distrib.sample()[0]
        self.past_values[self.t] = v
        self.past_action_distrib[self.t] = action_distrib
        with torch.no_grad():
            (avg_action_distrib, _, _), self.shared_recurrent_states = self._forward(
                self.shared_average_model, statevar, self.shared_recurrent_states)
        self.past_avg_action_distrib[self.t] = avg_action_distrib
        self.past_actions[self.t] = action
        self._update_stats(v, action_distrib)
        self.last_state = obs
        self.last_action = action.cpu().numpy()
        self.last_action_distrib = deepcopy_distribution(action_distrib)
        return self.last_action

    def _act_eval(self, obs):
        with torch.no_grad():
            statevar = batch_states([obs], self.device, self.phi)
            (action_distrib, _, _), self.test_recurrent_states = self._forward(
                self.model, statevar, self.test_recurrent_states)
            if self.act_deterministically:
                return mode_of_distribution(action_distrib).cpu().numpy()[0]
            return action_distrib.sample().cpu().numpy()[0]

    def _observe_train(self, state, reward, done, reset):
        assert self.last_state is not None
        assert self.last_action is not None
        if self.replay_buffer is not None:
            self.replay_buffer.append(state=self.last_state, action=self.last_action,
                                      reward=reward, next_state=state, is_state_terminal=done,
                                      mu=self.last_action_distrib)
            if done or reset:
                self.replay_buffer.stop_current_episode()
        self.t += 1
        self.past_rewards[self.t - 1] = reward
        if self.process_idx == 0:
            self.logger.debug("t:%s r:%s a:%s", self.t, reward, self.last_action)
        if self.t - self.t_start == self.t_max or done or reset:
            statevar = None if done else batch_states([state], self.device, self.phi)
            self.update_on_policy(statevar)
            for _ in range(self.n_times_replay):
                self.update_from_replay()
        if done or reset:
            self.train_recurrent_states = None
            self.shared_recurrent_states = None
        self.last_state = None
        self.last_action = None
        self.last_action_distrib = None

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
            ("average_kl", self.average_kl),
        ]
