"""Soft Actor-Critic (arXiv:1812.05905) on the device replay path.

Public surface = pfrl/agents/soft_actor_critic.py:40-385.  Changes: the
uniform replay lives in HBM (indices drawn on the host with the reference's
``sample_n_k`` stream, minibatch gathered by the fused kernel), the
temperature stays a device tensor (the reference converts it to a Python
float -- a D2H sync -- twice per update), statistics are device ring buffers
read lazily, and the two Polyak updates are multi-tensor launches.
"""
import copy
from logging import getLogger

import numpy as np
import torch
from torch import nn
from torch.nn import functional as F

from pfrl_b200.agent import AttributeSavingMixin, BatchAgent
from pfrl_b200.agents._graph import CapturedStep
from pfrl_b200.agents.dqn import _DeviceRing
from pfrl_b200.replay_buffer import ReplayUpdater, batch_experiences
from pfrl_b200.utils import clip_l2_grad_norm_
from pfrl_b200.utils.batch_states import batch_states
from pfrl_b200.utils.modes import evaluating
from pfrl_b200.utils.copy_param import synchronize_parameters
from pfrl_b200.utils.mode_of_distribution import mode_of_distribution  # NOQA (re-exported)


class TemperatureHolder(nn.Module):
    """Learnable log-temperature (soft_actor_critic.py:24-37)."""

    def __init__(self, initial_log_temperature=0):
        super().__init__()
        self.log_temperature = nn.Parameter(
            torch.tensor(initial_log_temperature, dtype=torch.float32))

    def forward(self):
        return torch.exp(self.log_temperature)


class SoftActorCritic(AttributeSavingMixin, BatchAgent):
    saved_attributes = (
        "policy", "q_func1", "q_func2", "target_q_func1", "target_q_func2",
        "policy_optimizer", "q_func1_optimizer", "q_func2_optimizer",
        "temperature_holder", "temperature_optimizer",
    )

    def __init__(self, policy, q_func1, q_func2, policy_optimizer, q_func1_optimizer,
                 q_func2_optimizer, replay_buffer, gamma, gpu=None, replay_start_size=10000,
                 minibatch_size=100, update_interval=1, phi=lambda x: x, soft_update_tau=5e-3,
                 max_grad_norm=None, logger=getLogger(__name__), batch_states=batch_states,
                 burnin_action_func=None, initial_temperature=1.0, entropy_target=None,
                 temperature_optimizer_lr=None, act_deterministically=True, grad_sync=None,
                 cuda_graph=False):
        self.policy = policy
        self.q_func1 = q_func1
        self.q_func2 = q_func2
        if gpu is not None and gpu >= 0:
            assert torch.cuda.is_available()
            self.device = torch.device("cuda:{}".format(gpu))
            self.policy.to(self.device)
            self.q_func1.to(self.device)
            self.q_func2.to(self.device)
        else:
            self.device = torch.device("cpu")
        self.replay_buffer = replay_buffer
        self.gamma = gamma
        self.gpu = gpu
        self.phi = phi
        self.soft_update_tau = soft_update_tau
        self.logger = logger
        self.policy_optimizer = policy_optimizer
        self.q_func1_optimizer = q_func1_optimizer
        self.q_func2_optimizer = q_func2_optimizer
        self.replay_updater = ReplayUpdater(
            replay_buffer=replay_buffer, update_func=self.update, batchsize=minibatch_size,
            n_times_update=1, replay_start_size=replay_start_size,
            update_interval=update_interval, episodic_update=False)
        self.replay_updater.agent = self
        self.max_grad_norm = max_grad_norm
        self.batch_states = batch_states
        self.burnin_action_func = burnin_action_func
        self.initial_temperature = initial_temperature
        self.entropy_target = entropy_target
        self.grad_sync = grad_sync
        if self.entropy_target is not None:
            self.temperature_holder = TemperatureHolder(
                initial_log_temperature=np.log(initial_temperature))
            if temperature_optimizer_lr is not None:
                self.temperature_optimizer = torch.optim.Adam(
                    self.temperature_holder.parameters(), lr=temperature_optimizer_lr)
            else:
                self.temperature_optimizer = torch.optim.Adam(self.temperature_holder.parameters())
            if gpu is not None and gpu >= 0:
                self.temperature_holder.to(self.device)
        else:
            self.temperature_holder = None
            self.temperature_optimizer = None
        self.act_deterministically = act_deterministically
        self.t = 0
        self.target_q_func1 = copy.deepcopy(self.q_func1).eval().requires_grad_(False)
        self.target_q_func2 = copy.deepcopy(self.q_func2).eval().requires_grad_(False)
        self.q1_record = _DeviceRing(1000)
        self.q2_record = _DeviceRing(1000)
        self.entropy_record = _DeviceRing(1000)
        self.q_func1_loss_record = _DeviceRing(100)
        self.q_func2_loss_record = _DeviceRing(100)
        self.n_policy_updates = 0
        # Optional: replay the whole update (5 small networks, 4 optimizers, 2
        # Polyak steps: ~300 launches of tiny kernels) as ONE CUDA graph.
        self._graph = None
        if cuda_graph and self.device.type == "cuda" and grad_sync is None:
            self._graph = CapturedStep(3, (policy_optimizer, q_func1_optimizer,
                                           q_func2_optimizer, self.temperature_optimizer))

    @property
    def temperature(self):
        """Python float (reads the device); the update path uses
        ``_temperature_tensor`` instead to stay asynchronous."""
        if self.entropy_target is None:
            return self.initial_temperature
        with torch.no_grad():
            return float(self.temperature_holder())

    def _temperature_tensor(self):
        if self.entropy_target is None:
            return self.initial_temperature
        return self.temperature_holder().detach()

    def sync_target_network(self):
        synchronize_parameters(src=self.q_func1, dst=self.target_q_func1, method="soft",
                               tau=self.soft_update_tau)
        synchronize_parameters(src=self.q_func2, dst=self.target_q_func2, method="soft",
                               tau=self.soft_update_tau)

    def _step(self, optimizer, module, loss):
        optimizer.zero_grad()
        loss.backward()
        if self.grad_sync is not None:
            self.grad_sync(module)
        if self.max_grad_norm is not None:
            clip_l2_grad_norm_(module.parameters(), self.max_grad_norm)
        optimizer.step()

    def update_q_func(self, batch):
        """Twin-Q regression on the entropy-regularised target
        (soft_actor_critic.py:214-262)."""
        next_state = batch["next_state"]
        with torch.no_grad(), evaluating(self.policy), evaluating(self.target_q_func1), \
                evaluating(self.target_q_func2):
            next_distrib = self.policy(next_state)
            # rsample() under no_grad draws the same law as sample() but skips
            # torch.normal(mean, std)'s host-side `std.min() >= 0` check (a D2H
            # sync per update in the reference, and illegal in graph capture)
            next_actions = next_distrib.rsample()
            next_log_prob = next_distrib.log_prob(next_actions)
            next_q1 = self.target_q_func1((next_state, next_actions))
            next_q2 = self.target_q_func2((next_state, next_actions))
            assert next_q1.shape == next_log_prob[..., None].shape
            if next_q1.is_cuda and next_q1.dtype == torch.float32:
                # min, entropy term, (1 - terminal), discount and reward in one launch
                # (b2rl_sac_target), rounded like the eager expression below
                from pfrl_b200.ops.sac import sac_target

                target_q = sac_target(batch["reward"], batch["discount"],
                                      batch["is_state_terminal"], next_q1, next_q2,
                                      next_log_prob, self._temperature_tensor())
            else:
                next_q = torch.min(next_q1, next_q2)
                entropy_term = self._temperature_tensor() * next_log_prob[..., None]
                target_q = batch["reward"] + batch["discount"] * (
                    1.0 - batch["is_state_terminal"]) * torch.flatten(next_q - entropy_term)
        state, actions = batch["state"], batch["action"]
        predict_q1 = torch.flatten(self.q_func1((state, actions)))
        predict_q2 = torch.flatten(self.q_func2((state, actions)))
        loss1 = 0.5 * F.mse_loss(target_q, predict_q1)
        loss2 = 0.5 * F.mse_loss(target_q, predict_q2)
        self._step(self.q_func1_optimizer, self.q_func1, loss1)
        self._step(self.q_func2_optimizer, self.q_func2, loss2)
        return predict_q1.detach(), predict_q2.detach(), loss1.detach(), loss2.detach()

    def update_temperature(self, log_prob):
        assert not log_prob.requires_grad
        loss = -torch.mean(self.temperature_holder() * (log_prob + self.entropy_target))
        self._step(self.temperature_optimizer, self.temperature_holder, loss)

    def update_policy_and_temperature(self, batch):
        """Reparameterised policy improvement (soft_actor_critic.py:273-308)."""
        state = batch["state"]
        action_distrib = self.policy(state)
        actions = action_distrib.rsample()
        log_prob = action_distrib.log_prob(actions)
        q = torch.min(self.q_func1((state, actions)), self.q_func2((state, actions)))
        entropy_term = self._temperature_tensor() * log_prob[..., None]
        assert q.shape == entropy_term.shape
        loss = torch.mean(entropy_term - q)
        self._step(self.policy_optimizer, self.policy, loss)
        if self.entropy_target is not None:
            self.update_temperature(log_prob.detach())
        with torch.no_grad():
            try:
                return action_distrib.entropy().detach()
            except NotImplementedError:
                return -log_prob.detach()

    def _update_core(self, batch):
        """The device work of one update; returns the tensors the statistics
        are read from (no Python-side state is touched, no host sync)."""
        q1, q2, l1, l2 = self.update_q_func(batch)
        entropy = self.update_policy_and_temperature(batch)
        self.sync_target_network()
        return q1, q2, l1, l2, entropy

    _GRAPH_KEYS = ("state", "next_state", "action", "reward", "discount", "is_state_terminal")

    def update(self, experiences, errors_out=None):
        batch = batch_experiences(experiences, self.device, self.phi, self.gamma)
        if self._graph is not None:
            self._graph.load((self.soft_update_tau, self.max_grad_norm, self.entropy_target,
                              self.initial_temperature if self.entropy_target is None else None),
                             {k: batch[k] for k in self._GRAPH_KEYS})
            q1, q2, l1, l2, entropy = self._graph.run(self._update_core)
        else:
            q1, q2, l1, l2, entropy = self._update_core(batch)
        self.n_policy_updates += 1
        self.q1_record.extend(q1)
        self.q2_record.extend(q2)
        self.q_func1_loss_record.append(l1)
        self.q_func2_loss_record.append(l2)
        self.entropy_record.extend(entropy)

    def batch_select_greedy_action(self, batch_obs, deterministic=False):
        with torch.no_grad(), evaluating(self.policy):
            policy_out = self.policy(self.batch_states(batch_obs, self.device, self.phi))
            if deterministic:
                return mode_of_distribution(policy_out).cpu().numpy()
            return policy_out.sample().cpu().numpy()

    def batch_act(self, batch_obs):
        if not self.training:
            return self.batch_select_greedy_action(
                batch_obs, deterministic=self.act_deterministically)
        if self.burnin_action_func is not None and self.n_policy_updates == 0:
            batch_action = [self.burnin_action_func() for _ in range(len(batch_obs))]
        else:
            batch_action = self.batch_select_greedy_action(batch_obs)
        self.batch_last_obs = list(batch_obs)
        self.batch_last_action = list(batch_action)
        return batch_action

    def batch_observe(self, batch_obs, batch_reward, batch_done, batch_reset):
        if not self.training:
            return
        for i in range(len(batch_obs)):
            self.t += 1
            if self.batch_last_obs[i] is not None:
                assert self.batch_last_action[i] is not None
                self.replay_buffer.append(
                    state=self.batch_last_obs[i], action=self.batch_last_action[i],
                    reward=batch_reward[i], next_state=batch_obs[i], next_action=None,
                    is_state_terminal=batch_done[i], env_id=i)
                if batch_reset[i] or batch_done[i]:
                    self.batch_last_obs[i] = None
                    self.batch_last_action[i] = None
                    self.replay_buffer.stop_current_episode(env_id=i)
            self.replay_updater.update_if_necessary(self.t)

    def get_statistics(self):
        return [
            ("average_q1", self.q1_record.mean()),
            ("average_q2", self.q2_record.mean()),
            ("average_q_func1_loss", self.q_func1_loss_record.mean()),
            ("average_q_func2_loss", self.q_func2_loss_record.mean()),
            ("n_updates", self.n_policy_updates),
            ("average_entropy", self.entropy_record.mean()),
            ("temperature", self.temperature),
        ]
