"""TD3 (arXiv:1802.09477) and DDPG on the device replay path.

SURVEY section 8f item 1: both reuse the uniform HBM replay + fused gather of
SAC unchanged; only the update differs.  Public surface as in the reference
(pfrl/agents/td3.py:27-330, pfrl/agents/ddpg.py:26-300): constructor
arguments, saved_attributes, statistics names.  Statistics stay on the device
(no per-update ``.item()`` / ``.cpu()`` as in td3.py:217-220,237) and the
Polyak steps are multi-tensor launches.

On CUDA with fp32 critics (``use_fused``, on by default) the critic update's tail runs in
csrc/sac.cu: TD3's default target-policy smoothing (``k_td3_smooth``, on the reference's
``torch.randn_like`` draw) and, in one launch, the target, both critics' ``mse_loss`` and
their gradients (``k_td3_critic_loss``).  The forwards keep the reference's order, so the
random stream is the reference's.  The fused update runs with the distributions' argument
checks off (each is a host sync), so an update on the device replay path does not wait for
the device.  ``cuda_graph=True`` replays each update as a CUDA graph: TD3 has two, the
critic-only update and the critic + policy + Polyak update, in one memory pool; DDPG has
one, critic and actor (its target sync stays in ``_on_step``).
"""
import contextlib
import copy
from logging import getLogger

import torch
from torch import nn
from torch.nn import functional as F

from pfrl_b200.agent import AttributeSavingMixin, BatchAgent
from pfrl_b200.agents._graph import CapturedStep
from pfrl_b200.agents.dqn import _DeviceRing
from pfrl_b200.ops import sac as sac_ops
from pfrl_b200.replay_buffer import ReplayUpdater, batch_experiences
from pfrl_b200.utils import clip_l2_grad_norm_
from pfrl_b200.utils.batch_states import batch_states
from pfrl_b200.utils.copy_param import synchronize_parameters
from pfrl_b200.utils.modes import evaluating, no_distribution_validation


def default_target_policy_smoothing_func(batch_action):
    """Clipped Gaussian noise on the target action (td3.py:20-24)."""
    noise = torch.clamp(0.2 * torch.randn_like(batch_action), -0.5, 0.5)
    return torch.clamp(batch_action + noise, -1, 1)


class _OffPolicyActorCritic(AttributeSavingMixin, BatchAgent):
    """Shared act / observe loop of the deterministic actor-critic agents:
    explorer (or burn-in) actions, per-env append to the replay buffer,
    ReplayUpdater schedule -- identical in td3.py:279-320 and ddpg.py:236-290."""

    def _init_common(self, policy, replay_buffer, gamma, explorer, gpu, phi, batch_states_fn,
                     burnin_action_func, logger):
        self.device = torch.device("cuda:{}".format(gpu)) if gpu is not None and gpu >= 0 \
            else torch.device("cpu")
        if self.device.type == "cuda":
            assert torch.cuda.is_available()
        self.replay_buffer = replay_buffer
        self.gamma = gamma
        self.explorer = explorer
        self.gpu = gpu
        self.phi = phi
        self.batch_states = batch_states_fn
        self.burnin_action_func = burnin_action_func
        self.logger = logger
        self.t = 0
        self.batch_last_obs = []
        self.batch_last_action = []

    def _n_policy_updates(self):
        raise NotImplementedError

    def batch_select_onpolicy_action(self, batch_obs):
        with torch.no_grad(), evaluating(self.policy):
            batch_xs = self.batch_states(batch_obs, self.device, self.phi)
            return list(self.policy(batch_xs).sample().cpu().numpy())

    def batch_act(self, batch_obs):
        if not self.training:
            return self.batch_select_onpolicy_action(batch_obs)
        if self.burnin_action_func is not None and self._n_policy_updates() == 0:
            batch_action = [self.burnin_action_func() for _ in range(len(batch_obs))]
        else:
            greedy = self.batch_select_onpolicy_action(batch_obs)
            batch_action = [self.explorer.select_action(self.t, lambda: greedy[i])
                            for i in range(len(greedy))]
        self.batch_last_obs = list(batch_obs)
        self.batch_last_action = list(batch_action)
        return batch_action

    def batch_observe(self, batch_obs, batch_reward, batch_done, batch_reset):
        if not self.training:
            return
        for i in range(len(batch_obs)):
            self.t += 1
            self._on_step()
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

    def _on_step(self):
        pass

    # the batch entries a graphed update reads
    _GRAPH_KEYS = ("state", "next_state", "action", "reward", "discount", "is_state_terminal")

    def _fused(self, *tensors):
        return self.use_fused and all(t.is_cuda and t.dtype == torch.float32 for t in tensors)

    def _update_context(self):
        """No distribution argument checks (a host sync each) in a fused update."""
        fused = self.use_fused and self.device.type == "cuda"
        return no_distribution_validation() if fused else contextlib.nullcontext()

    def _opt_step(self, optimizer, module, loss, max_grad_norm=None):
        optimizer.zero_grad()
        loss.backward()
        if max_grad_norm is not None:
            clip_l2_grad_norm_(module.parameters(), max_grad_norm)
        optimizer.step()


class TD3(_OffPolicyActorCritic):
    use_fused = True
    saved_attributes = (
        "policy", "q_func1", "q_func2", "target_policy", "target_q_func1", "target_q_func2",
        "policy_optimizer", "q_func1_optimizer", "q_func2_optimizer",
    )

    def __init__(self, policy, q_func1, q_func2, policy_optimizer, q_func1_optimizer,
                 q_func2_optimizer, replay_buffer, gamma, explorer, gpu=None,
                 replay_start_size=10000, minibatch_size=100, update_interval=1,
                 phi=lambda x: x, soft_update_tau=5e-3, n_times_update=1, max_grad_norm=None,
                 logger=getLogger(__name__), batch_states=batch_states, burnin_action_func=None,
                 policy_update_delay=2,
                 target_policy_smoothing_func=default_target_policy_smoothing_func,
                 cuda_graph=False):
        self._init_common(policy, replay_buffer, gamma, explorer, gpu, phi, batch_states,
                          burnin_action_func, logger)
        self.policy, self.q_func1, self.q_func2 = policy, q_func1, q_func2
        for m in (policy, q_func1, q_func2):
            m.to(self.device)
        self.soft_update_tau = soft_update_tau
        self.policy_optimizer = policy_optimizer
        self.q_func1_optimizer = q_func1_optimizer
        self.q_func2_optimizer = q_func2_optimizer
        self.replay_updater = ReplayUpdater(
            replay_buffer=replay_buffer, update_func=self.update, batchsize=minibatch_size,
            n_times_update=1, replay_start_size=replay_start_size,
            update_interval=update_interval, episodic_update=False)
        self.replay_updater.agent = self
        self.max_grad_norm = max_grad_norm
        self.policy_update_delay = policy_update_delay
        self.target_policy_smoothing_func = target_policy_smoothing_func
        self.policy_n_updates = 0
        self.q_func_n_updates = 0
        self.target_policy = copy.deepcopy(policy).eval().requires_grad_(False)
        self.target_q_func1 = copy.deepcopy(q_func1).eval().requires_grad_(False)
        self.target_q_func2 = copy.deepcopy(q_func2).eval().requires_grad_(False)
        self.q1_record = _DeviceRing(1000)
        self.q2_record = _DeviceRing(1000)
        self.q_func1_loss_record = _DeviceRing(100)
        self.q_func2_loss_record = _DeviceRing(100)
        self.policy_loss_record = _DeviceRing(100)
        # cuda_graph=True: the critic-only update and the critic + policy + Polyak update,
        # captured into one memory pool
        self._q_graph = self._full_graph = None
        if cuda_graph and self.device.type == "cuda":
            pool = torch.cuda.graph_pool_handle()
            self._q_graph = CapturedStep(3, (q_func1_optimizer, q_func2_optimizer), pool=pool)
            self._full_graph = CapturedStep(
                3, (q_func1_optimizer, q_func2_optimizer, policy_optimizer), pool=pool)

    def _n_policy_updates(self):
        return self.policy_n_updates

    def sync_target_network(self):
        for src, dst in ((self.policy, self.target_policy), (self.q_func1, self.target_q_func1),
                         (self.q_func2, self.target_q_func2)):
            synchronize_parameters(src=src, dst=dst, method="soft", tau=self.soft_update_tau)

    def _smooth(self, next_actions):
        if (self.target_policy_smoothing_func is default_target_policy_smoothing_func
                and self._fused(next_actions)):
            return sac_ops.td3_smooth(next_actions, torch.randn_like(next_actions))
        return self.target_policy_smoothing_func(next_actions)

    def _q_step(self, batch):
        """The device work of update_q_func; returns the predictions and the losses."""
        next_state = batch["next_state"]
        with torch.no_grad(), evaluating(self.target_policy), evaluating(self.target_q_func1), \
                evaluating(self.target_q_func2):
            next_actions = self._smooth(self.target_policy(next_state).sample())
            next_q1 = self.target_q_func1((next_state, next_actions))
            next_q2 = self.target_q_func2((next_state, next_actions))
        state, actions = batch["state"], batch["action"]
        predict_q1 = torch.flatten(self.q_func1((state, actions)))
        predict_q2 = torch.flatten(self.q_func2((state, actions)))
        if self._fused(next_q1, next_q2, predict_q1, predict_q2):
            _, loss1, loss2 = sac_ops.critic_loss(
                batch["reward"], batch["discount"], batch["is_state_terminal"], next_q1, next_q2,
                predict_q1, predict_q2)
        else:
            with torch.no_grad():
                next_q = torch.min(next_q1, next_q2)
                target_q = batch["reward"] + batch["discount"] * (
                    1.0 - batch["is_state_terminal"]) * torch.flatten(next_q)
            loss1 = F.mse_loss(target_q, predict_q1)
            loss2 = F.mse_loss(target_q, predict_q2)
        self._opt_step(self.q_func1_optimizer, self.q_func1, loss1, self.max_grad_norm)
        self._opt_step(self.q_func2_optimizer, self.q_func2, loss2, self.max_grad_norm)
        return predict_q1.detach(), predict_q2.detach(), loss1.detach(), loss2.detach()

    def _record_q_step(self, q1, q2, loss1, loss2):
        self.q1_record.extend(q1)
        self.q2_record.extend(q2)
        self.q_func1_loss_record.append(loss1)
        self.q_func2_loss_record.append(loss2)
        self.q_func_n_updates += 1

    def update_q_func(self, batch):
        """Clipped double-Q regression with target policy smoothing (td3.py:181-236)."""
        self._record_q_step(*self._q_step(batch))

    def _policy_step(self, batch):
        state = batch["state"]
        q = self.q_func1((state, self.policy(state).rsample()))
        loss = -torch.mean(q)
        self._opt_step(self.policy_optimizer, self.policy, loss, self.max_grad_norm)
        return loss.detach()

    def _record_policy_step(self, loss):
        self.policy_loss_record.append(loss)
        self.policy_n_updates += 1

    def update_policy(self, batch):
        self._record_policy_step(self._policy_step(batch))

    def _graphed_update(self, batch):
        policy = (self.q_func_n_updates + 1) % self.policy_update_delay == 0
        step = self._full_graph if policy else self._q_graph
        step.load((self.soft_update_tau, self.max_grad_norm, self.policy_update_delay,
                   self.target_policy_smoothing_func, self.use_fused),
                  {k: batch[k] for k in self._GRAPH_KEYS})

        def core(b):
            out = self._q_step(b)
            if policy:
                out += (self._policy_step(b),)
                self.sync_target_network()
            return out

        out = step.run(core)
        self._record_q_step(*out[:4])
        if policy:
            self._record_policy_step(out[4])

    def update(self, experiences, errors_out=None):
        batch = batch_experiences(experiences, self.device, self.phi, self.gamma)
        with self._update_context():
            if self._q_graph is not None:
                self._graphed_update(batch)
                return
            self.update_q_func(batch)
            if self.q_func_n_updates % self.policy_update_delay == 0:
                self.update_policy(batch)
                self.sync_target_network()

    def get_statistics(self):
        return [
            ("average_q1", self.q1_record.mean()),
            ("average_q2", self.q2_record.mean()),
            ("average_q_func1_loss", self.q_func1_loss_record.mean()),
            ("average_q_func2_loss", self.q_func2_loss_record.mean()),
            ("average_policy_loss", self.policy_loss_record.mean()),
            ("policy_n_updates", self.policy_n_updates),
            ("q_func_n_updates", self.q_func_n_updates),
        ]


class DDPG(_OffPolicyActorCritic):
    use_fused = True
    saved_attributes = ("model", "target_model", "actor_optimizer", "critic_optimizer")

    def __init__(self, policy, q_func, actor_optimizer, critic_optimizer, replay_buffer, gamma,
                 explorer, gpu=None, replay_start_size=50000, minibatch_size=32,
                 update_interval=1, target_update_interval=10000, phi=lambda x: x,
                 target_update_method="hard", soft_update_tau=1e-2, n_times_update=1,
                 recurrent=False, episodic_update_len=None, logger=getLogger(__name__),
                 batch_states=batch_states, burnin_action_func=None, cuda_graph=False):
        assert not recurrent, "recurrent=True is not implemented"
        self._init_common(policy, replay_buffer, gamma, explorer, gpu, phi, batch_states,
                          burnin_action_func, logger)
        self.model = nn.ModuleList([policy, q_func]).to(self.device)
        self.target_update_interval = target_update_interval
        self.target_update_method = target_update_method
        self.soft_update_tau = soft_update_tau
        self.actor_optimizer = actor_optimizer
        self.critic_optimizer = critic_optimizer
        self.replay_updater = ReplayUpdater(
            replay_buffer=replay_buffer, update_func=self.update, batchsize=minibatch_size,
            episodic_update=False, episodic_update_len=episodic_update_len,
            n_times_update=n_times_update, replay_start_size=replay_start_size,
            update_interval=update_interval)
        self.replay_updater.agent = self
        self.target_model = copy.deepcopy(self.model)
        self.target_model.eval()
        self.q_record = _DeviceRing(1000)
        self.actor_loss_record = _DeviceRing(100)
        self.critic_loss_record = _DeviceRing(100)
        self.n_updates = 0
        self.policy, self.q_function = self.model
        self.target_policy, self.target_q_function = self.target_model
        self.sync_target_network()
        # cuda_graph=True: the critic and actor steps as one graph
        self._graph = None
        if cuda_graph and self.device.type == "cuda":
            self._graph = CapturedStep(3, (critic_optimizer, actor_optimizer))

    def _n_policy_updates(self):
        return self.n_updates

    def _on_step(self):
        if self.t % self.target_update_interval == 0:  # ddpg.py:269-270
            self.sync_target_network()

    def sync_target_network(self):
        synchronize_parameters(src=self.model, dst=self.target_model,
                               method=self.target_update_method, tau=self.soft_update_tau)

    def _critic_loss(self, batch):
        n = len(batch["reward"])
        with torch.no_grad():
            next_state = batch["next_state"]
            next_q = self.target_q_function((next_state, self.target_policy(next_state).sample()))
        predict_q = self.q_function((batch["state"], batch["action"])).reshape((n,))
        if self._fused(next_q, predict_q):
            return sac_ops.critic_loss(batch["reward"], self.gamma, batch["is_state_terminal"],
                                       next_q, None, predict_q, None)[1]
        with torch.no_grad():
            target_q = batch["reward"] + self.gamma * (
                1.0 - batch["is_state_terminal"]) * next_q.reshape((n,))
        return F.mse_loss(target_q, predict_q)

    def compute_critic_loss(self, batch):
        """1-step TD regression; note gamma, not the n-step discount (ddpg.py:150-173)."""
        loss = self._critic_loss(batch)
        self.critic_loss_record.append(loss.detach())
        return loss

    def _actor_loss(self, batch):
        state = batch["state"]
        q = self.q_function((state, self.policy(state).rsample()))
        return -q.mean(), q

    def compute_actor_loss(self, batch):
        loss, q = self._actor_loss(batch)
        self.q_record.extend(q)
        self.actor_loss_record.append(loss.detach())
        return loss

    def _graph_step(self, batch):
        self.critic_optimizer.zero_grad()
        critic_loss = self._critic_loss(batch)
        critic_loss.backward()
        self.critic_optimizer.step()
        self.actor_optimizer.zero_grad()
        actor_loss, q = self._actor_loss(batch)
        actor_loss.backward()
        self.actor_optimizer.step()
        return critic_loss.detach(), actor_loss.detach(), q.detach()

    def update(self, experiences, errors_out=None):
        batch = batch_experiences(experiences, self.device, self.phi, self.gamma)
        with self._update_context():
            if self._graph is not None:
                self._graph.load((self.gamma, self.use_fused),
                                 {k: batch[k] for k in self._GRAPH_KEYS})
                critic_loss, actor_loss, q = self._graph.run(self._graph_step)
                self.critic_loss_record.append(critic_loss)
                self.q_record.extend(q)
                self.actor_loss_record.append(actor_loss)
            else:
                self.critic_optimizer.zero_grad()
                self.compute_critic_loss(batch).backward()
                self.critic_optimizer.step()
                self.actor_optimizer.zero_grad()
                self.compute_actor_loss(batch).backward()
                self.actor_optimizer.step()
        self.n_updates += 1

    def get_statistics(self):
        return [
            ("average_q", self.q_record.mean()),
            ("average_actor_loss", self.actor_loss_record.mean()),
            ("average_critic_loss", self.critic_loss_record.mean()),
            ("n_updates", self.n_updates),
        ]
