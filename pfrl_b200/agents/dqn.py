"""DQN and its update loop on the device replay path.

Public surface = pfrl/agents/dqn.py (DQN :150-819): constructor arguments,
``act/observe/batch_act/batch_observe``, ``update``, ``save/load`` (model,
target_model, optimizer), ``get_statistics`` names.  What changes is where
the work happens:

  reference (dqn.py:316-365)                 here
  -----------------------------------------  ---------------------------------
  batch_experiences: Python lists -> H2D     fused gather kernel out of HBM
  TD errors -> .cpu().numpy() -> Python      stay on the device; fused
    list -> update_errors (Python trees)       clip/+eps/pow + tree write-back
  loss / q statistics: D2H every update      device ring buffers, read lazily
                                               in get_statistics()

With ``recurrent=True`` (DQN and DoubleDQN) the model is a recurrent module
(``pfrl_b200.nn.RecurrentSequential`` ...) and updates come from episodes
(``update_from_episodes``).  Acting keeps the batched recurrent states on the
device, and the transitions handed to the device ``EpisodicReplayBuffer`` carry
detached device slices of them, so states never leave the GPU; a host buffer
gets numpy copies, as in the reference (dqn.py:533-545).  The actor-learner
mode is out of scope (SURVEY.md section 2).
"""
import collections
import copy
from logging import getLogger

import numpy as np
import torch
import torch.nn.functional as F

from pfrl_b200 import _lib, agent
from pfrl_b200.action_value import QuadraticActionValue
from pfrl_b200.agents import _advantage
from pfrl_b200.agents._graph import CapturedStep
from pfrl_b200.ops import losses as fused
from pfrl_b200.replay_buffer import (
    AbstractEpisodicReplayBuffer, ReplayUpdater, batch_experiences, batch_recurrent_experiences,
)
from pfrl_b200.replay_buffers import PrioritizedReplayBuffer
from pfrl_b200.replay_buffers.episodic import DeviceEpisodes, EpisodicReplayBuffer
from pfrl_b200.utils import clip_l2_grad_norm_
from pfrl_b200.utils.batch_states import batch_states
from pfrl_b200.utils.modes import evaluating
from pfrl_b200.utils.copy_param import synchronize_parameters
from pfrl_b200.utils.recurrent import (
    get_recurrent_state_at, mask_recurrent_state_at, one_step_forward, pack_and_forward,
    recurrent_state_as_numpy,
)


def compute_value_loss(y, t, clip_delta=True, batch_accumulator="mean"):
    """Huber (delta=1) or 0.5*MSE between predictions and targets,
    mean/sum over the batch (pfrl/agents/dqn.py:44-67)."""
    assert batch_accumulator in ("mean", "sum")
    y = y.reshape(-1, 1)
    t = t.reshape(-1, 1)
    if clip_delta:
        return F.smooth_l1_loss(y, t, reduction=batch_accumulator)
    return F.mse_loss(y, t, reduction=batch_accumulator) / 2


def compute_weighted_value_loss(y, t, weights, clip_delta=True, batch_accumulator="mean"):
    """sum_i w_i * l_i (divided by the batch size for "mean")
    (pfrl/agents/dqn.py:70-104)."""
    assert batch_accumulator in ("mean", "sum")
    y = y.reshape(-1, 1)
    t = t.reshape(-1, 1)
    if clip_delta:
        losses = F.smooth_l1_loss(y, t, reduction="none")
    else:
        losses = F.mse_loss(y, t, reduction="none") / 2
    loss_sum = torch.sum(losses.reshape(-1) * weights.to(losses.device))
    return loss_sum / y.shape[0] if batch_accumulator == "mean" else loss_sum


def _batch_reset_recurrent_states_when_episodes_end(batch_done, batch_reset, recurrent_states):
    """Zero the recurrent state of every env whose episode ended (done or reset)."""
    ended = [i for i, (done, reset) in enumerate(zip(batch_done, batch_reset)) if done or reset]
    if ended:
        return mask_recurrent_state_at(recurrent_states, ended)
    return recurrent_states


def make_target_model_as_copy(model):
    target = copy.deepcopy(model)

    def flatten(mod):
        # cuDNN RNN weights must be made contiguous again after a deep copy
        if isinstance(mod, torch.nn.RNNBase):
            mod.flatten_parameters()

    target.apply(flatten)
    target.eval()
    return target


class _DeviceRing:
    """Last ``maxlen`` scalars kept on the device; mean() syncs lazily."""

    def __init__(self, maxlen):
        self.maxlen = maxlen
        self.buf = None
        self.count = 0
        self.host = collections.deque(maxlen=maxlen)

    def extend(self, values):
        if not isinstance(values, torch.Tensor) or not values.is_cuda:
            vals = values.detach().cpu().numpy().ravel() if isinstance(values, torch.Tensor) \
                else np.asarray(values).ravel()
            self.host.extend(vals.tolist())
            return
        v = values.detach().reshape(-1).float()
        if self.buf is None:
            self.buf = torch.zeros(self.maxlen, device=v.device)
        if v.numel() >= self.maxlen:
            # the whole window is replaced: restart the ring at slot 0 so that the next
            # write overwrites the OLDEST value (count stays a multiple of maxlen)
            self.buf.copy_(v[-self.maxlen:])
            self.count = (self.count // self.maxlen + 2) * self.maxlen
            return
        pos = self.count % self.maxlen
        first = min(v.numel(), self.maxlen - pos)
        self.buf[pos:pos + first] = v[:first]
        if first < v.numel():
            self.buf[:v.numel() - first] = v[first:]
        self.count += v.numel()

    def append(self, value):
        if isinstance(value, torch.Tensor):
            self.extend(value.reshape(1))
        else:
            self.host.append(float(value))

    def mean(self):
        if self.buf is not None and self.count > 0:
            n = min(self.count, self.maxlen)
            return float(self.buf[:n].mean().item()) if self.count < self.maxlen \
                else float(self.buf.mean().item())
        return float(np.mean(self.host)) if self.host else np.nan

    def __len__(self):
        return min(self.count, self.maxlen) if self.buf is not None else len(self.host)


class DQN(agent.AttributeSavingMixin, agent.BatchAgent):
    """Deep Q-Network (same arguments as pfrl.agents.DQN, dqn.py:181-206)."""

    saved_attributes = ("model", "target_model", "optimizer")

    # recurrent=True is implemented by DQN and DoubleDQN; the subclasses that
    # change the target (distributional, quantile, advantage learning) refuse it
    _recurrent_supported = True

    def __init__(self, q_function, optimizer, replay_buffer, gamma, explorer, gpu=None,
                 replay_start_size=50000, minibatch_size=32, update_interval=1,
                 target_update_interval=10000, clip_delta=True, phi=lambda x: x,
                 target_update_method="hard", soft_update_tau=1e-2, n_times_update=1,
                 batch_accumulator="mean", episodic_update_len=None,
                 logger=getLogger(__name__), batch_states=batch_states, recurrent=False,
                 max_grad_norm=None, grad_sync=None, cuda_graph=False):
        if recurrent and not self._recurrent_supported:
            raise NotImplementedError(
                "recurrent=True is not implemented for %s" % type(self).__name__)
        if recurrent and (cuda_graph or grad_sync is not None):
            raise ValueError("recurrent=True cannot be combined with cuda_graph or grad_sync: "
                             "the packed shapes change with every update")
        self.model = q_function
        if gpu is not None and gpu >= 0:
            assert torch.cuda.is_available()
            self.device = torch.device("cuda:{}".format(gpu))
            self.model.to(self.device)
        else:
            self.device = torch.device("cpu")
        self.replay_buffer = replay_buffer
        self.optimizer = optimizer
        self.gamma = gamma
        self.explorer = explorer
        self.gpu = gpu
        self.target_update_interval = target_update_interval
        self.clip_delta = clip_delta
        self.phi = phi
        self.target_update_method = target_update_method
        self.soft_update_tau = soft_update_tau
        self.batch_accumulator = batch_accumulator
        assert batch_accumulator in ("mean", "sum")
        self.logger = logger
        self.batch_states = batch_states
        self.recurrent = bool(recurrent)
        if self.recurrent:
            assert isinstance(replay_buffer, AbstractEpisodicReplayBuffer)
            if isinstance(replay_buffer, EpisodicReplayBuffer) and minibatch_size > _lib.SEQ_MAX_B:
                raise ValueError("the device EpisodicReplayBuffer gathers at most %d sequences "
                                 "per update (minibatch_size=%d)" % (_lib.SEQ_MAX_B,
                                                                     minibatch_size))
        self.replay_updater = ReplayUpdater(
            replay_buffer=replay_buffer,
            update_func=self.update_from_episodes if self.recurrent else self.update,
            batchsize=minibatch_size,
            episodic_update=self.recurrent, episodic_update_len=episodic_update_len,
            n_times_update=n_times_update, replay_start_size=replay_start_size,
            update_interval=update_interval)
        self.replay_updater.agent = self
        self.minibatch_size = minibatch_size
        self.episodic_update_len = episodic_update_len
        self.replay_start_size = replay_start_size
        self.update_interval = update_interval
        self.max_grad_norm = max_grad_norm
        # optional hook called between backward() and optimizer.step() with the
        # model; the data-parallel launcher installs the NCCL gradient all-reduce
        self.grad_sync = grad_sync
        assert target_update_interval % update_interval == 0, \
            "target_update_interval should be a multiple of update_interval"
        self.t = 0
        self.optim_t = 0
        self._cumulative_steps = 0
        self.target_model = make_target_model_as_copy(self.model)
        self.q_record = _DeviceRing(1000)
        self.loss_record = _DeviceRing(100)
        self.batch_last_obs = []
        self.batch_last_action = []
        self.train_recurrent_states = None
        self.train_prev_recurrent_states = None
        self.test_recurrent_states = None
        # Optional: replay forward(s) + fused loss + backward + clip + optimizer
        # step as ONE CUDA graph (pays off when the minibatch is small and the
        # update is launch-bound, e.g. Nature-DQN at batch 32).
        # With a grad_sync hook (data-parallel ranks) the update is TWO graphs around the
        # eagerly issued all-reduce: forward + loss + backward + bucket packing, then
        # unpacking + clipping + optimizer step.  The acting forward is a third graph.
        self._graph = self._step_graph = self._act_graph = None
        if cuda_graph and self.device.type == "cuda" and (grad_sync is None or all(
                hasattr(grad_sync, a) for a in ("pack", "reduce", "unpack"))):
            self._graph = CapturedStep(3, (optimizer,))
            if grad_sync is not None:
                self._step_graph = CapturedStep(3, share_pool_with=self._graph)
            self._act_graph = CapturedStep(3)
        if (self.replay_buffer.capacity is not None
                and self.replay_buffer.capacity < self.replay_updater.replay_start_size):
            raise ValueError("Replay start size cannot exceed replay buffer capacity.")

    @property
    def cumulative_steps(self):
        return self._cumulative_steps

    def sync_target_network(self):
        synchronize_parameters(src=self.model, dst=self.target_model,
                               method=self.target_update_method, tau=self.soft_update_tau)

    # ------------------------------------------------------------------ update
    def update(self, experiences, errors_out=None):
        """One gradient step from sampled experiences (dqn.py:316-365)."""
        exp_batch = batch_experiences(experiences, device=self.device, phi=self.phi,
                                      gamma=self.gamma, batch_states=self.batch_states)
        if "weights" in exp_batch:
            has_weight = True
        else:
            has_weight = (not hasattr(experiences, "batch")) and "weight" in experiences[0][0]
            if has_weight:
                exp_batch["weights"] = torch.tensor(
                    [e[0]["weight"] for e in experiences], device=self.device,
                    dtype=torch.float32)
        want_list = errors_out is not None
        want_errors = has_weight or want_list
        if self._graph is not None:
            loss, delta, q = self._learn_graphed(exp_batch, want_errors)
        else:
            loss, delta, q = self._learn(exp_batch, want_errors)
        if want_list:
            del errors_out[:]
            errors_out.extend(delta.detach().cpu().numpy())
        if has_weight:
            assert isinstance(self.replay_buffer, PrioritizedReplayBuffer)
            # device tensor in, device trees updated: no host round trip.  (The
            # reference calls update_errors between forward and backward,
            # dqn.py:356; the priorities only depend on the forward pass.)
            self.replay_buffer.update_errors(delta.detach())
        self.loss_record.append(loss)
        self.q_record.extend(q)
        self.optim_t += 1

    def _learn(self, exp_batch, want_errors):
        """loss -> backward -> (all-reduce) -> clip -> optimizer step; touches no
        Python-side state, so it can be captured in a CUDA graph.  Returns the loss,
        |y - t| (or None) and the Q-values of the batch."""
        out = self._backward(exp_batch, want_errors)
        if self.grad_sync is not None:
            self.grad_sync(self.model)
        self._step()
        return out

    def _backward(self, exp_batch, want_errors):
        loss, delta = self._compute_loss(exp_batch, want_errors=want_errors)
        self.optimizer.zero_grad()
        loss.backward()
        return loss.detach(), delta, self._last_q

    def _step(self):
        if self.max_grad_norm is not None:
            clip_l2_grad_norm_(self.model.parameters(), self.max_grad_norm)
        self.optimizer.step()

    def _learn_graphed(self, exp_batch, want_errors):
        self._graph.load((self.clip_delta, self.batch_accumulator, self.max_grad_norm,
                          want_errors), exp_batch)
        if self.grad_sync is None:
            return self._graph.run(lambda b: self._learn(b, want_errors))

        def backward_and_pack(b):
            out = self._backward(b, want_errors)
            self.grad_sync.pack(self.model)
            return out

        out = self._graph.run(backward_and_pack)
        self.grad_sync.reduce(self.model)  # NCCL, eager, between the two graphs
        self._step_graph.load(self._graph.key, {})

        def unpack_and_step(_):
            self.grad_sync.unpack(self.model)
            self._step()

        self._step_graph.run(unpack_and_step)
        return out

    def _forward(self, model, exp_batch, key):
        """Q-values of exp_batch[key] ("state" / "next_state"); a recurrent model
        runs over the packed sequences from the batch's matching initial state."""
        if not self.recurrent:
            return model(exp_batch[key])
        rs = exp_batch["recurrent_state" if key == "state" else "next_recurrent_state"]
        qout, _ = pack_and_forward(model, exp_batch[key], rs)
        return qout

    def _next_q(self, exp_batch):
        """Value of the next state used in the target: max_a Q_target(s', a)."""
        return self._forward(self.target_model, exp_batch, "next_state").max

    def _compute_target_values(self, exp_batch):
        return exp_batch["reward"] + exp_batch["discount"] * (
            1.0 - exp_batch["is_state_terminal"]) * self._next_q(exp_batch)

    def _compute_y_and_t(self, exp_batch):
        batch_size = exp_batch["reward"].shape[0]
        qout = self._forward(self.model, exp_batch, "state")
        batch_q = torch.reshape(qout.evaluate_actions(exp_batch["action"]), (batch_size, 1))
        with torch.no_grad():
            batch_q_target = torch.reshape(self._compute_target_values(exp_batch), (batch_size, 1))
        return batch_q, batch_q_target

    use_fused_loss = True

    # the target the NAF kernel computes for this class (agents._advantage.fused_mode)
    _fused_mode = "dqn"

    def _compute_loss(self, exp_batch, want_errors=False):
        """Returns (loss, per-sample |y - t| or None); dqn.py:432-470."""
        if self.use_fused_loss and exp_batch["reward"].is_cuda:
            # one fused kernel: gather Q(s)[a], TD target, |y - t|, Huber / MSE,
            # importance weights and the deterministic batch reduction
            qout = self._forward(self.model, exp_batch, "state")
            if isinstance(qout, QuadraticActionValue):
                return self._compute_naf_loss(exp_batch, qout, want_errors)
            with torch.no_grad():
                next_q = self._next_q(exp_batch)
            loss, delta, y, _ = fused.td_loss(
                qout.q_values, exp_batch["action"], next_q, exp_batch["reward"],
                exp_batch["discount"], exp_batch["is_state_terminal"],
                exp_batch.get("weights"), clip_delta=self.clip_delta,
                mean=self.batch_accumulator == "mean")
            self._last_q = y.detach()
            return loss, delta
        return self._compute_loss_torch(exp_batch, want_errors)

    def _compute_naf_loss(self, exp_batch, qout, want_errors):
        """Loss of a continuous-action (NAF) Q-function whose output at s is ``qout``: the NAF
        kernel where it computes this class's target from fp32 values, else the reference's
        target in torch (after the same forward at s)."""
        mode = _advantage.fused_mode(self)
        if (mode in ("dqn", "double_dqn") and not self.recurrent
                and _advantage.naf_kernel_dtypes(qout)):
            return _advantage.naf_loss(self, exp_batch, qout, mode)
        batch_size = exp_batch["reward"].shape[0]
        y = torch.reshape(qout.evaluate_actions(exp_batch["action"]), (batch_size, 1))
        with torch.no_grad():
            t = torch.reshape(self._compute_target_values(exp_batch), (batch_size, 1))
        return self._value_loss(y, t, exp_batch, want_errors)

    def _compute_loss_torch(self, exp_batch, want_errors=False):
        """The reference's formulation: _compute_y_and_t, then the value loss."""
        y, t = self._compute_y_and_t(exp_batch)
        return self._value_loss(y, t, exp_batch, want_errors)

    def _value_loss(self, y, t, exp_batch, want_errors):
        self._last_q = y.detach()
        delta = None
        if want_errors:
            delta = torch.abs(y.detach() - t)
            if delta.ndim == 2:
                delta = torch.sum(delta, dim=1)
        if "weights" in exp_batch:
            loss = compute_weighted_value_loss(
                y, t, exp_batch["weights"], clip_delta=self.clip_delta,
                batch_accumulator=self.batch_accumulator)
        else:
            loss = compute_value_loss(y, t, clip_delta=self.clip_delta,
                                      batch_accumulator=self.batch_accumulator)
        return loss, delta

    # --------------------------------------------------------------- act/observe
    def _evaluate_model(self, batch_obs):
        batch_xs = self.batch_states(batch_obs, self.device, self.phi)
        if not self.recurrent:
            return self.model(batch_xs)
        if self.training:
            self.train_prev_recurrent_states = self.train_recurrent_states
            batch_av, self.train_recurrent_states = one_step_forward(
                self.model, batch_xs, self.train_recurrent_states)
        else:
            batch_av, self.test_recurrent_states = one_step_forward(
                self.model, batch_xs, self.test_recurrent_states)
        return batch_av

    def _greedy_graphed(self, batch_obs):
        """Acting forward (a few dozen tiny launches at num_envs images) replayed as one CUDA
        graph: observations are copied into a static buffer, the action values and greedy
        actions come back in static ones.  None when the observations are not one tensor."""
        x = self.batch_states(batch_obs, self.device, self.phi)
        if not isinstance(x, torch.Tensor):
            return None
        self._act_graph.load((), {"x": x})

        def greedy(b):
            av = self.model(b["x"])
            return av, av.greedy_actions

        return self._act_graph.run(greedy)

    def batch_act(self, batch_obs):
        with torch.no_grad(), evaluating(self.model):
            graphed = None
            if self._act_graph is not None and type(self)._evaluate_model is DQN._evaluate_model:
                graphed = self._greedy_graphed(batch_obs)
            if graphed is not None:
                batch_av, greedy = graphed
                batch_argmax = greedy.cpu().numpy()
            else:
                batch_av = self._evaluate_model(batch_obs)
                batch_argmax = batch_av.greedy_actions.detach().cpu().numpy()
        if not self.training:
            return batch_argmax
        batch_action = [
            self.explorer.select_action(self.t, lambda: batch_argmax[i],
                                        action_value=batch_av[i:i + 1])
            for i in range(len(batch_obs))
        ]
        self.batch_last_obs = list(batch_obs)
        self.batch_last_action = list(batch_action)
        return batch_action

    def _batch_observe_train(self, batch_obs, batch_reward, batch_done, batch_reset):
        # per-env interleaving of append and update exactly as dqn.py:509-549
        # (device-resident envs hand out CUDA tensors: one D2H copy per vector step instead of
        # a stream synchronisation per environment and field)
        if isinstance(batch_reward, torch.Tensor):
            batch_reward = batch_reward.detach().cpu().numpy()
        if isinstance(batch_done, torch.Tensor):
            batch_done = batch_done.detach().cpu().numpy()
        if isinstance(batch_reset, torch.Tensor):
            batch_reset = batch_reset.detach().cpu().numpy()
        for i in range(len(batch_obs)):
            self.t += 1
            self._cumulative_steps += 1
            if self.t % self.target_update_interval == 0:
                self.sync_target_network()
            if self.batch_last_obs[i] is not None:
                assert self.batch_last_action[i] is not None
                extra = {}
                if self.recurrent:
                    extra = dict(
                        recurrent_state=self._stored_state(self.train_prev_recurrent_states, i),
                        next_recurrent_state=self._stored_state(self.train_recurrent_states, i))
                self.replay_buffer.append(
                    state=self.batch_last_obs[i], action=self.batch_last_action[i],
                    reward=batch_reward[i], next_state=batch_obs[i], next_action=None,
                    is_state_terminal=batch_done[i], env_id=i, **extra)
                if batch_reset[i] or batch_done[i]:
                    self.batch_last_obs[i] = None
                    self.batch_last_action[i] = None
                    self.replay_buffer.stop_current_episode(env_id=i)
            self.replay_updater.update_if_necessary(self.t)
        if self.recurrent:
            self.train_prev_recurrent_states = None
            self.train_recurrent_states = _batch_reset_recurrent_states_when_episodes_end(
                batch_done, batch_reset, self.train_recurrent_states)

    def _stored_state(self, batch_state, i):
        """State of env i as a transition stores it: a detached device slice for the
        device episodic buffer (no device-to-host copy), numpy otherwise."""
        s = get_recurrent_state_at(batch_state, i, detach=True)
        if isinstance(self.replay_buffer, EpisodicReplayBuffer):
            return s
        return recurrent_state_as_numpy(s)

    def batch_observe(self, batch_obs, batch_reward, batch_done, batch_reset):
        if self.training:
            return self._batch_observe_train(batch_obs, batch_reward, batch_done, batch_reset)
        if self.recurrent:
            if isinstance(batch_done, torch.Tensor):
                batch_done = batch_done.detach().cpu().numpy()
            if isinstance(batch_reset, torch.Tensor):
                batch_reset = batch_reset.detach().cpu().numpy()
            self.test_recurrent_states = _batch_reset_recurrent_states_when_episodes_end(
                batch_done, batch_reset, self.test_recurrent_states)
        return None

    # ------------------------------------------------------------------- misc
    def stop_episode(self):
        """Forget the evaluation recurrent state (dqn.py:790-792)."""
        if self.recurrent:
            self.test_recurrent_states = None

    def update_from_episodes(self, episodes, errors_out=None):
        """One gradient step from sampled episodes (dqn.py:367-386): sort them by
        length (stable, longest first), batch them packed, loss, optimizer step.
        The loss is the scalar TD loss over the packed rows (the fused kernel on
        CUDA, as in ``update``)."""
        assert errors_out is None, "Recurrent DQN does not support PrioritizedBuffer"
        if isinstance(episodes, DeviceEpisodes):
            episodes = episodes.sorted_by_length()
        else:
            episodes = sorted(episodes, key=len, reverse=True)
        exp_batch = batch_recurrent_experiences(
            episodes, device=self.device, phi=self.phi, gamma=self.gamma,
            batch_states=self.batch_states)
        loss, _, q = self._learn(exp_batch, want_errors=False)
        self.loss_record.append(loss)
        self.q_record.extend(q)
        self.optim_t += 1

    def save_snapshot(self, dirname):
        self.save(dirname)
        torch.save(self.t, "{}/t.pt".format(dirname))
        torch.save(self.optim_t, "{}/optim_t.pt".format(dirname))
        torch.save(self._cumulative_steps, "{}/_cumulative_steps.pt".format(dirname))
        self.replay_buffer.save("{}/replay_buffer.pkl".format(dirname))

    def load_snapshot(self, dirname):
        self.load(dirname)
        self.t = torch.load("{}/t.pt".format(dirname))
        self.optim_t = torch.load("{}/optim_t.pt".format(dirname))
        self._cumulative_steps = torch.load("{}/_cumulative_steps.pt".format(dirname))
        self.replay_buffer.load("{}/replay_buffer.pkl".format(dirname))

    def get_statistics(self):
        return [
            ("average_q", self.q_record.mean()),
            ("average_loss", self.loss_record.mean()),
            ("cumulative_steps", self.cumulative_steps),
            ("n_updates", self.optim_t),
            ("rlen", len(self.replay_buffer)),
        ]
