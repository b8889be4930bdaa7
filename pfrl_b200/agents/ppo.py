"""Proximal Policy Optimization on a device-resident rollout.

Public surface = pfrl/agents/ppo.py:260-817 (constructor arguments,
act/observe, statistics names, saved_attributes).  The reference keeps the
rollout as Python lists of transition dicts, writes V(s), V(s'), log pi back
into them one float at a time and runs GAE as a Python loop per episode
(:36-53, :110-142); every minibatch rebuilds tensors from dict lists
(:488-511) and pulls two losses to the host (:662-663).

Here the rollout is a time-major set of device tensors [T, E, ...]; the
dataset is built by two batched forwards and ONE fused GAE kernel (segmented
reverse scan + advantage moments), minibatches are index gathers, and the
clipped-surrogate / value / entropy loss is one fused forward+backward kernel.
Episode segmentation (cut at done OR reset OR the flush of unfinished episodes
at update time, ppo.py:450-458,786-789) and the dataset order (episode
completion order, which fixes what ``random.sample`` draws) follow the
reference, so a seeded run visits the same minibatches.

With ``recurrent=True`` the model is a recurrent module (``nn.Recurrent``,
``RecurrentSequential``, ``RecurrentBranched``, ``nn.LSTM`` ...) and the update
follows ppo.py:56-107,157-180,534-631: acting advances the batched train / test
states on the device and every vector step appends the flattened states before
and after the step (``[E, 2, D]``) to a state ring, so stored states never leave
the GPU.  At update time the episodes are light spans ``(env, t0, length)``
over the rollout; the dataset pass packs whole episodes (``k_rollout_seq_gather``,
csrc/rollout.cu: observations, actions and both first states in one launch),
runs two forwards, scatters log pi, V and V' back to ``[T, E]`` and runs the same
fused GAE.  Each epoch shuffles the span list in place and cuts it into
minibatches of exactly ``minibatch_size`` transitions (the last span of a
minibatch may be split; its tail starts from its own stored state); each
minibatch is one pack launch, ``pack_and_forward`` and the fused loss.

The module also has the reference's list-of-dicts helpers (``_make_dataset``,
``_make_dataset_recurrent``, ``_limit_sequence_length`` ...), which work on
transition dicts as the reference's tests build them.
"""
import itertools
import random

import numpy as np
import torch
import torch.nn.functional as F
from torch.nn.utils.rnn import PackedSequence

from pfrl_b200 import agent
from pfrl_b200.agents._graph import CapturedStep
from pfrl_b200.agents.dqn import _DeviceRing
from pfrl_b200.agents.soft_actor_critic import mode_of_distribution
from pfrl_b200.ops import ppo as fused
from pfrl_b200.ops import rollout
from pfrl_b200.utils.batch_states import batch_states
from pfrl_b200.utils.modes import evaluating
from pfrl_b200.utils.recurrent import (
    concatenate_recurrent_states, flatten_sequences_time_first, mask_recurrent_state_at,
    one_step_forward, pack_and_forward,
)


def _elementwise_clip(x, x_min, x_max):
    return torch.min(torch.max(x, x_min), x_max)


def _yield_minibatch_indices(order, minibatch_size, num_epochs):
    """Index version of ppo.py:247-257: reshuffle the whole dataset with
    ``random.sample`` whenever the pool runs short, serve from its tail."""
    assert order
    n_total = len(order)
    pool = []
    served = 0
    while served < n_total * num_epochs:
        while len(pool) < minibatch_size:
            pool = random.sample(order, k=n_total) + pool
        yield pool[-minibatch_size:]
        served += minibatch_size
        pool = pool[:-minibatch_size]


_yield_minibatches = _yield_minibatch_indices  # the reference's name (works on any list)


# ---------------------------------------------------------------------------------------
# Sequences.  The agent runs these on ``_Span``s; the reference's tests run them on lists
# of transition dicts.  Both support len() and slicing, which is all they use.

def _limit_sequence_length(sequences, max_len):
    """Cut every sequence into consecutive pieces of at most ``max_len`` items, in
    order (ppo.py:145-154)."""
    assert max_len > 0
    out = []
    for seq in sequences:
        start = 0
        while len(seq) - start > max_len:
            out.append(seq[start:start + max_len])
            start += max_len
        out.append(seq[start:] if start else seq)
    return out


def _yield_subset_of_sequences_with_fixed_number_of_items(sequences, n_items):
    """Serve the sequences in order as minibatches of exactly ``n_items`` items
    (ppo.py:157-180).  The sequence that overflows a minibatch is split: its head
    ends the minibatch and its tail is served next.  A remainder shorter than
    ``n_items`` is dropped."""
    assert n_items > 0
    pending = list(reversed(sequences))  # next sequence at the end
    while pending:
        subset, count = [], 0
        while pending and count < n_items:
            subset.append(pending.pop())
            count += len(subset[-1])
        excess = count - n_items
        if excess > 0:
            last = subset[-1]
            subset[-1] = last[:len(last) - excess]
            pending.append(last[len(last) - excess:])
        if count >= n_items:
            yield subset


class _Span:
    """Steps ``t0 .. t0 + length - 1`` of env ``env`` of the rollout: a sequence
    as ``_limit_sequence_length`` and the minibatch split see it."""
    __slots__ = ("env", "t0", "length")

    def __init__(self, env, t0, length):
        self.env, self.t0, self.length = env, t0, length

    def __len__(self):
        return self.length

    def __getitem__(self, item):
        start, stop, step = item.indices(self.length)
        assert step == 1
        return _Span(self.env, self.t0 + start, max(0, stop - start))

    def first_slot(self, E):
        return self.t0 * E + self.env

    def __repr__(self):
        return "_Span(env=%d, t0=%d, length=%d)" % (self.env, self.t0, self.length)


def _state_leaves(recurrent_state):
    """The tensors of a batched state in order, and its nesting (to rebuild it)."""
    if recurrent_state is None:
        return [], None
    if isinstance(recurrent_state, torch.Tensor):
        return [recurrent_state], "leaf"
    leaves, nest = [], []
    for s in recurrent_state:
        sub, sub_nest = _state_leaves(s)
        leaves.extend(sub)
        nest.append(sub_nest)
    return leaves, tuple(nest)


def _state_from_leaves(nest, leaves):
    it = iter(leaves)

    def build(n):
        if n is None:
            return None
        if n == "leaf":
            return next(it)
        return tuple(build(c) for c in n)

    return build(nest)


# ---------------------------------------------------------------------------------------
# The reference's list-of-dicts dataset helpers (ppo.py:36-243).  Transitions are dicts
# with state, action, reward, next_state, nonterminal (and recurrent_state,
# next_recurrent_state); these add log_prob, v_pred, next_v_pred, adv and v_teacher.

def _add_advantage_and_value_target_to_episode(episode, gamma, lambd):
    adv = 0.0
    for tr in episode[::-1]:
        delta = tr["reward"] + gamma * tr["nonterminal"] * tr["next_v_pred"] - tr["v_pred"]
        adv = delta + gamma * lambd * adv
        tr["adv"] = adv
        tr["v_teacher"] = adv + tr["v_pred"]


def _add_advantage_and_value_target_to_episodes(episodes, gamma, lambd):
    for episode in episodes:
        _add_advantage_and_value_target_to_episode(episode, gamma, lambd)


def _normalized(states, obs_normalizer):
    return obs_normalizer(states, update=False) if obs_normalizer else states


def _add_log_prob_and_value_to_episodes(episodes, model, phi, batch_states, obs_normalizer,
                                        device):
    flat = list(itertools.chain.from_iterable(episodes))
    s = _normalized(batch_states([tr["state"] for tr in flat], device, phi), obs_normalizer)
    ns = _normalized(batch_states([tr["next_state"] for tr in flat], device, phi), obs_normalizer)
    with torch.no_grad(), evaluating(model):
        distribs, v = model(s)
        _, next_v = model(ns)
        actions = torch.tensor([tr["action"] for tr in flat], device=device)
        log_probs = distribs.log_prob(actions).cpu().numpy()
        v, next_v = v.cpu().numpy().ravel(), next_v.cpu().numpy().ravel()
    # Python floats, so that the advantages are fp64 as in the recurrent helper (NumPy 2
    # would keep fp32 scalars fp32 in the GAE recurrence; NumPy 1 promoted them to fp64)
    for tr, lp, vi, nvi in zip(flat, log_probs.tolist(), v.tolist(), next_v.tolist()):
        tr["log_prob"], tr["v_pred"], tr["next_v_pred"] = lp, vi, nvi


def _add_log_prob_and_value_to_episodes_recurrent(episodes, model, phi, batch_states,
                                                  obs_normalizer, device):
    by_len = sorted(episodes, key=len, reverse=True)  # pack_sequence keeps this order
    seqs = [_normalized(batch_states([tr["state"] for tr in ep], device, phi), obs_normalizer)
            for ep in by_len]
    next_seqs = [_normalized(batch_states([tr["next_state"] for tr in ep], device, phi),
                             obs_normalizer) for ep in by_len]
    flat = flatten_sequences_time_first(by_len)
    with torch.no_grad(), evaluating(model):
        rs = concatenate_recurrent_states([ep[0]["recurrent_state"] for ep in by_len])
        next_rs = concatenate_recurrent_states([ep[0]["next_recurrent_state"] for ep in by_len])
        (distribs, v), _ = pack_and_forward(model, seqs, rs)
        (_, next_v), _ = pack_and_forward(model, next_seqs, next_rs)
        actions = torch.tensor([tr["action"] for tr in flat], device=device)
        log_probs = distribs.log_prob(actions).cpu().numpy()
        v, next_v = v.cpu().numpy().ravel(), next_v.cpu().numpy().ravel()
    for tr, lp, vi, nvi in zip(flat, log_probs.tolist(), v.tolist(), next_v.tolist()):
        tr["log_prob"], tr["v_pred"], tr["next_v_pred"] = lp, vi, nvi


def _make_dataset(episodes, model, phi, batch_states, obs_normalizer, gamma, lambd, device):
    """Flat list of the episodes' transitions with log_prob, values and advantages."""
    _add_log_prob_and_value_to_episodes(episodes, model, phi, batch_states, obs_normalizer,
                                        device)
    _add_advantage_and_value_target_to_episodes(episodes, gamma, lambd)
    return list(itertools.chain.from_iterable(episodes))


def _make_dataset_recurrent(episodes, model, phi, batch_states, obs_normalizer, gamma, lambd,
                            max_recurrent_sequence_len, device):
    """The episodes (cut to ``max_recurrent_sequence_len``) with log_prob, values and
    advantages added to their transitions."""
    _add_log_prob_and_value_to_episodes_recurrent(episodes, model, phi, batch_states,
                                                  obs_normalizer, device)
    _add_advantage_and_value_target_to_episodes(episodes, gamma, lambd)
    if max_recurrent_sequence_len is None:
        return list(episodes)
    return _limit_sequence_length(episodes, max_recurrent_sequence_len)


def _compute_explained_variance(transitions):
    """1 - Var[v_teacher - v_pred] / Var[v_teacher], NaN when Var[v_teacher] = 0."""
    teacher = np.array([tr["v_teacher"] for tr in transitions])
    pred = np.array([tr["v_pred"] for tr in transitions])
    var = np.var(teacher)
    if var == 0:
        return np.nan
    return float(1 - np.var(teacher - pred) / var)


class _DeviceRollout:
    """The non-recurrent device rollout shared by PPO and TRPO: per vector step the raw
    states, actions, next states, rewards, nonterminal and episode-cut flags, the finished
    episodes in completion order, and the dataset pass (two forwards of ``self.model``,
    the fused GAE).  The agent provides ``model``, ``obs_normalizer``, ``gamma``,
    ``lambd``, ``use_fused`` and ``device``."""

    def _rollout_clear(self, E=None):
        self._states, self._next_states, self._actions = [], [], []
        self._rewards, self._nonterminal, self._cut = [], [], []
        self._segments = []     # finished episodes: (env, t_start, t_end) in completion order
        self._seg_start = None if E is None else [0] * E  # per env: first step of its episode

    def _record_act(self, raw, action, num_envs):
        self._cur_state = raw
        self._cur_action = action
        if self._seg_start is None:
            self._seg_start = [0] * num_envs

    def _record_observe(self, batch_obs, batch_reward, batch_done, batch_reset):
        """Append the step acted on last; returns the number of steps in the rollout."""
        assert self._cur_state is not None
        next_raw = self.batch_states(batch_obs, self.device, self.phi)
        done = np.asarray(batch_done, dtype=bool)
        end = np.logical_or(done, np.asarray(batch_reset, dtype=bool))
        t = len(self._rewards)
        self._states.append(self._cur_state)
        self._actions.append(self._cur_action)
        self._next_states.append(next_raw)
        self._rewards.append(np.asarray(batch_reward, dtype=np.float32))
        self._nonterminal.append((~done).astype(np.float32))
        self._cut.append(end.astype(np.uint8))
        for i in np.nonzero(end)[0]:  # episode completion order = env order within a step
            self._segments.append((int(i), self._seg_start[i], t))
            self._seg_start[i] = t + 1
        self._cur_state = None
        self._cur_action = None
        return t + 1

    def _dataset_order(self, T, E):
        """Flat indices t*E + e in the order of the reference's dataset list:
        finished episodes in completion order, then (flush, ppo.py:450-458)
        the unfinished ones by env index."""
        segs = list(self._segments)
        for e in range(E):
            if self._seg_start[e] <= T - 1:
                segs.append((e, self._seg_start[e], T - 1))
        order = list(itertools.chain.from_iterable(
            (range(s * E + e, (t_end + 1) * E + e, E)) for e, s, t_end in segs))
        assert len(order) == T * E
        return order

    def _rollout_dataset(self):
        """_make_dataset (ppo.py:110-142, :36-53) on the rollout: flat [T*E] states,
        actions, log pi_old, V, advantages, V targets, the advantage moments [2] = mean,
        std (unbiased=False), and the reference's dataset order."""
        T, dev = len(self._rewards), self.device
        states = torch.stack(self._states)            # [T, E, ...]
        next_states = torch.stack(self._next_states)
        actions = torch.stack(self._actions)
        E = states.shape[1]
        N = T * E
        reward = torch.as_tensor(np.stack(self._rewards), device=dev)
        nonterminal = torch.as_tensor(np.stack(self._nonterminal), device=dev)
        cut_np = np.stack(self._cut)
        cut_np[T - 1, :] = 1  # flush of unfinished episodes
        cut = torch.as_tensor(cut_np, device=dev)
        order = self._dataset_order(T, E)

        flat_s = states.reshape((N,) + states.shape[2:])
        flat_ns = next_states.reshape((N,) + states.shape[2:])
        flat_a = actions.reshape((N,) + actions.shape[2:])
        norm = self.obs_normalizer
        with torch.no_grad(), evaluating(self.model):
            distribs, vs_pred = self.model(norm(flat_s, update=False) if norm else flat_s)
            _, next_vs_pred = self.model(norm(flat_ns, update=False) if norm else flat_ns)
            log_probs_old = distribs.log_prob(flat_a).float()
            v = vs_pred.reshape(T, E).float()
            v_next = next_vs_pred.reshape(T, E).float()
        if self.use_fused and dev.type == "cuda":
            adv, v_teacher, stats = fused.gae(reward, nonterminal, v, v_next, cut, self.gamma,
                                              self.lambd)
        else:
            adv, v_teacher = _gae_torch(reward, nonterminal, v, v_next, cut, self.gamma, self.lambd)
            std, mean = torch.std_mean(adv, unbiased=False)
            stats = torch.stack([mean, std])
        return dict(flat_s=flat_s, flat_a=flat_a, log_probs_old=log_probs_old, v_old=v.reshape(N),
                    adv=adv, v_teacher=v_teacher, stats=stats, order=order, E=E, N=N)

    def _explained_variance_from(self, v_teacher, v_old):
        """ppo.py:56-62 on the device; read lazily by get_statistics."""
        var_t = torch.var(v_teacher, unbiased=False)
        ev = 1 - torch.var(v_teacher - v_old, unbiased=False) / var_t
        self._explained_variance_t = torch.where(var_t == 0, torch.full_like(ev, float("nan")), ev)
        self.explained_variance = None


class PPO(_DeviceRollout, agent.AttributeSavingMixin, agent.BatchAgent):
    saved_attributes = ("model", "optimizer", "obs_normalizer")

    def __init__(self, model, optimizer, obs_normalizer=None, gpu=None, gamma=0.99, lambd=0.95,
                 phi=lambda x: x, value_func_coef=1.0, entropy_coef=0.01, update_interval=2048,
                 minibatch_size=64, epochs=10, clip_eps=0.2, clip_eps_vf=None,
                 standardize_advantages=True, batch_states=batch_states, recurrent=False,
                 max_recurrent_sequence_len=None, act_deterministically=False,
                 max_grad_norm=None, value_stats_window=1000, entropy_stats_window=1000,
                 value_loss_stats_window=100, policy_loss_stats_window=100, grad_sync=None,
                 stats_sync=None, cuda_graph=False):
        if recurrent and (cuda_graph or grad_sync is not None or stats_sync is not None):
            raise ValueError("recurrent=True cannot be combined with cuda_graph, grad_sync or "
                             "stats_sync: the minibatches have variable shapes and recurrent "
                             "PPO runs on one device")
        self.model = model
        self.optimizer = optimizer
        self.obs_normalizer = obs_normalizer
        if gpu is not None and gpu >= 0:
            assert torch.cuda.is_available()
            self.device = torch.device("cuda:{}".format(gpu))
            self.model.to(self.device)
            if self.obs_normalizer is not None:
                self.obs_normalizer.to(self.device)
        else:
            self.device = torch.device("cpu")
        self.gamma = gamma
        self.lambd = lambd
        self.phi = phi
        self.value_func_coef = value_func_coef
        self.entropy_coef = entropy_coef
        self.update_interval = update_interval
        self.minibatch_size = minibatch_size
        self.epochs = epochs
        self.clip_eps = clip_eps
        self.clip_eps_vf = clip_eps_vf
        self.standardize_advantages = standardize_advantages
        self.batch_states = batch_states
        self.recurrent = bool(recurrent)
        self.max_recurrent_sequence_len = max_recurrent_sequence_len
        self.act_deterministically = act_deterministically
        self.max_grad_norm = max_grad_norm
        # data-parallel hooks: grad_sync(model) all-reduces gradients,
        # stats_sync(tensor[3] = count, sum, sumsq) all-reduces advantage moments
        self.grad_sync = grad_sync
        self.stats_sync = stats_sync
        self.use_fused = True
        # Optional: the minibatch step (gather, forward, fused loss, backward, clip,
        # Adam: ~100 launches of tiny kernels, 320 times per update) replayed as ONE
        # CUDA graph over persistent dataset buffers.
        self._graph = None
        if cuda_graph and self.device.type == "cuda" and grad_sync is None:
            self._graph = CapturedStep(3, (optimizer,))
        # rollout (device tensors per vector step)
        self._rollout_clear()
        self._cur_state = None
        self._cur_action = None
        # recurrent: batched states on the device, and per vector step the flattened
        # states before / after it ([E, 2, D]) plus whether the one before was None
        self.train_recurrent_states = None
        self.test_recurrent_states = None
        self._rstates, self._rpresent = [], []
        self._cur_rs = None
        self._state_spec = None
        self._state_nest = None
        self._seq_gather = None
        self.value_record = _DeviceRing(value_stats_window)
        self.entropy_record = _DeviceRing(entropy_stats_window)
        self.value_loss_record = _DeviceRing(value_loss_stats_window)
        self.policy_loss_record = _DeviceRing(policy_loss_stats_window)
        self.explained_variance = np.nan
        self.n_updates = 0

    # ----------------------------------------------------------------- acting
    def _features(self, batch_obs):
        b_state = self.batch_states(batch_obs, self.device, self.phi)
        if self.obs_normalizer:
            return b_state, self.obs_normalizer(b_state, update=False)
        return b_state, b_state

    def batch_act(self, batch_obs):
        raw, feat = self._features(batch_obs)
        with torch.no_grad(), evaluating(self.model):
            if self.recurrent:
                action_distrib, batch_value = self._recurrent_step(feat)
            else:
                action_distrib, batch_value = self.model(feat)
            if not self.training:
                if self.act_deterministically:
                    return mode_of_distribution(action_distrib).cpu().numpy()
                return action_distrib.sample().cpu().numpy()
            action = action_distrib.sample()
            self.entropy_record.extend(action_distrib.entropy())
            self.value_record.extend(batch_value)
        self._record_act(raw, action, len(batch_obs))
        return action.cpu().numpy()

    def _recurrent_step(self, feat):
        """One step of the train or test states (ppo.py:706-740); in training, also the
        ring rows of this step: the state before it (zeros if None) and after it."""
        if not self.training:
            out, self.test_recurrent_states = one_step_forward(
                self.model, feat, self.test_recurrent_states)
            return out
        prev = self.train_recurrent_states
        out, self.train_recurrent_states = one_step_forward(self.model, feat, prev)
        leaves, nest = _state_leaves(self.train_recurrent_states)
        if not leaves:  # a state of no tensors (only None entries): nothing to store
            self._cur_rs = (None, False)
            return out
        if self._state_spec is None:
            self._state_spec = rollout.StateSpec([(x.shape[0], x.shape[2]) for x in leaves])
            self._state_nest = nest
        after = self._state_spec.flatten(leaves)
        before = torch.zeros_like(after) if prev is None else \
            self._state_spec.flatten(_state_leaves(prev)[0])
        self._cur_rs = (torch.stack([before, after], dim=1), prev is not None)
        return out

    def _mask_ended(self, states, batch_done, batch_reset):
        ended = [i for i, (d, r) in enumerate(zip(batch_done, batch_reset)) if d or r]
        return mask_recurrent_state_at(states, ended) if ended else states

    def batch_observe(self, batch_obs, batch_reward, batch_done, batch_reset):
        if not self.training:
            if self.recurrent:  # ppo.py:742-754
                self.test_recurrent_states = self._mask_ended(
                    self.test_recurrent_states, batch_done, batch_reset)
            return
        num_envs = len(batch_obs)
        steps = self._record_observe(batch_obs, batch_reward, batch_done, batch_reset)
        if self.recurrent:
            rows, present = self._cur_rs
            self._rstates.append(rows)
            self._rpresent.append(present)
            self._cur_rs = None
            self.train_recurrent_states = self._mask_ended(
                self.train_recurrent_states, batch_done, batch_reset)
        if steps * num_envs >= self.update_interval:
            if self.recurrent:
                self._update_recurrent_from_rollout()
            else:
                self._update_from_rollout()

    # ------------------------------------------------------------ the update
    def _update_from_rollout(self):
        dev = self.device
        d = self._rollout_dataset()
        flat_s, flat_a, log_probs_old = d["flat_s"], d["flat_a"], d["log_probs_old"]
        adv, v_teacher, stats, order, E, N = (d["adv"], d["v_teacher"], d["stats"], d["order"],
                                              d["E"], d["N"])
        if self.stats_sync is not None and self.standardize_advantages:
            stats = self.stats_sync(adv)
        adv, v_teacher = adv.reshape(N), v_teacher.reshape(N)
        v_old = d["v_old"]
        norm = self.obs_normalizer

        if norm:  # _update_obs_normalizer (ppo.py:460-463), after the dataset is built
            norm.experience(flat_s)

        adv_stats = stats if self.standardize_advantages else None
        if self._graph is not None:
            self._minibatches_graphed(order, flat_s, flat_a, log_probs_old, v_old, adv, v_teacher,
                                      adv_stats)
        else:
            for mb in _yield_minibatch_indices(order, self.minibatch_size, self.epochs):
                idx = torch.as_tensor(mb, device=dev)
                s = flat_s[idx]
                self._record_losses(self._minibatch_step(
                    norm(s, update=False) if norm else s, flat_a[idx], log_probs_old[idx],
                    v_old[idx], adv[idx], v_teacher[idx], adv_stats))
                self.n_updates += 1

        self._explained_variance_from(v_teacher, v_old)
        self._rollout_clear(E)

    # -------------------------------------------------------- recurrent update
    def _episode_spans(self, T, E):
        """The rollout's episodes in the reference's memory order (as _dataset_order)."""
        spans = [_Span(e, s, t_end + 1 - s) for e, s, t_end in self._segments]
        spans += [_Span(e, self._seg_start[e], T - self._seg_start[e])
                  for e in range(E) if self._seg_start[e] <= T - 1]
        return spans

    def _gather_sequences(self, spans, E, columns, index=False, states=None):
        """Pack ``spans`` (sorted stably, longest first, here) out of the rollout:
        the kernel on CUDA, the index_select formulation on CPU or with use_fused=False.
        Returns (packed columns, flat slots or None, {side: state}, batch_sizes)."""
        spans = sorted(spans, key=len, reverse=True)
        first = np.array([s.first_slot(E) for s in spans], dtype=np.int64)
        lens = np.array([len(s) for s in spans], dtype=np.int64)
        if self.use_fused and self.device.type == "cuda":
            if self._seq_gather is None:
                self._seq_gather = rollout.SequenceGather(self.device)
            outs, idx, leaves = self._seq_gather(first, lens, E, columns, index, states)
        else:
            outs, idx, leaves = rollout.gather_sequences_torch(first, lens, E, columns, index,
                                                              states)
        rs = {side: _state_from_leaves(self._state_nest, ls) for side, ls in leaves.items()}
        batch_sizes = torch.as_tensor(rollout.packed_layout(lens)[0])
        return outs, idx, rs, batch_sizes

    def _update_recurrent_from_rollout(self):
        """_make_dataset_recurrent + _update_recurrent (ppo.py:196-243,608-631) on the rollout."""
        T, dev = len(self._rewards), self.device
        states = torch.stack(self._states)
        E = states.shape[1]
        N = T * E
        flat_s = states.reshape((N,) + states.shape[2:])
        flat_ns = torch.stack(self._next_states).reshape(flat_s.shape)
        actions = torch.stack(self._actions)
        flat_a = actions.reshape((N,) + actions.shape[2:]).contiguous()
        reward = torch.as_tensor(np.stack(self._rewards), device=dev)
        nonterminal = torch.as_tensor(np.stack(self._nonterminal), device=dev)
        cut_np = np.stack(self._cut)
        cut_np[T - 1, :] = 1  # flush of unfinished episodes
        cut = torch.as_tensor(cut_np, device=dev)
        if self._state_spec is None:  # the model's states hold no tensors
            both_states = first_states = None
        else:
            ring = torch.stack(self._rstates).reshape(N, 2, -1).contiguous()  # [T*E][2][D]
            present = np.ones((T, E, 2), dtype=np.uint8)
            present[:, :, 0] = np.asarray(self._rpresent, dtype=np.uint8)[:, None]
            present = torch.as_tensor(present.reshape(N, 2), device=dev)
            both_states = (ring, present, self._state_spec, (0, 1))
            first_states = (ring, present, self._state_spec, (0,))
        episodes = self._episode_spans(T, E)
        norm = self.obs_normalizer

        # _add_log_prob_and_value_to_episodes_recurrent: whole episodes, both first states
        (s_p, ns_p, a_p), idx, rs, batch_sizes = self._gather_sequences(
            episodes, E, [_normalized(flat_s, norm).contiguous(),
                          _normalized(flat_ns, norm).contiguous(), flat_a],
            index=True, states=both_states)
        with torch.no_grad(), evaluating(self.model):
            (distribs, vs), _ = pack_and_forward(self.model, PackedSequence(s_p, batch_sizes),
                                                 rs.get(0))
            (_, next_vs), _ = pack_and_forward(self.model, PackedSequence(ns_p, batch_sizes),
                                               rs.get(1))
            lp = distribs.log_prob(a_p).float()
        log_probs_old = torch.empty(N, dtype=torch.float32, device=dev).index_copy_(0, idx, lp)
        v = torch.empty(N, dtype=torch.float32, device=dev).index_copy_(
            0, idx, vs.reshape(-1).float()).reshape(T, E)
        v_next = torch.empty(N, dtype=torch.float32, device=dev).index_copy_(
            0, idx, next_vs.reshape(-1).float()).reshape(T, E)
        if self.use_fused and dev.type == "cuda":
            adv, v_teacher, stats = fused.gae(reward, nonterminal, v, v_next, cut, self.gamma,
                                              self.lambd)
        else:
            adv, v_teacher = _gae_torch(reward, nonterminal, v, v_next, cut, self.gamma, self.lambd)
            std, mean = torch.std_mean(adv, unbiased=False)
            stats = torch.stack([mean, std])
        adv, v_teacher, v_old = adv.reshape(N), v_teacher.reshape(N), v.reshape(N)
        if self.max_recurrent_sequence_len is not None:
            dataset = _limit_sequence_length(episodes, self.max_recurrent_sequence_len)
        else:
            dataset = list(episodes)

        # _update_recurrent
        if norm:
            norm.experience(flat_s)
        obs = _normalized(flat_s, norm).contiguous()
        adv_stats = stats if self.standardize_advantages else None
        columns = [obs, flat_a, adv, log_probs_old, v_old, v_teacher]
        for _ in range(self.epochs):
            random.shuffle(dataset)
            for mb in _yield_subset_of_sequences_with_fixed_number_of_items(
                    dataset, self.minibatch_size):
                (s, a, adv_mb, lp_mb, vo_mb, vt_mb), _, rs, batch_sizes = self._gather_sequences(
                    mb, E, columns, states=first_states)
                (distribs, vs_pred), _ = pack_and_forward(
                    self.model, PackedSequence(s, batch_sizes), rs.get(0))
                self.model.zero_grad()
                loss, parts = self._lossfun(
                    distribs.entropy(), vs_pred, distribs.log_prob(a),
                    vs_pred_old=vo_mb[..., None], log_probs_old=lp_mb, advs=adv_mb,
                    vs_teacher=vt_mb[..., None], adv_stats=adv_stats)
                self._record_losses(parts)
                loss.backward()
                if self.max_grad_norm is not None:
                    torch.nn.utils.clip_grad_norm_(self.model.parameters(), self.max_grad_norm)
                self.optimizer.step()
                self.n_updates += 1

        self._explained_variance_from(v_teacher, v_old)
        self._rollout_clear(E)
        self._rstates, self._rpresent = [], []

    def _minibatch_step(self, s, a, log_probs_old, v_old, advs, v_teacher, adv_stats):
        """One gradient step on one minibatch (ppo.py:480-532); returns the detached
        (policy loss, value loss)."""
        distribs, vs_pred = self.model(s)
        self.model.zero_grad()
        loss, parts = self._lossfun(
            distribs.entropy(), vs_pred, distribs.log_prob(a), vs_pred_old=v_old[..., None],
            log_probs_old=log_probs_old, advs=advs, vs_teacher=v_teacher[..., None],
            adv_stats=adv_stats)
        loss.backward()
        if self.grad_sync is not None:
            self.grad_sync(self.model)
        if self.max_grad_norm is not None:
            torch.nn.utils.clip_grad_norm_(self.model.parameters(), self.max_grad_norm)
        self.optimizer.step()
        return parts

    def _record_losses(self, parts):
        self.policy_loss_record.append(parts[0])
        self.value_loss_record.append(parts[1])

    def _minibatches_graphed(self, order, flat_s, flat_a, log_probs_old, v_old, adv, v_teacher,
                             adv_stats):
        """The minibatch steps over persistent dataset buffers, loaded once per update; each
        row writes its minibatch's indices into the index buffer and runs the step."""
        norm = self.obs_normalizer
        mbs = list(_yield_minibatch_indices(order, self.minibatch_size, self.epochs))
        all_idx = torch.as_tensor(np.asarray(mbs, dtype=np.int64), device=self.device)
        # the normaliser is frozen during the epochs (update=False): apply it once
        data = dict(s=norm(flat_s, update=False) if norm else flat_s, a=flat_a,
                    lp=log_probs_old, vo=v_old, adv=adv, vt=v_teacher, idx=all_idx[0])
        if adv_stats is not None:
            data["stats"] = adv_stats
        g = self._graph.load((self.clip_eps, self.clip_eps_vf, self.value_func_coef,
                              self.entropy_coef, self.max_grad_norm, self.minibatch_size), data)

        def step(g):
            i = g["idx"]
            return self._minibatch_step(g["s"][i], g["a"][i], g["lp"][i], g["vo"][i],
                                        g["adv"][i], g["vt"][i], g.get("stats"))

        for row in all_idx:
            g["idx"].copy_(row)
            self._record_losses(self._graph.run(step))
            self.n_updates += 1

    def _lossfun(self, entropy, vs_pred, log_probs, vs_pred_old, log_probs_old, advs, vs_teacher,
                 adv_stats=None):
        """ppo.py:495 + :634-671; returns the loss and the detached (policy loss, value
        loss)."""
        if self.use_fused and log_probs.is_cuda:
            loss, parts = fused.ppo_loss(
                log_probs, entropy, vs_pred, log_probs_old, vs_pred_old, advs, vs_teacher,
                adv_stats, self.clip_eps, self.clip_eps_vf, self.value_func_coef,
                self.entropy_coef)
            return loss, (parts[1], parts[2])
        if adv_stats is not None:
            advs = (advs - adv_stats[0]) / (adv_stats[1] + 1e-8)
        prob_ratio = torch.exp(log_probs - log_probs_old)
        loss_policy = -torch.mean(torch.min(
            prob_ratio * advs,
            torch.clamp(prob_ratio, 1 - self.clip_eps, 1 + self.clip_eps) * advs))
        if self.clip_eps_vf is None:
            loss_value_func = F.mse_loss(vs_pred, vs_teacher)
        else:
            clipped = _elementwise_clip(vs_pred, vs_pred_old - self.clip_eps_vf,
                                        vs_pred_old + self.clip_eps_vf)
            loss_value_func = torch.mean(torch.max(
                F.mse_loss(vs_pred, vs_teacher, reduction="none"),
                F.mse_loss(clipped, vs_teacher, reduction="none")))
        loss_entropy = -torch.mean(entropy)
        loss = (loss_policy + self.value_func_coef * loss_value_func
                + self.entropy_coef * loss_entropy)
        return loss, (loss_policy.detach(), loss_value_func.detach())

    def get_statistics(self):
        if self.explained_variance is None:
            self.explained_variance = float(self._explained_variance_t.item())
        return [
            ("average_value", self.value_record.mean()),
            ("average_entropy", self.entropy_record.mean()),
            ("average_value_loss", self.value_loss_record.mean()),
            ("average_policy_loss", self.policy_loss_record.mean()),
            ("n_updates", self.n_updates),
            ("explained_variance", self.explained_variance),
        ]


def _gae_torch(reward, nonterminal, v, v_next, cut, gamma, lambd):
    """Host formulation of the GAE recurrence (CPU agents; fp64 like the kernel)."""
    T, E = reward.shape
    adv = torch.zeros((T, E), dtype=torch.float64, device=reward.device)
    run = torch.zeros(E, dtype=torch.float64, device=reward.device)
    r, nt = reward.double(), nonterminal.double()
    vv, vn = v.double(), v_next.double()
    for t in range(T - 1, -1, -1):
        run = torch.where(cut[t].bool(), torch.zeros_like(run), run)
        run = (r[t] + gamma * nt[t] * vn[t] - vv[t]) + gamma * lambd * run
        adv[t] = run
    return adv.float(), (adv + vv).float()
