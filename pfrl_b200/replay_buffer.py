"""Replay-buffer interface, minibatch builder and update schedule.

Mirrors pfrl/replay_buffer.py (AbstractReplayBuffer :15-114,
AbstractEpisodicReplayBuffer :117-146, random_subseq :149-154,
batch_experiences :157-212, batch_recurrent_experiences :215-287,
ReplayUpdater :290-356).  ``batch_experiences`` gathers straight from HBM when
it is handed the ``DeviceExperiences`` that the device buffers' ``sample``
returns, and ``batch_recurrent_experiences`` likewise for the
``DeviceEpisodes`` of the device ``EpisodicReplayBuffer.sample_episodes``;
otherwise both follow the reference's host algorithm on lists of transition
dicts.
"""
from abc import ABCMeta, abstractmethod

import numpy as np
import torch

from pfrl_b200.replay_buffers.device_buffer import DeviceExperiences
from pfrl_b200.replay_buffers.episodic import DeviceEpisodes
from pfrl_b200.utils.batch_states import batch_states
from pfrl_b200.utils.recurrent import (
    concatenate_recurrent_states,
    flatten_sequences_time_first,
    recurrent_state_from_numpy,
)


class AbstractReplayBuffer(object, metaclass=ABCMeta):
    """Interface shared by replay buffers (pfrl/replay_buffer.py:15-114)."""

    @abstractmethod
    def append(self, state, action, reward, next_state=None, next_action=None,
               is_state_terminal=False, env_id=0, **kwargs):
        raise NotImplementedError

    @abstractmethod
    def sample(self, n):
        raise NotImplementedError

    @abstractmethod
    def __len__(self):
        raise NotImplementedError

    @abstractmethod
    def save(self, filename):
        raise NotImplementedError

    @abstractmethod
    def load(self, filename):
        raise NotImplementedError

    @property
    @abstractmethod
    def capacity(self):
        raise NotImplementedError

    @abstractmethod
    def stop_current_episode(self, env_id=0):
        raise NotImplementedError


class AbstractEpisodicReplayBuffer(AbstractReplayBuffer):
    """Replay buffer that also samples whole episodes
    (pfrl/replay_buffer.py:117-146)."""

    @abstractmethod
    def sample_episodes(self, n_episodes, max_len=None):
        """n distinct episodes, each cut to a random window of at most
        ``max_len`` transitions when ``max_len`` is not None."""
        raise NotImplementedError

    @property
    @abstractmethod
    def n_episodes(self):
        raise NotImplementedError


def random_subseq(seq, subseq_len):
    """``seq`` itself if it is not longer than ``subseq_len``, else a window of
    ``subseq_len`` items whose start is one ``np.random.randint`` draw."""
    if len(seq) <= subseq_len:
        return seq
    i = np.random.randint(0, len(seq) - subseq_len + 1)
    return seq[i:i + subseq_len]


def _register_device_buffers():
    from pfrl_b200.replay_buffers import device_buffer, episodic

    from pfrl_b200.replay_buffers import host

    AbstractReplayBuffer.register(device_buffer.DeviceNStepBuffer)
    AbstractReplayBuffer.register(host.HostReplayBuffer)
    AbstractEpisodicReplayBuffer.register(episodic.EpisodicReplayBuffer)
    AbstractEpisodicReplayBuffer.register(host.HostEpisodicReplayBuffer)


_register_device_buffers()


def batch_experiences(experiences, device, phi, gamma, batch_states=batch_states):
    """Vectorise k experiences of 1..n transitions each into a dict of
    tensors: state / action of the first transition, next_state of the last,
    reward = sum_i gamma^i r_i, is_state_terminal = any, discount = gamma^len
    (pfrl/replay_buffer.py:157-212)."""
    if isinstance(experiences, DeviceExperiences):
        return experiences.batch(gamma, phi, device)
    firsts = [e[0] for e in experiences]
    lasts = [e[-1] for e in experiences]
    batch = {
        "state": batch_states([t["state"] for t in firsts], device, phi),
        "action": torch.as_tensor([t["action"] for t in firsts], device=device),
        "reward": torch.as_tensor(
            [sum((gamma ** i) * e[i]["reward"] for i in range(len(e))) for e in experiences],
            dtype=torch.float32, device=device),
        "next_state": batch_states([t["next_state"] for t in lasts], device, phi),
        "is_state_terminal": torch.as_tensor(
            [any(t["is_state_terminal"] for t in e) for e in experiences],
            dtype=torch.float32, device=device),
        "discount": torch.as_tensor(
            [gamma ** len(e) for e in experiences], dtype=torch.float32, device=device),
    }
    if all(t["next_action"] is not None for t in lasts):
        batch["next_action"] = torch.as_tensor([t["next_action"] for t in lasts], device=device)
    return batch


def _is_sorted_desc_by_lengths(seqs):
    return all(len(a) >= len(b) for a, b in zip(seqs, seqs[1:]))


def _state_to(recurrent_state, device):
    """Stored states are numpy (reference agents, host buffers) or tensors."""
    if isinstance(recurrent_state, tuple):
        return tuple(_state_to(s, device) for s in recurrent_state)
    if isinstance(recurrent_state, torch.Tensor):
        return recurrent_state.to(device)
    return recurrent_state_from_numpy(recurrent_state, device)


def batch_recurrent_experiences(experiences, device, phi, gamma, batch_states=batch_states):
    """Batch episodes for a recurrent update (pfrl/replay_buffer.py:219-287).

    ``experiences`` are episodes (lists of transition dicts) sorted by length,
    longest first.  "state" / "next_state" are lists of per-episode batches
    (``pack_and_forward`` packs them); action, reward, is_state_terminal and
    discount are flat in the time-major packed order; "recurrent_state" /
    "next_recurrent_state" are the batched states of each episode's first
    transition.  Handed the ``DeviceEpisodes`` of the device
    ``EpisodicReplayBuffer``, it gathers the packed batch in one launch
    instead, and "state" / "next_state" come back as ``PackedSequence``."""
    if isinstance(experiences, DeviceEpisodes):
        return experiences.batch(gamma, phi, device)
    assert _is_sorted_desc_by_lengths(experiences)
    flat = flatten_sequences_time_first(experiences)
    batch = {
        "state": [batch_states([t["state"] for t in ep], device, phi) for ep in experiences],
        "action": torch.as_tensor([t["action"] for t in flat], device=device),
        "reward": torch.as_tensor([t["reward"] for t in flat], dtype=torch.float,
                                  device=device),
        "next_state": [batch_states([t["next_state"] for t in ep], device, phi)
                       for ep in experiences],
        "is_state_terminal": torch.as_tensor([t["is_state_terminal"] for t in flat],
                                             dtype=torch.float, device=device),
        "discount": torch.full((len(flat),), gamma, dtype=torch.float, device=device),
        "recurrent_state": _state_to(concatenate_recurrent_states(
            [ep[0]["recurrent_state"] for ep in experiences]), device),
        "next_recurrent_state": _state_to(concatenate_recurrent_states(
            [ep[0]["next_recurrent_state"] for ep in experiences]), device),
    }
    if all(t["next_action"] is not None for t in flat):
        batch["next_action"] = torch.as_tensor([t["next_action"] for t in flat], device=device)
    return batch


class ReplayUpdater(object):
    """When and how often to update from replay (pfrl/replay_buffer.py:290-356)."""

    def __init__(self, replay_buffer, update_func, batchsize, episodic_update, n_times_update,
                 replay_start_size, update_interval, episodic_update_len=None):
        assert batchsize <= replay_start_size
        self.replay_buffer = replay_buffer
        self.update_func = update_func
        self.batchsize = batchsize
        self.episodic_update = episodic_update
        self.episodic_update_len = episodic_update_len
        self.n_times_update = n_times_update
        self.replay_start_size = replay_start_size
        self.update_interval = update_interval
        # data-parallel runs (parallel.GradSync): the agent that owns this updater; every
        # update ends in a gradient all-reduce, so all ranks must update at the SAME
        # iterations although their replay shards cross replay_start_size at different
        # ones (n-step windows depend on each rank's episode boundaries)
        self.agent = None
        self._all_ranks_ready = False

    def update_if_necessary(self, iteration):
        if self.episodic_update:
            # recurrent agents: no data-parallel ranks (DQN refuses grad_sync with recurrent)
            if len(self.replay_buffer) < self.replay_start_size:
                return False
            if self.replay_buffer.n_episodes < self.batchsize:
                return False
            if iteration % self.update_interval != 0:
                return False
            for _ in range(self.n_times_update):
                self.update_func(self.replay_buffer.sample_episodes(
                    self.batchsize, self.episodic_update_len))
            return True
        ready = len(self.replay_buffer) >= self.replay_start_size
        gs = getattr(self.agent, "grad_sync", None)
        if gs is None:
            if not ready or iteration % self.update_interval != 0:
                return False
        else:
            # `iteration` advances identically on every rank, so this collective is
            # entered by all of them or by none; once every shard is ready it stays so
            if iteration % self.update_interval != 0:
                return False
            if not self._all_ranks_ready:
                self._all_ranks_ready = gs.all_ready(ready)
            if not self._all_ranks_ready:
                return False
        for _ in range(self.n_times_update):
            self.update_func(self.replay_buffer.sample(self.batchsize))
        return True
