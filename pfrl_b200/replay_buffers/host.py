"""Host-memory uniform replay buffer for CPU-only agents (``gpu=None``), e.g.
the CartPole quickstart configuration.  This is an explicit, separate class:
the device buffers never fall back to it.  Semantics follow
pfrl/replay_buffers/replay_buffer.py:11-94 (n-step window per env_id, uniform
``sample_n_k`` sampling, pickle save/load)."""
import collections
import pickle

from pfrl_b200.collections.random_access_queue import RandomAccessQueue


class HostReplayBuffer:
    def __init__(self, capacity=None, num_steps=1):
        assert num_steps > 0
        self._capacity = capacity
        self.num_steps = num_steps
        self.memory = RandomAccessQueue(maxlen=capacity)   # O(1) indexing for sample()
        self.last_n_transitions = collections.defaultdict(
            lambda: collections.deque([], maxlen=num_steps))

    @property
    def capacity(self):
        return self._capacity

    def append(self, state, action, reward, next_state=None, next_action=None,
               is_state_terminal=False, env_id=0, **kwargs):
        window = self.last_n_transitions[env_id]
        window.append(dict(state=state, action=action, reward=reward, next_state=next_state,
                           next_action=next_action, is_state_terminal=is_state_terminal,
                           **kwargs))
        if is_state_terminal:
            while window:
                self.memory.append(list(window))
                window.popleft()
        elif len(window) == self.num_steps:
            self.memory.append(list(window))

    def stop_current_episode(self, env_id=0):
        window = self.last_n_transitions[env_id]
        if 0 < len(window) < self.num_steps:
            self.memory.append(list(window))
        if 0 < len(window) <= self.num_steps:
            window.popleft()
        while window:
            self.memory.append(list(window))
            window.popleft()

    def sample(self, num_experiences):
        assert len(self.memory) >= num_experiences
        return self.memory.sample(num_experiences)

    def __len__(self):
        return len(self.memory)

    def save(self, filename):
        with open(filename, "wb") as f:
            pickle.dump(list(self.memory), f)

    def load(self, filename):
        """Own format (a pickled list) or a checkpoint written by the
        reference's ReplayBuffer.save (replay_buffer.py:85-94)."""
        from pfrl_b200.replay_buffers import reference_pickle

        items = reference_pickle.read(filename).experiences
        self.memory = RandomAccessQueue(items, maxlen=self._capacity)


class HostEpisodicReplayBuffer:
    """Host-memory episodic replay buffer for CPU-only recurrent agents
    (``gpu=None``).  Semantics follow pfrl/replay_buffers/episodic.py:9-98:
    each ``env_id`` collects its current episode, which is committed whole at
    ``stop_current_episode`` or at a terminal transition; ``len()`` counts
    transitions and ``n_episodes`` episodes; when the transitions exceed
    ``capacity`` the oldest whole episodes are dropped; ``sample(n)`` draws
    transitions and ``sample_episodes`` episodes, both uniformly through
    ``sample_n_k``."""

    def __init__(self, capacity=None):
        self._capacity = capacity
        self.current_episode = collections.defaultdict(list)
        self.episodic_memory = RandomAccessQueue()
        self.memory = RandomAccessQueue()

    @property
    def capacity(self):
        return self._capacity

    def append(self, state, action, reward, next_state=None, next_action=None,
               is_state_terminal=False, env_id=0, **kwargs):
        self.current_episode[env_id].append(dict(
            state=state, action=action, reward=reward, next_state=next_state,
            next_action=next_action, is_state_terminal=is_state_terminal, **kwargs))
        if is_state_terminal:
            self.stop_current_episode(env_id=env_id)

    def stop_current_episode(self, env_id=0):
        episode = self.current_episode[env_id]
        if episode:
            self.episodic_memory.append(episode)
            for transition in episode:
                self.memory.append([transition])
            self.current_episode[env_id] = []
            while self._capacity is not None and len(self.memory) > self._capacity:
                for _ in range(len(self.episodic_memory.popleft())):
                    self.memory.popleft()

    def sample(self, n):
        assert len(self.memory) >= n
        return self.memory.sample(n)

    def sample_episodes(self, n_episodes, max_len=None):
        from pfrl_b200.replay_buffer import random_subseq

        assert len(self.episodic_memory) >= n_episodes
        episodes = self.episodic_memory.sample(n_episodes)
        if max_len is None:
            return episodes
        return [random_subseq(ep, max_len) for ep in episodes]

    def __len__(self):
        return len(self.memory)

    @property
    def n_episodes(self):
        return len(self.episodic_memory)

    def save(self, filename):
        with open(filename, "wb") as f:
            pickle.dump(list(self.episodic_memory), f)

    def load(self, filename):
        """Own format: the pickled list of committed episodes."""
        with open(filename, "rb") as f:
            episodes = pickle.load(f)
        self.episodic_memory = RandomAccessQueue(episodes)
        self.memory = RandomAccessQueue([t] for ep in episodes for t in ep)
