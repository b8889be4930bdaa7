from pfrl_b200.replay_buffers.device_buffer import DeviceExperiences  # NOQA
from pfrl_b200.replay_buffers.device_buffer import PrioritizedReplayBuffer  # NOQA
from pfrl_b200.replay_buffers.device_buffer import PriorityWeightError  # NOQA
from pfrl_b200.replay_buffers.device_buffer import ReplayBuffer  # NOQA
from pfrl_b200.replay_buffers.host import HostReplayBuffer  # NOQA
from pfrl_b200.replay_buffers.episodic import DeviceEpisodes  # NOQA
from pfrl_b200.replay_buffers.episodic import EpisodicReplayBuffer  # NOQA
from pfrl_b200.replay_buffers.host import HostEpisodicReplayBuffer  # NOQA
