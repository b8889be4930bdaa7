"""Agent interfaces (same public surface as pfrl/agent.py:9-200).

``Agent.act / observe / save / load / get_statistics / eval_mode``,
``BatchAgent.batch_act / batch_observe`` and the ``saved_attributes``
checkpoint layout (one ``<attr>.pt`` state_dict per attribute, nested
directories for nested savers) are the drop-in boundary for training loops.
"""
import contextlib
import os
from abc import ABCMeta, abstractmethod

import torch


class Agent(object, metaclass=ABCMeta):
    """What a training loop needs from an agent (pfrl/agent.py:9-70)."""

    training = True

    @abstractmethod
    def act(self, obs):
        raise NotImplementedError()

    @abstractmethod
    def observe(self, obs, reward, done, reset):
        raise NotImplementedError()

    @abstractmethod
    def save(self, dirname):
        pass

    @abstractmethod
    def load(self, dirname):
        pass

    @abstractmethod
    def get_statistics(self):
        """List of (name, value) pairs, e.g. [('average_loss', 0), ...]."""
        pass

    @contextlib.contextmanager
    def eval_mode(self):
        previous = self.training
        try:
            self.training = False
            yield
        finally:
            self.training = previous


_WRAPPERS = (torch.nn.parallel.DistributedDataParallel, torch.nn.DataParallel)


class AttributeSavingMixin(object):
    """save()/load() of the attributes named in ``saved_attributes``
    (pfrl/agent.py:73-137): ``dirname/<attr>.pt`` holds ``state_dict()``;
    an attribute that is itself a saver gets the sub-directory
    ``dirname/<attr>/``; parallel wrappers are unwrapped first."""

    saved_attributes = ()

    def save(self, dirname):
        self._save_into(dirname, ())

    def _save_into(self, dirname, chain):
        os.makedirs(dirname, exist_ok=True)
        chain = chain + (self,)
        for name in self.saved_attributes:
            assert hasattr(self, name)
            value = getattr(self, name)
            if value is None:
                continue
            if isinstance(value, AttributeSavingMixin):
                assert all(value is not c for c in chain), "Avoid an infinite loop"
                value._save_into(os.path.join(dirname, name), chain)
                continue
            if isinstance(value, _WRAPPERS):
                value = value.module
            torch.save(value.state_dict(), os.path.join(dirname, name + ".pt"))

    def load(self, dirname):
        self._load_from(dirname, ())

    def _load_from(self, dirname, chain):
        where = None if torch.cuda.is_available() else torch.device("cpu")
        chain = chain + (self,)
        for name in self.saved_attributes:
            assert hasattr(self, name)
            value = getattr(self, name)
            if value is None:
                continue
            if isinstance(value, AttributeSavingMixin):
                assert all(value is not c for c in chain), "Avoid an infinite loop"
                value._load_from(os.path.join(dirname, name), chain)
                continue
            if isinstance(value, _WRAPPERS):
                value = value.module
            value.load_state_dict(torch.load(os.path.join(dirname, name + ".pt"), where))


class AsyncAgent(Agent, metaclass=ABCMeta):
    """Agent whose training is shared between processes (pfrl/agent.py:140-154)."""

    @property
    @abstractmethod
    def process_idx(self):
        """Index of the process, 0 for the representative one; None if not assigned."""
        pass

    @property
    @abstractmethod
    def shared_attributes(self):
        """Names of the attributes the processes share."""
        pass


def assert_shared_memory(agent, models=("model", "shared_model")):
    """The check of an ``AsyncAgent``'s ``assert_shared_memory`` (pfrl/agents/a3c.py:
    110-123).  On the CPU, the reference's: ``agent.shared_model`` and the optimizer's
    state are in shared memory and ``agent.model`` is not.  CUDA storages always report
    ``is_shared()``, so on CUDA what sharing is for is checked instead: the modules named in
    ``models`` share no storage, and ``agent.optimizer`` steps ``agent.shared_model``'s
    parameters."""
    if agent.device.type != "cuda":
        for k, v in agent.shared_model.state_dict().items():
            assert v.is_shared(), "{} is not in shared memory".format(k)
        for k, v in agent.model.state_dict().items():
            assert not v.is_shared(), "{} is in shared memory".format(k)
        for param_state in agent.optimizer.state_dict()["state"].values():
            for k, v in param_state.items():
                if isinstance(v, torch.Tensor):
                    assert v.is_shared(), "{} is not in shared memory".format(k)
        return
    ptrs = {}
    for name in models:
        for k, v in getattr(agent, name).state_dict().items():
            if v.numel():
                owner = ptrs.setdefault(v.untyped_storage().data_ptr(), name)
                assert owner == name, "{}.{} shares storage with {}".format(name, k, owner)
    stepped = {id(p) for group in agent.optimizer.param_groups for p in group["params"]}
    assert stepped == {id(p) for p in agent.shared_model.parameters()}, \
        "the optimizer must step shared_model's parameters"


class BatchAgent(Agent, metaclass=ABCMeta):
    """Agent that steps a batch of environments; the single-env calls are
    the batch calls with a batch of one (pfrl/agent.py:157-200)."""

    def act(self, obs):
        return self.batch_act([obs])[0]

    def observe(self, obs, reward, done, reset):
        self.batch_observe([obs], [reward], [done], [reset])

    @abstractmethod
    def batch_act(self, batch_obs):
        raise NotImplementedError()

    @abstractmethod
    def batch_observe(self, batch_obs, batch_reward, batch_done, batch_reset):
        raise NotImplementedError()
