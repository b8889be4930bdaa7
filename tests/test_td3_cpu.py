"""CPU: TD3 and DDPG accept ``cuda_graph=True`` and, off CUDA, it changes nothing (the seeded
reference runs of tests/test_agent_traces_cpu.py reproduce with it set); the C ABI declares
and exports the fused critic-update entry points."""
import os
import sys
from unittest import mock

import pytest

sys.path.insert(0, os.path.dirname(__file__))
from test_abi_cpu import header_functions  # noqa: E402
from test_agent_traces_cpu import test_more_agents_reproduce_the_reference_run as _trace  # noqa: E402

NEW_ENTRY_POINTS = ("b2rl_td3_smooth", "b2rl_td3_critic_loss")


@pytest.mark.parametrize("kind", ["td3", "ddpg"])
def test_cuda_graph_on_cpu_reproduces_the_reference_run(kind):
    import pfrl_b200.agents as agents

    cls = getattr(agents, kind.upper())
    made = []

    def make(*args, **kw):
        made.append(cls(*args, cuda_graph=True, **kw))
        return made[-1]

    with mock.patch.object(agents, cls.__name__, make):
        _trace(kind)
    (agent,) = made
    assert agent.device.type == "cpu"
    graphs = (agent._q_graph, agent._full_graph) if kind == "td3" else (agent._graph,)
    assert graphs == (None,) * len(graphs)


def test_fused_critic_update_entry_points_are_declared_and_bound():
    import ctypes

    from pfrl_b200 import _lib

    names = header_functions()
    lib = ctypes.CDLL(_lib.build())
    for name in NEW_ENTRY_POINTS:
        assert name in names and name in _lib.SIGNATURES, name
        assert hasattr(lib, name), name


def test_fused_switch_is_a_class_attribute():
    from pfrl_b200.agents import DDPG, TD3

    assert TD3.use_fused is True and DDPG.use_fused is True
