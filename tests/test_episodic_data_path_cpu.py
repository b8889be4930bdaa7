"""The episodic data-path model checks of tests/test_episodic_data_path_gpu.py without a
GPU: the device EpisodicReplayBuffer's host logic (episode table, whole-episode
eviction, state and mu rings with their present flags, dtypes, materialised view, save
and load) runs over the numpy store of tests/fake_episodic_store.py, and every sample
is compared with the plain model of the reference's buffer."""
from unittest import mock

import pytest
import torch

import test_episodic_data_path_gpu as T
from fake_episodic_store import EpisodicOracleStore
from pfrl_b200.replay_buffers import EpisodicReplayBuffer

CPU = torch.device("cpu")
# the host logic at smaller batch sizes: the numpy store packs in Python
B_CPU = (1, 2, 33)
NAMES = ["f32x376-nested8", "f16x7-np-f64", "f64x3-gru-f16", "i32x6-np-lstm",
         "u8x13-host-phi", "lazy4", "tiny-ring", "overlong"]


@pytest.fixture
def fake_store():
    with mock.patch("pfrl_b200.replay_buffers.device_buffer.DeviceReplayStore",
                    EpisodicOracleStore), \
            mock.patch("torch.cuda.current_device", return_value=0):
        yield


@pytest.mark.parametrize("name", NAMES)
def test_scenario(fake_store, name, tmp_path):
    sc = T.SCENARIOS[name]
    buf, model = T.build(sc, seed=sorted(T.SCENARIOS).index(name) + 1, dev=CPU)
    T.check_scenario(buf, model, sc, B_CPU)
    if name == "overlong":
        assert model.overlong > 0
    buf.save(str(tmp_path / "buf.pkl"))
    back = EpisodicReplayBuffer(sc.capacity, device=CPU)
    back.load(str(tmp_path / "buf.pkl"))
    for seed in range(3):
        T.check_sample_episodes(back, model, 2, 7, T.PHIS[sc.phis[0]], seed, materialise=False,
                                mu=sc.mu == "gauss")


@pytest.mark.parametrize("mu_kind", ["cat", "cat_f64", "gauss"])
def test_mu_rows_and_rewards_across_the_ring_end(fake_store, mu_kind):
    T.ring_wrap_case(CPU, mu_kind)


def test_refused_appends_leave_nothing_behind(fake_store):
    T.refusal_case(CPU)
