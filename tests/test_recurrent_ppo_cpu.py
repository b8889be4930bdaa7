"""Recurrent PPO on CPU: the sequence helpers, the agent's dataset against the
list-of-dicts helpers, construction errors, save/load, evaluation states and the
untouched non-recurrent path."""
import copy
import itertools
import random
from unittest import mock

import numpy as np
import pytest
import torch
from torch import nn

from pfrl_b200 import nn as pnn
from pfrl_b200.agents import ppo
from pfrl_b200.agents.ppo import PPO, _Span
from pfrl_b200.envs.abc import ABC
from pfrl_b200.nn import RecurrentBranched, RecurrentSequential
from pfrl_b200.ops import rollout
from pfrl_b200.policies import GaussianHeadWithStateIndependentCovariance, SoftmaxCategoricalHead
from pfrl_b200.utils.batch_states import batch_states


def make_model(kind, obs_size=5, n_actions=3, hidden=8):
    """"lstm": RecurrentBranched(LSTM pi, LSTM v) (4 state leaves);
    "gru": GRU trunk + Gaussian head and value (1 leaf)."""
    if kind == "lstm":
        pi = RecurrentSequential(nn.LSTM(num_layers=1, input_size=obs_size, hidden_size=hidden),
                                 nn.Linear(hidden, n_actions), SoftmaxCategoricalHead())
        v = RecurrentSequential(nn.LSTM(num_layers=1, input_size=obs_size, hidden_size=hidden),
                                nn.Linear(hidden, 1))
        return RecurrentBranched(pi, v)
    return RecurrentSequential(
        nn.GRU(num_layers=1, input_size=obs_size, hidden_size=hidden),
        pnn.Branched(
            nn.Sequential(nn.Linear(hidden, n_actions),
                          GaussianHeadWithStateIndependentCovariance(
                              action_size=n_actions, var_type="diagonal",
                              var_func=lambda x: torch.exp(2 * x), var_param_init=0)),
            nn.Linear(hidden, 1)))


def make_agent(kind="lstm", gpu=None, seed=0, n_envs=3, **kw):
    torch.manual_seed(seed)
    discrete = kind == "lstm"
    model = make_model(kind, n_actions=3 if discrete else 2)
    opt = torch.optim.Adam(model.parameters(), lr=1e-2, eps=1e-5)
    args = dict(gpu=gpu, gamma=0.9, lambd=0.95, update_interval=6 * n_envs, minibatch_size=5,
                epochs=2, recurrent=True, max_recurrent_sequence_len=None, clip_eps_vf=0.2,
                standardize_advantages=True)
    args.update(kw)
    return PPO(model, opt, **args)


def drive(agent, n_steps, seed=0, n_envs=3, discrete=True, obs_size=5):
    """Batch acting on a partially observable toy: episodes of random length that
    end by terminal or by reset, observations from a seeded stream."""
    rng = np.random.RandomState(seed)
    obs = [rng.randn(obs_size).astype(np.float32) for _ in range(n_envs)]
    actions = []
    for _ in range(n_steps):
        a = agent.batch_act(obs)
        actions.append(np.asarray(a).copy())
        obs = [rng.randn(obs_size).astype(np.float32) for _ in range(n_envs)]
        reward = rng.randn(n_envs).astype(np.float32)
        done = rng.rand(n_envs) < 0.15
        reset = (~done) & (rng.rand(n_envs) < 0.1)
        agent.batch_observe(obs, reward, done, reset)
    return actions


# ------------------------------------------------------------------ sequence helpers

def _limit_plain(seqs, max_len):
    out = []
    for s in seqs:
        for i in range(0, len(s), max_len):
            out.append(s[i:i + max_len])
    return out


def _subsets_plain(seqs, n):
    flat = [(k, j) for k, s in enumerate(seqs) for j in range(len(s))]
    usable = len(flat) - len(flat) % n
    for i in range(0, usable, n):
        yield flat[i:i + n]


@pytest.mark.parametrize("seed", range(20))
def test_sequence_helpers_on_random_lists_and_spans(seed):
    rng = random.Random(seed)
    seqs = [list(range(100 * k, 100 * k + rng.randint(1, 12))) for k in range(rng.randint(1, 9))]
    max_len = rng.randint(1, 6)
    n_items = rng.randint(1, 15)
    limited = ppo._limit_sequence_length(seqs, max_len)
    assert limited == _limit_plain(seqs, max_len)
    # every minibatch holds n_items items, in order; the remainder is dropped
    got = list(ppo._yield_subset_of_sequences_with_fixed_number_of_items(limited, n_items))
    items = [list(itertools.chain.from_iterable(sub)) for sub in got]
    want = [[seqs_item for seqs_item in
             (limited[k][j] for k, j in part)] for part in _subsets_plain(limited, n_items)]
    assert items == want
    assert all(len(sub) >= 1 and all(len(s) >= 1 for s in sub) for sub in got)
    # spans cut and split exactly like the lists they stand for
    E = 4
    spans = [_Span(k % E, 2 * k, len(s)) for k, s in enumerate(seqs)]

    def slots(span):
        return [(span.t0 + j) * E + span.env for j in range(len(span))]

    lists = [slots(s) for s in spans]
    sp_lim = ppo._limit_sequence_length(spans, max_len)
    assert [slots(s) for s in sp_lim] == ppo._limit_sequence_length(lists, max_len)
    sp_sub = list(ppo._yield_subset_of_sequences_with_fixed_number_of_items(sp_lim, n_items))
    li_sub = list(ppo._yield_subset_of_sequences_with_fixed_number_of_items(
        ppo._limit_sequence_length(lists, max_len), n_items))
    assert [[slots(s) for s in sub] for sub in sp_sub] == li_sub


def test_limit_sequence_length_keeps_short_sequences_as_they_are():
    a, b = [1, 2], [3, 4, 5, 6, 7]
    out = ppo._limit_sequence_length([a, b], 2)
    assert out[0] is a and out[1:] == [[3, 4], [5, 6], [7]]


def test_gae_and_explained_variance_helpers():
    rng = np.random.RandomState(0)
    ep = [dict(reward=float(r), nonterminal=1.0, v_pred=float(v), next_v_pred=float(nv))
          for r, v, nv in rng.randn(6, 3)]
    ep[-1]["nonterminal"] = 0.0
    ppo._add_advantage_and_value_target_to_episode(ep, 0.9, 0.8)
    adv = 0.0
    for tr in reversed(ep):
        adv = tr["reward"] + 0.9 * tr["nonterminal"] * tr["next_v_pred"] - tr["v_pred"] \
            + 0.9 * 0.8 * adv
        assert tr["adv"] == pytest.approx(adv, rel=1e-12)
        assert tr["v_teacher"] == pytest.approx(adv + tr["v_pred"], rel=1e-12)
    t = np.array([tr["v_teacher"] for tr in ep])
    y = np.array([tr["v_pred"] for tr in ep])
    assert ppo._compute_explained_variance(ep) == pytest.approx(1 - np.var(t - y) / np.var(t))
    for tr in ep:
        tr["v_teacher"] = 1.0
    assert np.isnan(ppo._compute_explained_variance(ep))


# -------------------------------------------------- the agent against the dict helpers

def _record_transitions(agent):
    """The transition dicts the reference would have stored, per episode in memory
    order (states rebuilt from the agent's ring rows), and their (t, e) slots."""
    E = agent._rstates[0].shape[0]
    spec, nest = agent._state_spec, agent._state_nest
    T = len(agent._rewards)

    def state(rows, side, present):
        if not present:
            return None
        return ppo._state_from_leaves(nest, [
            rows[side, off:off + d0 * inner].reshape(d0, inner)
            for off, (d0, inner) in zip(spec.offsets, spec.shapes)])

    episodes, slots = [], []
    for span in agent._episode_spans(T, E):
        e = span.env
        ts = range(span.t0, span.t0 + len(span))
        slots.append([(t, e) for t in ts])
        episodes.append([dict(
            state=agent._states[t][e], action=agent._actions[t][e].item(),
            reward=float(agent._rewards[t][e]), next_state=agent._next_states[t][e],
            nonterminal=float(agent._nonterminal[t][e]),
            recurrent_state=state(agent._rstates[t][e], 0, agent._rpresent[t]),
            next_recurrent_state=state(agent._rstates[t][e], 1, True)) for t in ts])
    return episodes, slots


def test_dataset_matches_make_dataset_recurrent():
    """The spans' dataset pass (pack, two forwards, scatter back, GAE) gives the
    values _make_dataset_recurrent writes into the reference's transition dicts."""
    agent = make_agent("lstm", update_interval=10 ** 9)
    drive(agent, 9)
    episodes, slots = _record_transitions(agent)
    ref_eps = copy.deepcopy(episodes)
    ppo._make_dataset_recurrent(ref_eps, agent.model, lambda x: x, batch_states, None,
                                agent.gamma, agent.lambd, 4, "cpu")
    seen = {}
    real_gae = ppo._gae_torch

    def spy(reward, nonterminal, v, v_next, cut, gamma, lambd):
        adv, vt = real_gae(reward, nonterminal, v, v_next, cut, gamma, lambd)
        seen.update(v=v.clone(), v_next=v_next.clone(), adv=adv.clone())
        return adv, vt

    with mock.patch.object(ppo, "_gae_torch", spy):
        agent._update_recurrent_from_rollout()
    T, E = seen["v"].shape
    assert sum(len(ep) for ep in ref_eps) == T * E
    for ep_slots, ep in zip(slots, ref_eps):
        for (t, e), tr in zip(ep_slots, ep):
            assert seen["v"][t, e].item() == pytest.approx(tr["v_pred"], abs=1e-6)
            assert seen["v_next"][t, e].item() == pytest.approx(tr["next_v_pred"], abs=1e-6)
            assert seen["adv"][t, e].item() == pytest.approx(tr["adv"], abs=1e-5)


# ----------------------------------------------------------------- agent behaviour

@pytest.mark.parametrize("kw", [dict(cuda_graph=True), dict(grad_sync=lambda m: None),
                                dict(stats_sync=lambda a: a)])
def test_recurrent_construction_errors(kw):
    with pytest.raises(ValueError):
        make_agent("lstm", **kw)


@pytest.mark.parametrize("kind", ["lstm", "gru"])
def test_recurrent_agent_trains_on_cpu(kind):
    agent = make_agent(kind, max_recurrent_sequence_len=3 if kind == "gru" else None,
                       minibatch_size=7, lambd=0.5 if kind == "gru" else 0.95,
                       obs_normalizer=pnn.EmpiricalNormalization(5) if kind == "gru" else None)
    before = [p.detach().clone() for p in agent.model.parameters()]
    drive(agent, 20, discrete=kind == "lstm")
    stats = dict(agent.get_statistics())
    assert stats["n_updates"] > 0
    assert np.isfinite(stats["average_value_loss"]) and np.isfinite(stats["average_policy_loss"])
    assert any(not torch.equal(a, b) for a, b in zip(before, agent.model.parameters()))
    # the rollout is cleared after every update
    assert len(agent._rstates) == len(agent._rewards) < 6


def test_minibatches_hold_exactly_minibatch_size_transitions():
    agent = make_agent("lstm", max_recurrent_sequence_len=2, minibatch_size=4, epochs=3)
    sizes = []
    real = PPO._gather_sequences

    def spy(self, spans, E, columns, index=False, states=None):
        out = real(self, spans, E, columns, index, states)
        if not index:
            sizes.append(sum(len(s) for s in spans))
            lens = sorted((len(s) for s in spans), reverse=True)
            assert out[3].tolist() == rollout.packed_layout(lens)[0].tolist()
        return out

    with mock.patch.object(PPO, "_gather_sequences", spy):
        drive(agent, 6)
    N = 6 * 3
    assert sizes == [4] * ((N // 4) * 3)
    assert agent.n_updates == len(sizes)


def test_save_load_round_trip(tmp_path):
    agent = make_agent("lstm")
    drive(agent, 8)
    agent.save(str(tmp_path / "a"))
    other = make_agent("lstm", seed=1)
    other.load(str(tmp_path / "a"))
    for a, b in zip(agent.model.state_dict().values(), other.model.state_dict().values()):
        assert torch.equal(a, b)
    obs = [np.ones(5, np.float32)] * 3
    with agent.eval_mode(), other.eval_mode():
        torch.manual_seed(3)
        x = agent.batch_act(obs)
        torch.manual_seed(3)
        y = other.batch_act(obs)
    assert np.array_equal(x, y)


def test_eval_acting_uses_and_resets_its_own_states():
    agent = make_agent("lstm")
    drive(agent, 2)
    train_states = agent.train_recurrent_states
    obs = [np.ones(5, np.float32)] * 3
    with agent.eval_mode():
        agent.batch_act(obs)
        assert agent.test_recurrent_states is not None
        assert agent.train_recurrent_states is train_states
        agent.batch_observe(obs, [0.0] * 3, [True, False, False], [False, False, True])
        for leaf in ppo._state_leaves(agent.test_recurrent_states)[0]:
            assert torch.count_nonzero(leaf[:, 0]) == 0 and torch.count_nonzero(leaf[:, 2]) == 0
            assert torch.count_nonzero(leaf[:, 1]) > 0
    assert agent.train_recurrent_states is train_states
    assert len(agent._rstates) == len(agent._rewards)


def test_train_states_are_masked_at_episode_ends_and_stored_before_masking():
    agent = make_agent("lstm", update_interval=10 ** 9)
    obs = [np.ones(5, np.float32) * k for k in range(3)]
    agent.batch_act(obs)
    assert agent._cur_rs[1] is False  # the state before the first step is None
    agent.batch_observe(obs, [0.0] * 3, [True, False, False], [False, False, False])
    row = agent._rstates[0]
    assert torch.count_nonzero(row[:, 0]) == 0 and torch.count_nonzero(row[0, 1]) > 0
    for leaf in ppo._state_leaves(agent.train_recurrent_states)[0]:
        assert torch.count_nonzero(leaf[:, 0]) == 0 and torch.count_nonzero(leaf[:, 1]) > 0
    masked = agent.train_recurrent_states
    agent.batch_act(obs)
    assert agent._cur_rs[1] is True
    assert torch.equal(agent._cur_rs[0][:, 0], agent._state_spec.flatten(
        ppo._state_leaves(masked)[0]))


def test_non_recurrent_ppo_never_enters_the_recurrent_path():
    torch.manual_seed(0)
    model = pnn.Branched(nn.Sequential(nn.Linear(5, 3), SoftmaxCategoricalHead()),
                         nn.Linear(5, 1))
    agent = PPO(model, torch.optim.Adam(model.parameters()), update_interval=12,
                minibatch_size=4, epochs=2)
    boom = mock.Mock(side_effect=AssertionError("recurrent path"))
    with mock.patch.object(PPO, "_update_recurrent_from_rollout", boom), \
            mock.patch.object(PPO, "_recurrent_step", boom), \
            mock.patch.object(PPO, "_gather_sequences", boom):
        drive(agent, 8)
    assert agent.n_updates > 0 and not agent._rstates and agent.recurrent is False


def test_abc_partially_observable_runs():
    env = ABC(size=2, discrete=True, partially_observable=True)
    agent = make_agent("lstm", n_envs=1, update_interval=16)
    agent.model = make_model("lstm", obs_size=env.observation_space.low.size, n_actions=3)
    agent.optimizer = torch.optim.Adam(agent.model.parameters(), lr=1e-2)
    obs = env.reset()
    for _ in range(40):
        a = agent.act(obs)
        obs, r, done, _ = env.step(a)
        agent.observe(obs, r, done, False)
        if done:
            obs = env.reset()
    assert agent.n_updates > 0


def test_model_whose_state_holds_no_tensors():
    """A RecurrentSequential of feed-forward modules only has an empty state; the agent
    keeps no state ring and passes None as the first state, as the reference does."""
    torch.manual_seed(0)
    model = RecurrentSequential(
        pnn.Branched(nn.Sequential(nn.Linear(5, 3), SoftmaxCategoricalHead()), nn.Linear(5, 1)))
    agent = PPO(model, torch.optim.Adam(model.parameters()), update_interval=12,
                minibatch_size=4, epochs=2, recurrent=True, max_recurrent_sequence_len=2)
    drive(agent, 9)
    assert agent.n_updates > 0 and agent._state_spec is None
