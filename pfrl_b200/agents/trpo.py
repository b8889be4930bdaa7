"""Trust Region Policy Optimization on the device rollout.

Public surface = pfrl/agents/trpo.py (constructor arguments, saved_attributes,
batch_act / batch_observe, statistics names and order).  Non-recurrent only.

The rollout, its episode segmentation, the dataset order and the dataset pass
(two forwards, the fused GAE kernel) are PPO's (``ppo._DeviceRollout``).  The
value function is trained on fixed-size minibatches of PPO's index stream.

The policy update is the reference's full-batch pass (trpo.py:415-699).  With
an fp32 Gaussian (``Independent(Normal)``) or categorical policy on CUDA it runs
without a device-to-host copy or synchronisation (csrc/trpo.cu):
  * one forward, and the objective kernel for the gain and d gain / d(dist
    params), back-propagated once to the parameters;
  * conjugate gradient (``utils.conjugate_gradient``) through the Gauss-Newton
    Fisher-vector product J^T M J v + damping v: J v by forward-mode AD
    (``torch.func.jvp``), M by the Fisher kernel, J^T by one backward on the
    retained forward graph (the reference differentiates twice);
  * the KL-scaled full step in one kernel;
  * every line-search candidate theta_old + 2^-i full_step evaluated with
    ``torch.func.functional_call`` (the module is not mutated per candidate),
    then one kernel picks the first acceptable one and writes the parameters.
The reference's per-candidate log lines are written after the update from one
copy of the candidates' values, and only when the logger takes INFO.  With ``cuda_graph=True`` the
fused policy update and the value-function minibatch step are each replayed as one
CUDA graph.

Everything else (CPU, ``use_fused = False``, other distributions, fp64 or half
policies) runs the
reference's algorithm in the reference's operation order.
"""
from logging import INFO, getLogger

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

from pfrl_b200 import agent
from pfrl_b200.agents._graph import CapturedStep
from pfrl_b200.agents.dqn import _DeviceRing
from pfrl_b200.agents.ppo import (  # NOQA
    _DeviceRollout, _compute_explained_variance, _make_dataset, _yield_minibatch_indices,
    _yield_minibatches,
)
from pfrl_b200.agents.soft_actor_critic import mode_of_distribution
from pfrl_b200.nn.branched import Branched
from pfrl_b200.ops import trpo as fused
from pfrl_b200.utils.batch_states import batch_states
from pfrl_b200.utils.clip_l2_grad_norm import clip_l2_grad_norm_
from pfrl_b200.utils.conjugate_gradient import _conjugate_gradient_torch, conjugate_gradient
from pfrl_b200.utils.modes import evaluating, no_distribution_validation


def _flatten_and_concat_variables(vs):
    """Flatten and concat variables to make a single flat vector variable."""
    return torch.cat([torch.flatten(v) for v in vs], dim=0)


def _split_and_reshape_to_ndarrays(flat_v, sizes, shapes):
    """Split and reshape a single flat vector to make a list of tensors."""
    vs = torch.split(flat_v, sizes)
    return [v.reshape(shape) for v, shape in zip(vs, shapes)]


def _replace_params_data(params, new_params_data):
    """Replace data of params with new data."""
    for param, new_param_data in zip(params, new_params_data):
        assert param.shape == new_param_data.shape
        assert isinstance(param, nn.Parameter)
        param.data.copy_(new_param_data)


def _hessian_vector_product(flat_grads, params, vec):
    """Hessian-vector product by backprop through ``flat_grads`` (made with
    create_graph=True)."""
    vec = vec.detach()
    grads = torch.autograd.grad([torch.sum(flat_grads * vec)], params, retain_graph=True)
    assert all(grad is not None for grad in grads), "The Hessian-vector product contains None."
    return _flatten_and_concat_variables(grads)


def _mean_or_nan(xs):
    return np.mean(xs) if xs else np.nan


def _distribution_params(distrib):
    """(kind, [params]) for the distributions the kernels cover, else None."""
    D = torch.distributions
    if isinstance(distrib, D.Independent) and type(distrib.base_dist) is D.Normal \
            and distrib.reinterpreted_batch_ndims == 1 and distrib.base_dist.loc.dim() == 2:
        return fused.GAUSSIAN, [distrib.base_dist.loc, distrib.base_dist.scale]
    if type(distrib) is D.Categorical and distrib.logits.dim() == 2:
        return fused.CATEGORICAL, [distrib.logits]
    return None


def _fp32_on(device, tensors):
    return all(t.dtype == torch.float32 and t.device == device for t in tensors)


class _RecordRing(_DeviceRing):
    """Window of per-update records (accepted KL, step size).  Host floats until the first
    device value; from then on every value, host floats included, lives in the device
    buffer and so does the count, so that an append may depend on a device flag (the KL of
    an accepted step) without a synchronisation."""

    def _to_device(self, device):
        vals = list(self.host)
        self.buf = torch.zeros(self.maxlen, device=device)
        if vals:
            self.buf[:len(vals)] = torch.tensor(vals, dtype=torch.float32)
        # fill_ with a Python int is a kernel, not a host-to-device copy
        self._n = torch.zeros((), dtype=torch.int64, device=device).fill_(len(vals))
        self.host.clear()

    def append_if(self, value, flag):
        """Append the device scalar ``value`` where the device bool ``flag`` is set."""
        if self.buf is None:
            self._to_device(value.device)
        pos = (self._n % self.maxlen).view(1)
        self.buf.index_put_((pos,), torch.where(flag, value.float(), self.buf[pos]).view(1))
        self._n += flag.to(torch.int64)

    def append(self, value):
        on_device = isinstance(value, torch.Tensor) and value.is_cuda
        if self.buf is None and not on_device:
            self.host.append(float(value))
            return
        if not on_device:
            value = torch.tensor(float(value), device=self.buf.device)
        self.append_if(value.reshape(()), torch.ones((), dtype=torch.bool, device=value.device))

    def extend(self, values):
        for v in (values.reshape(-1) if isinstance(values, torch.Tensor) else values):
            self.append(v)

    def mean(self):
        if self.buf is None:
            return super().mean()
        n = min(int(self._n), self.maxlen)
        return float(self.buf[:n].mean().item()) if n else np.nan

    def __len__(self):
        return len(self.host) if self.buf is None else min(int(self._n), self.maxlen)


class TRPO(_DeviceRollout, agent.AttributeSavingMixin, agent.BatchAgent):
    """Trust Region Policy Optimization (https://arxiv.org/abs/1502.05477) with GAE.

    Arguments as the reference's ``pfrl.agents.TRPO``.  ``recurrent=True`` is not
    supported here.  ``cuda_graph=True`` (CUDA only) replays the value-function minibatch
    step and the fused policy update as CUDA graphs.

    Statistics: average_value, average_entropy, average_kl, average_policy_step_size,
    explained_variance.
    """

    saved_attributes = ("policy", "vf", "vf_optimizer", "obs_normalizer")

    def __init__(self, policy, vf, vf_optimizer, obs_normalizer=None, gpu=None, gamma=0.99,
                 lambd=0.95, phi=lambda x: x, entropy_coef=0.01, update_interval=2048,
                 max_kl=0.01, vf_epochs=3, vf_batch_size=64, standardize_advantages=True,
                 batch_states=batch_states, recurrent=False, max_recurrent_sequence_len=None,
                 line_search_max_backtrack=10, conjugate_gradient_max_iter=10,
                 conjugate_gradient_damping=1e-2, act_deterministically=False,
                 max_grad_norm=None, value_stats_window=1000, entropy_stats_window=1000,
                 kl_stats_window=100, policy_step_size_stats_window=100,
                 logger=getLogger(__name__), cuda_graph=False):
        if recurrent:
            raise NotImplementedError(
                "TRPO(recurrent=True) is not implemented in pfrl_b200: use a feed-forward "
                "policy and value function (recurrent PPO is available as PPO(recurrent=True))")
        self.policy = policy
        self.vf = vf
        self.vf_optimizer = vf_optimizer
        self.obs_normalizer = obs_normalizer
        self.gamma = gamma
        self.lambd = lambd
        self.phi = phi
        self.entropy_coef = entropy_coef
        self.update_interval = update_interval
        self.max_kl = max_kl
        self.vf_epochs = vf_epochs
        self.vf_batch_size = vf_batch_size
        self.standardize_advantages = standardize_advantages
        self.batch_states = batch_states
        self.recurrent = False
        self.max_recurrent_sequence_len = max_recurrent_sequence_len
        self.line_search_max_backtrack = line_search_max_backtrack
        self.conjugate_gradient_max_iter = conjugate_gradient_max_iter
        self.conjugate_gradient_damping = conjugate_gradient_damping
        self.act_deterministically = act_deterministically
        self.max_grad_norm = max_grad_norm
        self.logger = logger
        if gpu is not None and gpu >= 0:
            assert torch.cuda.is_available()
            self.device = torch.device("cuda:{}".format(gpu))
            self.policy.to(self.device)
            self.vf.to(self.device)
            if self.obs_normalizer is not None:
                self.obs_normalizer.to(self.device)
        else:
            self.device = torch.device("cpu")
        self.model = Branched(policy, vf)
        self.use_fused = True
        self.value_record = _DeviceRing(value_stats_window)
        self.entropy_record = _DeviceRing(entropy_stats_window)
        self.kl_record = _RecordRing(kl_stats_window)
        self.policy_step_size_record = _RecordRing(policy_step_size_stats_window)
        self.explained_variance = np.nan
        self.train_recurrent_states = None
        self.test_recurrent_states = None
        self._rollout_clear()
        self._cur_state = None
        self._cur_action = None
        self._line_search_log = None
        self._policy_kind = None  # the kernels' distribution kind, False if not covered
        # Optional (cuda_graph=True): the value-function minibatch step and the fused policy
        # update (fixed shapes for a given N, CG iterations and backtracks) are each
        # captured and replayed
        self._vf_graph = self._policy_graph = None
        if cuda_graph and self.device.type == "cuda":
            self._vf_graph = CapturedStep(3, (vf_optimizer,))
            self._policy_graph = CapturedStep(2)

    # ----------------------------------------------------------------- acting
    def batch_act(self, batch_obs):
        raw = self.batch_states(batch_obs, self.device, self.phi)
        feat = self.obs_normalizer(raw, update=False) if self.obs_normalizer else raw
        with torch.no_grad(), evaluating(self.model):
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

    def batch_observe(self, batch_obs, batch_reward, batch_done, batch_reset):
        if not self.training:
            return
        steps = self._record_observe(batch_obs, batch_reward, batch_done, batch_reset)
        if steps * len(batch_obs) >= self.update_interval:
            self._update_from_rollout()

    # ------------------------------------------------------------ the update
    def _update_from_rollout(self):
        d = self._rollout_dataset()
        E, N = d["E"], d["N"]
        order = d["order"]
        idx = torch.as_tensor(order, device=self.device)
        adv, v_teacher = d["adv"].reshape(N), d["v_teacher"].reshape(N)
        norm = self.obs_normalizer
        if norm:  # _update_obs_normalizer: the dataset's states, in dataset order
            norm.experience(d["flat_s"][idx])
        obs = norm(d["flat_s"], update=False) if norm else d["flat_s"]
        # the policy's full batch in dataset order (trpo.py:432-451)
        s, a = obs[idx], d["flat_a"][idx]
        lp_old, adv_b = d["log_probs_old"][idx], adv[idx]
        self._update_policy(s, a, lp_old, adv_b,
                            d["stats"] if self.standardize_advantages else None)
        self._update_vf(obs, v_teacher, order)
        self._explained_variance_from(v_teacher, d["v_old"])
        self._rollout_clear(E)
        if self._line_search_log is not None and self.logger.isEnabledFor(INFO):
            self._log_line_search(*self._line_search_log)

    def _update_policy(self, states, actions, log_prob_old, advs, adv_stats):
        """The fused update where it applies, else the reference's formulation.
        ``adv_stats`` (mean, std of ``advs``) is given when advantages are standardised."""
        self._line_search_log = None
        if not (self.use_fused and self.device.type == "cuda"
                and self._update_policy_fused(states, actions, log_prob_old, advs, adv_stats)):
            self._update_policy_torch(states, actions, log_prob_old, self._standardized(advs))

    def _standardized(self, advs):
        if not self.standardize_advantages:
            return advs
        std_advs, mean_advs = torch.std_mean(advs, unbiased=False)
        return (advs - mean_advs) / (std_advs + 1e-8)

    def _update_vf(self, obs, v_teacher, order):
        """trpo.py:387-413 over PPO's minibatch index stream."""
        mbs = list(_yield_minibatch_indices(order, self.vf_batch_size, self.vf_epochs))
        # every minibatch has vf_batch_size indices: one upload for the whole stream
        all_idx = torch.as_tensor(np.asarray(mbs, dtype=np.int64), device=self.device)
        if self._vf_graph is not None:
            self._update_vf_graphed(obs, v_teacher, all_idx)
            return
        for i in all_idx:
            self._vf_step(obs[i], v_teacher[i])

    def _vf_step(self, states, vs_teacher):
        vs_pred = self.vf(states)
        vf_loss = F.mse_loss(vs_pred, vs_teacher[..., None])
        self.vf.zero_grad()
        vf_loss.backward()
        if self.max_grad_norm is not None:
            clip_l2_grad_norm_(self.vf.parameters(), self.max_grad_norm)
        self.vf_optimizer.step()

    def _update_vf_graphed(self, obs, v_teacher, all_idx):
        """The minibatch steps over persistent buffers, loaded once per update
        (PPO._minibatches_graphed)."""
        g = self._vf_graph.load((self.max_grad_norm, self.vf_batch_size),
                                dict(obs=obs, vt=v_teacher, idx=all_idx[0]))
        for row in all_idx:
            g["idx"].copy_(row)
            self._vf_graph.run(lambda g: self._vf_step(g["obs"][g["idx"]], g["vt"][g["idx"]]))

    def _compute_gain(self, log_prob, log_prob_old, entropy, advs):
        """Compute a gain to maximize."""
        prob_ratio = torch.exp(log_prob - log_prob_old)
        mean_entropy = torch.mean(entropy)
        surrogate_gain = torch.mean(prob_ratio * advs)
        return surrogate_gain + self.entropy_coef * mean_entropy

    # ------------------------------------------------- reference formulation
    def _update_policy_torch(self, states, actions, log_prob_old, advs):
        """trpo.py:422-477, 557-699 in the reference's operation order."""
        action_distrib = self.policy(states)
        gain = self._compute_gain(log_prob=action_distrib.log_prob(actions),
                                  log_prob_old=log_prob_old, entropy=action_distrib.entropy(),
                                  advs=advs)
        with torch.no_grad():
            action_distrib_old = self.policy(states)
        full_step = self._compute_kl_constrained_step(action_distrib, action_distrib_old, gain)
        self._line_search(full_step, states, actions, log_prob_old, advs, action_distrib_old,
                          gain)

    def _compute_kl_constrained_step(self, action_distrib, action_distrib_old, gain):
        policy_params = list(self.policy.parameters())
        kl = torch.mean(torch.distributions.kl_divergence(action_distrib_old, action_distrib))
        kl_grads = torch.autograd.grad([kl], policy_params, create_graph=True)
        assert all(g is not None for g in kl_grads), \
            "The gradient contains None. The policy may have unused parameters."
        flat_kl_grads = _flatten_and_concat_variables(kl_grads)

        def fisher_vector_product_func(vec):
            vec = torch.as_tensor(vec)
            fvp = _hessian_vector_product(flat_kl_grads, policy_params, vec)
            return fvp + self.conjugate_gradient_damping * vec

        gain_grads = torch.autograd.grad([gain], policy_params, create_graph=True)
        assert all(g is not None for g in gain_grads), \
            "The gradient contains None. The policy may have unused parameters."
        flat_gain_grads = _flatten_and_concat_variables(gain_grads).detach()
        step_direction = _conjugate_gradient_torch(fisher_vector_product_func, flat_gain_grads,
                                       max_iter=self.conjugate_gradient_max_iter)
        dId = float(step_direction.dot(fisher_vector_product_func(step_direction)))
        scale = (2.0 * self.max_kl / (dId + 1e-8)) ** 0.5
        return scale * step_direction

    def _line_search(self, full_step, states, actions, log_prob_old, advs, action_distrib_old,
                     gain):
        policy_params = list(self.policy.parameters())
        sizes = [p.numel() for p in policy_params]
        shapes = [p.shape for p in policy_params]
        step_size = 1.0
        flat_params = _flatten_and_concat_variables(policy_params).detach()
        for i in range(self.line_search_max_backtrack + 1):
            self.logger.info("Line search iteration: %s step size: %s", i, step_size)
            new_flat_params = flat_params + step_size * full_step
            _replace_params_data(policy_params,
                                 _split_and_reshape_to_ndarrays(new_flat_params, sizes, shapes))
            with torch.no_grad(), evaluating(self.policy):
                new_action_distrib = self.policy(states)
                new_gain = self._compute_gain(
                    log_prob=new_action_distrib.log_prob(actions), log_prob_old=log_prob_old,
                    entropy=new_action_distrib.entropy(), advs=advs)
                new_kl = torch.mean(torch.distributions.kl_divergence(action_distrib_old,
                                                                      new_action_distrib))
            improve = float(new_gain) - float(gain)
            self.logger.info("Surrogate objective improve: %s", improve)
            self.logger.info("KL divergence: %s", float(new_kl))
            if not torch.isfinite(new_gain):
                self.logger.info("Surrogate objective is not finite. Bakctracking...")
            elif not torch.isfinite(new_kl):
                self.logger.info("KL divergence is not finite. Bakctracking...")
            elif improve < 0:
                self.logger.info("Surrogate objective didn't improve. Bakctracking...")
            elif float(new_kl) > self.max_kl:
                self.logger.info("KL divergence exceeds max_kl. Bakctracking...")
            else:
                self.kl_record.append(float(new_kl))
                self.policy_step_size_record.append(step_size)
                break
            step_size *= 0.5
        else:
            self.logger.info("Line search couldn't find a good step size. The policy was not"
                             " updated.")
            self.policy_step_size_record.append(0.0)
            _replace_params_data(policy_params,
                                 _split_and_reshape_to_ndarrays(flat_params, sizes, shapes))

    # ------------------------------------------------------ the fused update
    def _fused_kind(self, states):
        """The kernels' kind of the policy's distribution, or False where they do not apply:
        a distribution they do not cover, or a policy whose parameters or distribution
        parameters are not all fp32 on the agent's device (the kernels are fp32; an fp64 or
        half policy takes the reference's formulation).  The distribution is classified
        once, on a one-row forward; the parameters are checked on every call."""
        if not _fp32_on(self.device, self.policy.parameters()):
            return False
        if self._policy_kind is None:
            with torch.no_grad(), evaluating(self.policy), no_distribution_validation():
                kind_params = _distribution_params(self.policy(states[:1]))
            covered = kind_params is not None and _fp32_on(self.device, kind_params[1])
            self._policy_kind = kind_params[0] if covered else False
        return self._policy_kind

    def _update_policy_fused(self, states, actions, log_prob_old, advs, adv_stats):
        """The update on the kernels; False (and nothing done) for other distributions."""
        kind = self._fused_kind(states)
        if kind is False:
            return False
        if self._policy_graph is not None:
            out = self._policy_kernels_graphed(kind, states, actions, log_prob_old, advs,
                                               adv_stats)
        else:
            out = self._policy_kernels(kind, states, actions, log_prob_old, advs, adv_stats)
        cand_out, gain_out, record = out
        self.kl_record.append_if(record[0], record[2] > 0)
        self.policy_step_size_record.append(record[1])
        self._line_search_log = out
        return True

    def _policy_kernels(self, kind, states, actions, log_prob_old, advs, adv_stats):
        """Gain and its gradient, CG through the Fisher-vector product, the KL-scaled step,
        every line-search candidate, the decision and the parameter write.  No host
        synchronisation.  Returns (candidates [C, 3], gain [3], record [3])."""
        names = [n for n, _ in self.policy.named_parameters()]
        params = [p for _, p in self.policy.named_parameters()]
        sizes = [p.numel() for p in params]
        shapes = [p.shape for p in params]
        theta_old = _flatten_and_concat_variables([p.detach() for p in params])
        ent = self.entropy_coef
        with no_distribution_validation():
            kind_got, dparams = _distribution_params(self.policy(states))
            assert kind_got == kind
            old = [x.detach() for x in dparams]
            gain, gain_out = fused.gain(kind, dparams, old, actions, log_prob_old, advs,
                                        adv_stats, ent)
            flat_gain_grads = _flatten_and_concat_variables(
                torch.autograd.grad([gain], params, retain_graph=True))
            fisher_vector_product = self._fisher_vector_product(states, kind, dparams, old)
            x = conjugate_gradient(fisher_vector_product, flat_gain_grads,
                                   max_iter=self.conjugate_gradient_max_iter)
            full_step, _ = fused.cg_step(x, fisher_vector_product(x), self.max_kl)
            del gain, dparams

            n_cand = self.line_search_max_backtrack + 1
            steps = torch.pow(0.5, torch.arange(n_cand, dtype=torch.float32,
                                                device=theta_old.device))
            cands = theta_old[None] + steps[:, None] * full_step[None]
            cand_out = torch.empty(n_cand, 3, dtype=torch.float32, device=theta_old.device)
            with torch.no_grad(), evaluating(self.policy):
                for i in range(n_cand):
                    ps = _split_and_reshape_to_ndarrays(cands[i], sizes, shapes)
                    d = torch.func.functional_call(self.policy, dict(zip(names, ps)), (states,))
                    cand_out[i] = fused.objective(kind, _distribution_params(d)[1], old, actions,
                                                  log_prob_old, advs, adv_stats, ent)
        theta, record = fused.line_search(cand_out, gain_out, self.max_kl, theta_old, full_step)
        with torch.no_grad():
            torch._foreach_copy_(params, _split_and_reshape_to_ndarrays(theta, sizes, shapes))
        return cand_out, gain_out, record

    def _policy_kernels_graphed(self, kind, states, actions, log_prob_old, advs, adv_stats):
        """_policy_kernels over persistent input buffers."""
        inputs = dict(s=states, a=actions, lp=log_prob_old, adv=advs)
        if adv_stats is not None:
            inputs["stats"] = adv_stats
        self._policy_graph.load((kind, self.max_kl, self.entropy_coef,
                                 self.conjugate_gradient_max_iter,
                                 self.conjugate_gradient_damping,
                                 self.line_search_max_backtrack), inputs)
        return self._policy_graph.run(lambda g: self._policy_kernels(
            kind, g["s"], g["a"], g["lp"], g["adv"], g.get("stats")))

    def _fisher_vector_product(self, states, kind, dparams, old):
        """v -> J^T (M J v) + damping v at the current parameters: J v by forward-mode AD
        through ``functional_call``, M by the Fisher kernel, J^T by one backward on the
        retained graph of ``dparams`` (the distribution parameters of ``states``)."""
        names = [n for n, _ in self.policy.named_parameters()]
        params = [p for _, p in self.policy.named_parameters()]
        sizes = [p.numel() for p in params]
        shapes = [p.shape for p in params]
        primals = tuple(p.detach() for p in params)
        with_grad = [i for i, x in enumerate(dparams) if x.requires_grad]

        def dist_params_at(*ps):
            d = torch.func.functional_call(self.policy, dict(zip(names, ps)), (states,))
            return tuple(_distribution_params(d)[1])

        def fisher_vector_product(vec):
            tangents = tuple(_split_and_reshape_to_ndarrays(vec, sizes, shapes))
            _, u = torch.func.jvp(dist_params_at, primals, tangents)
            m = fused.fisher(kind, old, list(u))
            g = torch.autograd.grad([dparams[i] for i in with_grad], params,
                                    [m[i] for i in with_grad], retain_graph=True)
            return _flatten_and_concat_variables(g) + self.conjugate_gradient_damping * vec

        return fisher_vector_product

    def _log_line_search(self, cand_out, gain_out, record):
        """The reference's per-candidate log lines (trpo.py:649-693) from the device records."""
        host = torch.cat([cand_out.reshape(-1), gain_out[:1], record]).cpu().tolist()
        n = cand_out.numel()
        c, g0, rec = host[:n], host[n], host[n + 1:]
        step_size = 1.0
        for i, (g, kl) in enumerate(zip(c[0::3], c[1::3])):
            self.logger.info("Line search iteration: %s step size: %s", i, step_size)
            improve = g - g0
            self.logger.info("Surrogate objective improve: %s", improve)
            self.logger.info("KL divergence: %s", kl)
            if not np.isfinite(g):
                self.logger.info("Surrogate objective is not finite. Bakctracking...")
            elif not np.isfinite(kl):
                self.logger.info("KL divergence is not finite. Bakctracking...")
            elif improve < 0:
                self.logger.info("Surrogate objective didn't improve. Bakctracking...")
            elif kl > self.max_kl:
                self.logger.info("KL divergence exceeds max_kl. Bakctracking...")
            else:
                return
            step_size *= 0.5
        assert rec[2] == 0
        self.logger.info("Line search couldn't find a good step size. The policy was not"
                         " updated.")

    def get_statistics(self):
        if self.explained_variance is None:
            self.explained_variance = float(self._explained_variance_t.item())
        return [
            ("average_value", self.value_record.mean()),
            ("average_entropy", self.entropy_record.mean()),
            ("average_kl", self.kl_record.mean()),
            ("average_policy_step_size", self.policy_step_size_record.mean()),
            ("explained_variance", self.explained_variance),
        ]

