"""The fused loss of the advantage-learning and DPP agents (AL, PAL, DoublePAL, DPP, DPPL,
DPPGreedy): the same network forwards as their _compute_y_and_t, in the same order (with
factorised-noisy layers the noise stream depends on it), then one ``adv_td_loss`` launch for
the target, |y - t| and the loss.  On CPU, with ``use_fused_loss = False``, or for a subclass
whose target the kernel does not restate, the agent's torch formulation runs instead.

A Q-function that returns a ``QuadraticActionValue`` (NAF) takes ``naf_loss`` instead: the
same forwards, then one ``ops.naf.td_loss`` launch.  DPP and DPPL have no NAF target; with
such a model they fail in their L operator as the reference does."""
import torch

from pfrl_b200.action_value import QuadraticActionValue
from pfrl_b200.ops import losses as fused
from pfrl_b200.utils.modes import evaluating

# the methods that define these agents' targets
_TARGET_METHODS = ("_compute_y_and_t", "_compute_target_values", "_l_operator",
                   "_persistent_target", "_next_q")


def _defining_class(cls, name):
    return next(k for k in cls.__mro__ if name in vars(k))


def fused_mode(agent):
    """The kernel mode (ops.losses.ADV_MODES) that computes ``agent``'s target, or None.

    The mode is the ``_fused_mode`` of the nearest class that sets it.  It holds only while
    no subclass below that class redefines a method the target is built from: a user's own
    ``_l_operator`` or ``_compute_y_and_t`` is not what the kernel computes."""
    cls = type(agent)
    owner = _defining_class(cls, "_fused_mode")
    if owner._fused_mode is None:
        return None
    for name in _TARGET_METHODS:
        if hasattr(cls, name) and not issubclass(owner, _defining_class(cls, name)):
            return None
    return owner._fused_mode


def compute_loss(agent, exp_batch, want_errors, alpha=0.0, eta=1.0):
    """(loss, per-sample |y - t|) of ``agent``: fused on CUDA where ``fused_mode`` allows."""
    mode = fused_mode(agent)
    if mode is None or not (agent.use_fused_loss and exp_batch["reward"].is_cuda):
        return agent._compute_loss_torch(exp_batch, want_errors)
    state, next_state = exp_batch["state"], exp_batch["next_state"]
    qout = agent.model(state)
    if isinstance(qout, QuadraticActionValue):
        if mode in ("dpp", "dppl"):
            agent._l_operator(qout)  # AttributeError: no expectation or q_values
        if not naf_kernel_dtypes(qout):  # the reference's target and loss, from this forward
            y, t = agent._compute_y_and_t(exp_batch, qout=qout)
            return agent._value_loss(y, t, exp_batch, want_errors)
        return naf_loss(agent, exp_batch, qout, mode, alpha=alpha)
    with torch.no_grad():
        next_q = agent.model(next_state).q_values if mode == "double_pal" else None
        target_q = agent.target_model(state).q_values
        target_next_q = agent.target_model(next_state).q_values
    loss, delta, y, _ = fused.adv_td_loss(
        qout.q_values, exp_batch["action"], target_q, target_next_q, exp_batch["reward"],
        exp_batch["discount"], exp_batch["is_state_terminal"], exp_batch.get("weights"), mode,
        alpha=alpha, eta=eta, next_q=next_q, clip_delta=agent.clip_delta,
        mean=agent.batch_accumulator == "mean")
    agent._last_q = y.detach()
    return loss, delta


def naf_kernel_dtypes(qout):
    """Whether the NAF kernel computes the loss of ``qout``: mu, P and V in fp32 (a model in
    another dtype keeps the reference's formulation, as FCQuadraticStateQFunction's head does)."""
    return all(x.dtype == torch.float32 for x in qout.params)


def naf_loss(agent, exp_batch, qout, mode, alpha=0.0):
    """(loss, per-sample |y - t|) of ``agent`` with a NAF Q-function whose output at s is
    ``qout``, for the ``ops.naf.NAF_MODES`` target ``mode``.  The other forwards run in the
    reference's order: [online(s')], [target(s)], target(s'); DoubleDQN's online(s') in eval
    mode, DoublePAL's in the model's own mode."""
    from pfrl_b200.ops import naf

    state, next_state = exp_batch["state"], exp_batch["next_state"]
    with torch.no_grad():
        next_qout = None
        if mode == "double_dqn":
            with evaluating(agent.model):
                next_qout = agent.model(next_state)
        elif mode == "double_pal":
            next_qout = agent.model(next_state)
        target_qout = None if mode in ("dqn", "double_dqn") else agent.target_model(state)
        target_next_qout = agent.target_model(next_state)
    loss, delta, y, _ = naf.td_loss(
        qout, exp_batch["action"], target_next_qout, exp_batch["reward"], exp_batch["discount"],
        exp_batch["is_state_terminal"], exp_batch.get("weights"), mode, target=target_qout,
        next_online=next_qout, alpha=alpha, clip_delta=agent.clip_delta,
        mean=agent.batch_accumulator == "mean")
    agent._last_q = y.detach()
    return loss, delta
