"""Diff this package's public API against the reference's (build container
only: imports /root/reference through oracle/refimport.py).

For every class / function on or next to the rebuilt path: constructor /
function parameters (names, order, defaults; extra keyword-only parameters of
ours are allowed), and for the main classes every public method (presence and
parameter names).  Prints the differences; exit status 0 means drop-in.

    python tools/api_diff.py
"""
import inspect
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.refimport import import_reference  # noqa: E402

CALLABLES = """
agents.DQN agents.DoubleDQN agents.CategoricalDQN agents.CategoricalDoubleDQN agents.IQN
agents.AL agents.PAL agents.DoublePAL agents.DPP agents.dpp.DPPL agents.dpp.DPPGreedy
agents.PPO agents.A2C agents.SoftActorCritic agents.TD3 agents.DDPG agents.A3C
replay_buffers.ReplayBuffer replay_buffers.PrioritizedReplayBuffer replay_buffers.EpisodicReplayBuffer
nn.RecurrentSequential nn.RecurrentBranched replay_buffer.batch_recurrent_experiences
replay_buffer.random_subseq replay_buffer.batch_experiences replay_buffer.ReplayUpdater utils.batch_states
experiments.train_agent_batch experiments.train_agent_batch_with_evaluation
experiments.train_agent experiments.train_agent_with_evaluation
experiments.evaluator.Evaluator experiments.LinearInterpolationHook
explorers.ConstantEpsilonGreedy explorers.LinearDecayEpsilonGreedy
explorers.ExponentialDecayEpsilonGreedy explorers.AdditiveGaussian explorers.AdditiveOU
explorers.Boltzmann nn.MLP nn.EmpiricalNormalization nn.FactorizedNoisyLinear
nn.to_factorized_noisy nn.LargeAtariCNN nn.SmallAtariCNN nn.Branched nn.BoundByTanh
q_functions.DuelingDQN q_functions.DistributionalDuelingDQN
q_functions.FCStateQFunctionWithDiscreteAction
q_functions.DistributionalFCStateQFunctionWithDiscreteAction
policies.GaussianHeadWithStateIndependentCovariance policies.GaussianHeadWithDiagonalCovariance
policies.GaussianHeadWithFixedCovariance policies.SoftmaxCategoricalHead
policies.DeterministicHead envs.MultiprocessVectorEnv envs.SerialVectorEnv envs.abc.ABC
wrappers.VectorFrameStack wrappers.atari_wrappers.FrameStack wrappers.atari_wrappers.LazyFrames
collections.prioritized.PrioritizedBuffer collections.random_access_queue.RandomAccessQueue
optimizers.RMSpropEpsInsideSqrt action_value.DiscreteActionValue
action_value.DistributionalDiscreteActionValue action_value.QuantileDiscreteActionValue
action_value.SingleActionValue action_value.QuadraticActionValue
q_functions.FCQuadraticStateQFunction functions.lower_triangular_matrix.lower_triangular_matrix
""".split()

METHOD_CLASSES = """
agents.DQN agents.CategoricalDoubleDQN agents.IQN agents.PPO agents.A2C agents.SoftActorCritic
agents.AL agents.PAL agents.DoublePAL agents.DPP agents.dpp.DPPL agents.dpp.DPPGreedy
agents.TD3 agents.DDPG agents.TRPO replay_buffers.ReplayBuffer replay_buffers.PrioritizedReplayBuffer
replay_buffer.ReplayUpdater replay_buffers.EpisodicReplayBuffer nn.EmpiricalNormalization nn.FactorizedNoisyLinear
envs.MultiprocessVectorEnv envs.SerialVectorEnv wrappers.VectorFrameStack
action_value.DiscreteActionValue action_value.DistributionalDiscreteActionValue
action_value.QuantileDiscreteActionValue explorers.LinearDecayEpsilonGreedy explorers.AdditiveOU
collections.random_access_queue.RandomAccessQueue experiments.evaluator.Evaluator
action_value.QuadraticActionValue q_functions.FCQuadraticStateQFunction
""".split()

# methods of the reference that belong to features outside the rebuilt path
OUT_OF_SCOPE = {"setup_actor_learner_training",
                "popleft"}  # PrioritizedBuffer.popleft: episodic buffers only
# per class: recurrent DDPG is outside the rebuilt path (only DQN / DoubleDQN are recurrent)
OUT_OF_SCOPE_FOR = {"agents.DDPG": {"update_from_episodes"}}


def resolve(root, dotted):
    import importlib

    obj = root
    for part in dotted.split("."):
        if not hasattr(obj, part):
            obj = importlib.import_module(obj.__name__ + "." + part)
        else:
            obj = getattr(obj, part)
    return obj


def params(obj):
    fn = obj.__init__ if inspect.isclass(obj) else obj
    return [p for p in inspect.signature(fn).parameters.values() if p.name != "self"]


def main():
    ref = import_reference()
    import pfrl_b200 as ours

    problems = 0
    for path in CALLABLES:
        a, b = params(resolve(ref, path)), params(resolve(ours, path))
        mine = {p.name: p for p in b}
        notes = []
        ref_pos = [p.name for p in a if p.kind == p.POSITIONAL_OR_KEYWORD]
        my_pos = [p.name for p in b if p.kind == p.POSITIONAL_OR_KEYWORD]
        if my_pos[:len(ref_pos)] != ref_pos:
            notes.append("positional order: reference %s, ours %s" % (ref_pos, my_pos))
        for p in a:
            if p.kind in (p.VAR_POSITIONAL, p.VAR_KEYWORD):
                continue
            q = mine.get(p.name)
            if q is None:
                notes.append("missing parameter %s" % p.name)
                continue
            da, db = p.default, q.default
            if callable(da) and callable(db):
                continue
            try:
                same = (da is db) or bool(da == db) or (da != da and db != db)
            except Exception:
                same = True
            if not same and not (hasattr(da, "name") and hasattr(db, "name")):  # loggers
                notes.append("default of %s: reference %r, ours %r" % (p.name, da, db))
        for n in notes:
            print("%s: %s" % (path, n))
        problems += len(notes)
    for path in METHOD_CLASSES:
        A, B = resolve(ref, path), resolve(ours, path)
        for name, member in inspect.getmembers(A):
            if (name.startswith("_") or name in OUT_OF_SCOPE
                    or name in OUT_OF_SCOPE_FOR.get(path, ())):
                continue
            if not hasattr(B, name):
                print("%s: missing attribute %s" % (path, name))
                problems += 1
                continue
            other = getattr(B, name)
            if inspect.isfunction(member) and inspect.isfunction(other):
                pa = [p.name for p in inspect.signature(member).parameters.values()]
                pb = [p.name for p in inspect.signature(other).parameters.values()]
                if pb[:len(pa)] != pa and not {"args", "kwargs"} & set(pb):
                    print("%s.%s: parameters reference %s, ours %s" % (path, name, pa, pb))
                    problems += 1
    print("%d difference(s) over %d callables and %d classes' public methods"
          % (problems, len(CALLABLES), len(METHOD_CLASSES)))
    return 1 if problems else 0


if __name__ == "__main__":
    sys.exit(main())
