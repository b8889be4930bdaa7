from pfrl_b200.experiments.evaluator import Evaluator, eval_performance, save_agent  # NOQA
from pfrl_b200.experiments.train_agent import train_agent  # NOQA
from pfrl_b200.experiments.train_agent_batch import train_agent_batch  # NOQA
from pfrl_b200.experiments.train_agent_batch import train_agent_batch_with_evaluation  # NOQA
from pfrl_b200.experiments.hooks import LinearInterpolationHook, StepHook  # NOQA
from pfrl_b200.experiments.train_agent import train_agent_with_evaluation  # NOQA
from pfrl_b200.experiments.evaluator import batch_run_evaluation_episodes  # NOQA
from pfrl_b200.experiments.evaluator import run_evaluation_episodes  # NOQA
from pfrl_b200.experiments import evaluation_hooks  # NOQA
from pfrl_b200.experiments.evaluation_hooks import EvaluationHook  # NOQA
from pfrl_b200.experiments.train_agent_async import train_agent_async  # NOQA
