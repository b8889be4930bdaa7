"""The reference's module path (pfrl/experiments/train_agent_async.py).  Asynchronous
(A3C-style, multi-process) training is outside the rebuilt path: agents such as ACER
train single-process through ``train_agent`` / ``train_agent_with_evaluation``."""


def train_agent_async(*args, **kwargs):
    """Asynchronous (A3C-style, multi-process) training is outside the rebuilt path."""
    raise NotImplementedError("train_agent_async is out of scope of pfrl_b200")
