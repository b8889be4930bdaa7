"""The agents' CUDA-graph capture (``cuda_graph=True``): persistent input buffers, eager
warm-up, one capture, then replays."""
import torch

from pfrl_b200.utils.modes import no_distribution_validation


def make_capturable(*optimizers):
    """``capturable=True`` on every param group that has the option (torch's Adam and
    relatives): the step then keeps its state and bias corrections on the device."""
    for opt in optimizers:
        for group in opt.param_groups:
            if "capturable" in group:
                group["capturable"] = True


class CapturedStep:
    """One graphed call.  ``load(key, inputs)`` copies ``inputs`` (a dict of tensors) into
    persistent buffers and returns them; ``run(fn)`` calls ``fn(buffers)`` eagerly ``warmup``
    times, then captures one call and from then on replays it and returns the captured
    outputs.  With ``share_pool_with``, the graph is captured into that step's memory pool;
    the two must then replay in the order they were captured.  With ``pool`` (a
    ``torch.cuda.graph_pool_handle()``), it is captured into that pool, which several steps
    can share whichever of them captures first; such steps must replay one after another on
    one stream, each one's outputs consumed before another replays.

    A capture bakes in the addresses of the tensors the call reads and every Python number
    it reads: an optimizer's scalar ``lr``, a loss coefficient handed to a kernel.  So the
    graph is replayed only while its key is unchanged.  The key is the input layout (names,
    shapes, dtypes), every hyperparameter of ``optimizers`` (the optimizers the call steps,
    None entries skipped, made capturable here) and the caller's ``key``: the agent
    attributes the call reads as Python numbers.  Attributes that are set in the constructor
    and that no hook changes (C51's atoms, IQN's quantile counts, the α and η of AL and DPP)
    are left out.  A changed key drops the graph: the call warms up and is captured again."""

    def __init__(self, warmup, optimizers=(), share_pool_with=None, pool=None):
        self.warmup = warmup
        self.optimizers = [opt for opt in optimizers if opt is not None]
        make_capturable(*self.optimizers)
        self.share_pool_with = share_pool_with
        self.pool = pool
        self.key = self.graph = None

    def load(self, key, inputs):
        # a tensor hyperparameter (a tensor lr) is read from memory by the graph: it is
        # keyed by identity and never read on the host
        key = (key, tuple((k, v.shape, v.dtype) for k, v in inputs.items()),
               tuple((k, id(v) if isinstance(v, torch.Tensor) else v)
                     for opt in self.optimizers for group in opt.param_groups
                     for k, v in group.items() if k != "params"))
        if key != self.key:
            self.key, self.graph, self.warm = key, None, 0
            self.buffers = {k: torch.empty_like(v) for k, v in inputs.items()}
        for k, v in inputs.items():
            self.buffers[k].copy_(v)
        return self.buffers

    def run(self, fn):
        if self.graph is None:
            if self.warm < self.warmup:  # optimizer state, cuBLAS / cuDNN plans
                self.warm += 1
                return fn(self.buffers)
            pool = self.share_pool_with.graph.pool() if self.share_pool_with else self.pool
            self.graph = torch.cuda.CUDAGraph()
            # torch.cuda.graph synchronises the device before it captures
            with no_distribution_validation(), torch.cuda.graph(self.graph, pool=pool):
                self.out = fn(self.buffers)
        self.graph.replay()  # capture only records: the captured call is replayed too
        return self.out
