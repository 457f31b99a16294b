"""CUDA-graph capture of launch-bound calls: inference forwards (GraphedForward) and whole training steps on one GPU
(GraphedTrainStep).

Small-batch (decoder) MoE inference is a dozen kernels of a few microseconds each: issued one by one from Python the
GPU idles between them and the layer costs whatever the CPU needs to launch it.  With a positive capacity factor, or
with the bound-based dropless mode (``capacity_factor <= 0`` + ``megablocks_size > 0`` on one GPU, see
models/moe_layer.py), a forward pass never touches the host, so the whole call can be recorded once and replayed as
ONE graph launch:

    fast = GraphedForward(lambda x: layer(x, megablocks_size=1), example_x)
    y = fast(x)                      # copies x into the static input, replays, returns the static output

The reference cannot do this: its dropless path reads the capacity and the per-expert counts back to the host
(tutel/impls/fast_dispatch.py:192-193, tutel/custom/custom_kernel.cpp:875).
"""
from __future__ import annotations

from typing import Callable, Sequence

import torch


class GraphedForward:
    """Record ``fn(*inputs)`` (no autograd) into a CUDA graph; calls replay it on fresh input values of the same shapes."""

    def __init__(self, fn: Callable, *example_inputs: torch.Tensor, warmup: int = 3):
        assert all(t.is_cuda for t in example_inputs), 'GraphedForward needs CUDA tensors'
        self._inputs = [t.detach().clone() for t in example_inputs]
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side), torch.no_grad():
            for _ in range(max(warmup, 1)):       # lazy initialisation (kernel attributes, workspaces, caches) happens here
                fn(*self._inputs)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self._graph = torch.cuda.CUDAGraph()
        with torch.no_grad(), torch.cuda.graph(self._graph):
            self._outputs = fn(*self._inputs)

    def __call__(self, *inputs: torch.Tensor):
        for dst, src in zip(self._inputs, inputs):
            if dst.data_ptr() != src.data_ptr():
                dst.copy_(src, non_blocking=True)
        self._graph.replay()
        return self._outputs

    @property
    def static_inputs(self) -> Sequence[torch.Tensor]:
        return self._inputs


class GraphedTrainStep:
    """Record a whole training step - ``zero_grad``, forward, loss, backward, ``optimizer.step()`` - into ONE CUDA graph.

    A training step of one MoE layer is ~40 launches; when the host has to wait for a result of every step (the loss
    that is logged, an LR schedule that looks at it) it cannot run ahead, and the GPU idles at the start of each step
    until the launches catch up (0.3 ms of a 9.4 ms step on the flagship layer).  Nothing in a step of this framework
    touches the host on ONE GPU (routing, capacity and dispatch tables stay on the device), so the step can be replayed
    as a single graph launch:

        fast = GraphedTrainStep(step_fn, x_example, y_example)     # step_fn(x, y) -> loss; runs warm-up steps, captures
        loss = fast(x, y)                                          # copies the values in, replays, returns the loss

    ``step_fn`` must do its own ``optimizer.zero_grad(set_to_none=True)`` (gradients then live in the graph's memory
    pool) and must not synchronise.  If the model already ran eagerly, drop every tensor of those steps that still has a
    ``grad_fn`` (losses, auxiliary losses) before constructing this object: a live autograd graph keeps the parameters'
    gradient accumulators bound to the eager stream, and the capture fails with ``cudaErrorStreamCaptureInvalidated``
    (``MOELayer`` releases its own ``l_aux`` at the start of every forward).  Multi-GPU steps are not capturable this way: the peer-to-peer protocol numbers its
    transactions with host-side epochs that would be frozen into the graph.
    Dropless training steps (a gate with ``capacity_factor=0``) are capturable too: on one GPU they run on the
    expert-packed layout (ops/packed.py), whose buffer shapes are static bounds and whose offsets stay on the device.
    The reference's step cannot be captured at all: its dispatch reads the capacity back to the host every forward
    (tutel/impls/fast_dispatch.py:192-193).
    """

    def __init__(self, step_fn: Callable, *example_inputs: torch.Tensor, warmup: int = 3):
        assert all(t.is_cuda for t in example_inputs), 'GraphedTrainStep needs CUDA tensors'
        from ..ops import backend
        self._inputs = [t.detach().clone().requires_grad_(t.requires_grad) for t in example_inputs]
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(max(warmup, 1)):       # lazy initialisation and allocator warm-up happen outside the capture
                step_fn(*self._inputs)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self._graph = torch.cuda.CUDAGraph()
        before = backend.launch_count()
        with torch.cuda.graph(self._graph):
            self._loss = step_fn(*self._inputs)
        self.launches_per_replay = backend.launch_count() - before     # native kernels recorded in the graph
        self._count = backend.count_launch
        # optimizer-step hooks do not run during a replay: tell the fp8 / MX weight caches (ops/gemm.py, ops/mx.py) that the
        # weights moved, so that an eager forward after replays re-quantises them (the replays themselves re-quantise
        # inside the graph and never consult the cache)
        from ..ops import gemm as _gemm
        self._weights_moved = _gemm.invalidate_fp8_cache

    def __call__(self, *inputs: torch.Tensor):
        with torch.no_grad():
            for dst, src in zip(self._inputs, inputs):
                if dst.data_ptr() != src.data_ptr():
                    dst.copy_(src, non_blocking=True)
        self._graph.replay()
        self._count(self.launches_per_replay)
        self._weights_moved()
        return self._loss

    @property
    def static_inputs(self) -> Sequence[torch.Tensor]:
        return self._inputs
