"""Whole-step CUDA-graph capture for the SegMamba training step.

One training step of the default model enqueues several thousand kernels (cuDNN / cuBLAS / ATen / native), and the host's time
to launch them (bench.py: host_enqueue_ms_per_step) is a large fraction of the step's GPU time, so kernel speed-ups push the
step towards being launch-bound.  ``GraphedTrainStep`` captures forward + loss + backward + gradient clipping + optimizer step once and
replays it with a single ``cudaGraphLaunch`` per step (static input / label buffers, private memory pool).  All native
kernels are capture-safe by construction: they only enqueue work on the current stream and allocate through the PyTorch
caching allocator.

This replaces nothing in the reference (its trainer launches eagerly, light_training/trainer.py:422-483); it is the
"CUDA graphs instead of a tracing compiler" part of the design.
"""
from __future__ import annotations

from typing import Callable

import torch


class GraphedTrainStep:
    """step = GraphedTrainStep(model, optimizer, loss_fn, x_example, y_example); loss = step(x, y)

    ``model`` may be a DistributedDataParallel wrapper (construct it, run the warm-up and capture on the same side stream,
    as PyTorch's CUDA-graph notes require).  ``loss_fn(logits, y) -> scalar``.  The returned loss is a static device tensor
    that is overwritten by the next replay.

    ``scheduler``: anything with ``step()`` that rewrites ``optimizer.param_groups[i]["lr"]`` (the reference steps its poly
    schedule after every iteration, light_training/trainer.py:476-477).  A captured ``optimizer.step()`` bakes the Python-float
    learning rate of capture time into the graph, so with a scheduler the graph ends after gradient clipping and the optimizer
    step runs eagerly after each replay (a handful of multi-tensor kernels), followed by ``scheduler.step()``.
    ``restore_after_warmup`` (default True): the warm-up iterations and the capture pass are real optimizer steps on the example
    batch; afterwards the parameters are copied back to their values from before the warm-up and every optimizer state tensor
    (momentum buffers) is zeroed in place -- for SGD with dampening 0 a zero buffer reproduces the first-step rule
    ``buf = grad`` exactly -- so training starts from the state the caller handed in.
    """

    def __init__(self, model: torch.nn.Module, optimizer: torch.optim.Optimizer, loss_fn: Callable, x_example: torch.Tensor,
                 y_example: torch.Tensor, autocast_dtype: torch.dtype | None = torch.bfloat16, clip_grad_norm: float | None = 12.0,
                 warmup_iters: int = 3, master_weights=None, scheduler=None, restore_after_warmup: bool = True):
        self.model, self.optimizer, self.loss_fn = model, optimizer, loss_fn
        self.scheduler = scheduler
        self._opt_in_graph = scheduler is None
        self.autocast_dtype, self.clip = autocast_dtype, clip_grad_norm
        self.static_x = x_example.clone()
        self.static_y = y_example.clone()
        self.master_weights = master_weights                  # optional MasterWeights (bf16 parameters, fp32 masters)
        self.params = (master_weights.optimizer_parameters() if master_weights is not None
                       else [p for p in model.parameters() if p.requires_grad])
        saved = [p.detach().clone() for p in self.params] if restore_after_warmup else None
        saved_model = ([p.detach().clone() for p in model.parameters()] if (restore_after_warmup and master_weights is not None) else None)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(warmup_iters):                # warm-up on the capture stream (cuDNN autotune, lazy inits, allocator)
                self._eager_step()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        self._zero()
        with torch.cuda.graph(self.graph):
            self.static_loss = self._eager_step(zero=False, optimizer_step=self._opt_in_graph)
        if not self._opt_in_graph:
            self._optimizer_step()                          # the capture pass's own update, eagerly (state stays consistent)
        if restore_after_warmup:
            with torch.no_grad():
                for p, v in zip(self.params, saved):
                    p.copy_(v)
                if saved_model is not None:
                    for p, v in zip(model.parameters(), saved_model):
                        p.copy_(v)
                for st in optimizer.state.values():
                    for k, t in st.items():
                        if torch.is_tensor(t) and t.is_floating_point() and t.dim() > 0:
                            t.zero_()

    def _zero(self):
        self.optimizer.zero_grad(set_to_none=True)
        if self.master_weights is not None:
            self.master_weights.zero_grad()

    def _optimizer_step(self):
        self.optimizer.step()
        if self.master_weights is not None:
            self.master_weights.master_to_model()

    def _eager_step(self, zero: bool = True, optimizer_step: bool = True):
        if zero:
            self._zero()
        with torch.autocast("cuda", dtype=self.autocast_dtype, enabled=self.autocast_dtype is not None):
            logits = self.model(self.static_x)
            loss = self.loss_fn(logits.float(), self.static_y)
        loss.backward()
        if self.master_weights is not None:
            self.master_weights.grads_to_master()
        if self.clip is not None:
            torch.nn.utils.clip_grad_norm_(self.params, self.clip, foreach=True)
        if optimizer_step:
            self._optimizer_step()
        return loss.detach()

    def __call__(self, x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        self.static_x.copy_(x, non_blocking=True)
        self.static_y.copy_(y, non_blocking=True)
        self.graph.replay()
        if not self._opt_in_graph:
            self._optimizer_step()
            self.scheduler.step()
        return self.static_loss
