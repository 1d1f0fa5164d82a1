"""bf16 model parameters with fp32 master copies, for the autocast training step.

Under ``torch.autocast`` every convolution / linear weight is cast fp32 -> bf16 at its first use of each forward and its bf16
gradient is cast back to fp32 in the backward: for the default SegMamba that is ~400 tiny cast kernels per training step
(172 + 175 + 48 launches).  ``MasterWeights`` keeps the
arithmetic and removes the launches: the matmul / convolution parameters of the model are stored in bf16 (exactly the values the
autocast cast would produce, so the forward and backward are bit-identical), the optimizer owns fp32 masters, and the two
directions of the copy are one multi-tensor op each per step:

    backward (bf16 grads on the model)  ->  grads_to_master()  ->  clip / optimizer.step() on the masters  ->  master_to_model()

Parameters the hot path reads in fp32 (LayerNorm affine, A_log, D, dt_proj bias, the depthwise conv1d taps -- the native kernels
take them as fp32, selective_scan.cpp:280-294) are left alone and are their own masters.  ``state_dict()`` returns the fp32
values under the reference's 291 keys, so checkpoints stay loadable by 4_predict.py; under DistributedDataParallel (wrap AFTER
constructing ``MasterWeights``) the gradient all-reduce moves bf16 instead of fp32.

The reference has no counterpart (its trainer relies on autocast's per-forward casts, light_training/trainer.py:450); this is
part of the training-step row of the scope table (SURVEY.md section 8 a18 / f3).  Opt-in: ``bench.py --bf16-params``,
``TrainStep(..., master_weights=MasterWeights(model))``.
"""
from __future__ import annotations

from typing import Callable, Iterable

import torch
import torch.nn as nn

_MATMUL_MODULES = (nn.Conv3d, nn.ConvTranspose3d, nn.Linear)


def default_low_precision_filter(module: nn.Module, module_name: str, param_name: str) -> bool:
    """weights and biases of dense Conv3d / ConvTranspose3d / Linear layers, except the dt_proj biases (used as fp32 delta_bias)."""
    if not isinstance(module, _MATMUL_MODULES):
        return False
    leaf = module_name.rsplit(".", 1)[-1]
    if param_name == "bias" and leaf.startswith("dt_proj"):
        return False
    return True


class MasterWeights:
    """Convert the selected parameters of ``model`` to ``dtype`` IN PLACE and keep fp32 masters for the optimizer."""

    def __init__(self, model: nn.Module, dtype: torch.dtype = torch.bfloat16,
                 low_precision: Callable[[nn.Module, str, str], bool] = default_low_precision_filter):
        self.model, self.dtype = model, dtype
        self._names: list[str] = []            # state_dict keys of the converted parameters
        self._model_params: list[nn.Parameter] = []
        self._masters: list[nn.Parameter] = []
        self._others: list[nn.Parameter] = []  # parameters that stay fp32: they are their own masters
        seen = set()
        for mname, module in model.named_modules():
            for pname, p in module.named_parameters(recurse=False):
                if id(p) in seen or not p.requires_grad:
                    continue
                seen.add(id(p))
                if p.dtype == torch.float32 and low_precision(module, mname, pname):
                    master = nn.Parameter(p.detach().clone().float(), requires_grad=True)
                    p.data = p.data.to(dtype)                    # same storage format (e.g. channels-last) as before
                    self._names.append(f"{mname}.{pname}" if mname else pname)
                    self._model_params.append(p)
                    self._masters.append(master)
                else:
                    self._others.append(p)

    # ---- what the optimizer / clipping see ------------------------------------------------------------------------
    def optimizer_parameters(self) -> list[nn.Parameter]:
        """fp32 tensors in the order of ``model.parameters()`` (masters in place of the converted parameters)."""
        by_id = {id(p): m for p, m in zip(self._model_params, self._masters)}
        return [by_id.get(id(p), p) for p in self.model.parameters() if p.requires_grad]

    # ---- the two multi-tensor copies of a step --------------------------------------------------------------------
    @torch.no_grad()
    def grads_to_master(self) -> None:
        """master.grad <- float(model_param.grad) for every converted parameter (one fused multi-tensor copy)."""
        src, dst = [], []
        for p, m in zip(self._model_params, self._masters):
            if p.grad is None:
                m.grad = None
                continue
            if m.grad is None:
                m.grad = torch.empty_like(m)
            src.append(p.grad)
            dst.append(m.grad)
        if src:
            torch._foreach_copy_(dst, src)

    @torch.no_grad()
    def master_to_model(self) -> None:
        """model_param <- dtype(master): the values the next forward's autocast cast would have produced."""
        if self._masters:
            torch._foreach_copy_([p.data for p in self._model_params], [m.data for m in self._masters])

    def zero_grad(self) -> None:
        for p in self._model_params:
            p.grad = None
        for m in self._masters:
            m.grad = None
        for p in self._others:
            p.grad = None

    # ---- checkpoints: fp32 values under the reference's keys ------------------------------------------------------
    def state_dict(self) -> dict:
        sd = self.model.state_dict()
        for name, m in zip(self._names, self._masters):
            sd[name] = m.detach().clone()
        return sd

    @torch.no_grad()
    def load_state_dict(self, state: dict, strict: bool = True) -> None:
        self.model.load_state_dict({k: (v.to(self.dtype) if k in set(self._names) else v) for k, v in state.items()}, strict=strict)
        for name, m in zip(self._names, self._masters):
            if name in state:
                m.data.copy_(state[name].to(m.device, torch.float32))
        self.master_to_model()

    def converted_names(self) -> Iterable[str]:
        return tuple(self._names)
