"""Fused LayerNorm over the channel axis of the (B, L, C) token matrix (smb_layernorm_fwd / _bwd).

Replaces ``nn.LayerNorm(dim)`` in ``MambaLayer.forward`` (model_segmamba/segmamba.py:54,70).  Same arithmetic (biased
variance, eps inside the square root, fp32 statistics, fp32 weight / bias); the output keeps the activation dtype: under
autocast the reference produces an fp32 LayerNorm result that ``in_proj`` immediately casts to the autocast dtype, so the
values that reach the GEMM are identical.  The backward recomputes the row statistics instead of saving them.
"""
from __future__ import annotations

import ctypes
import os

import torch
from torch.amp import custom_bwd, custom_fwd

from . import _lib

# Default on (hardware parity: tests/test_gpu_layernorm.py);
# SMB_FUSED_LAYERNORM=0 keeps nn.LayerNorm for A/B runs.
ENABLED = os.environ.get("SMB_FUSED_LAYERNORM", "1") != "0"


def supported(x: torch.Tensor, normalized_dim: int) -> bool:
    """shapes the kernel takes: contiguous rows of `normalized_dim` channels, a multiple of one 16-byte vector, <= 768."""
    v = 16 // x.element_size()
    return (x.dtype in (torch.float32, torch.float16, torch.bfloat16) and x.shape[-1] == normalized_dim and x.is_contiguous()
            and normalized_dim % v == 0 and normalized_dim // v <= 128 and normalized_dim <= 768 and x.data_ptr() % 16 == 0)


class _FusedLayerNorm(torch.autograd.Function):
    @staticmethod
    @custom_fwd(device_type="cuda")
    def forward(ctx, x, weight, bias, eps):
        _lib.require_cuda(x, weight, bias)
        C = x.shape[-1]
        rows = x.numel() // C
        w32 = weight.float().contiguous()
        b32 = bias.float().contiguous() if bias is not None else None
        dev = x.device
        with torch.cuda.device(dev):
            y = torch.empty_like(x)
            a = _lib.LayerNormArgs()
            a.rows, a.channels, a.dtype, a.eps = rows, C, _lib.dtype_code(x.dtype), float(eps)
            a.x, a.gamma, a.beta, a.y = _lib.ptr(x), _lib.ptr(w32), _lib.ptr(b32), _lib.ptr(y)
            sp = _lib.stream_ptr(dev)
            _lib.call("layernorm_fwd", (rows, C, x.element_size()), lambda: _lib.lib().smb_layernorm_fwd(ctypes.byref(a), sp), dev)
        ctx.save_for_backward(x, w32)
        ctx.eps, ctx.has_bias = eps, bias is not None
        ctx.wdtype = weight.dtype
        return y

    @staticmethod
    @custom_bwd(device_type="cuda")
    def backward(ctx, dy):
        x, w32 = ctx.saved_tensors
        C = x.shape[-1]
        rows = x.numel() // C
        dy = dy.to(x.dtype).contiguous()
        dev = x.device
        with torch.cuda.device(dev):
            dx = torch.empty_like(x)
            dgb = torch.zeros(2, C, dtype=torch.float32, device=dev)       # one zero-fill for both accumulators
            a = _lib.LayerNormBwdArgs()
            a.rows, a.channels, a.dtype, a.eps = rows, C, _lib.dtype_code(x.dtype), float(ctx.eps)
            a.x, a.dy, a.gamma, a.dx = _lib.ptr(x), _lib.ptr(dy), _lib.ptr(w32), _lib.ptr(dx)
            a.dgamma, a.dbeta = dgb[0].data_ptr(), dgb[1].data_ptr()
            sp = _lib.stream_ptr(dev)
            _lib.call("layernorm_bwd", (rows, C, x.element_size()), lambda: _lib.lib().smb_layernorm_bwd(ctypes.byref(a), sp), dev)
        return dx, dgb[0].to(ctx.wdtype), (dgb[1].to(ctx.wdtype) if ctx.has_bias else None), None


def fused_layer_norm(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor | None, eps: float = 1e-5) -> torch.Tensor:
    """LayerNorm over the last axis of a contiguous tensor; raises for shapes `supported()` rejects."""
    if not supported(x, weight.shape[0]):
        raise RuntimeError(f"fused_layer_norm: unsupported input (shape {tuple(x.shape)}, dtype {x.dtype}, contiguous={x.is_contiguous()})")
    return _FusedLayerNorm.apply(x, weight, bias, eps)
