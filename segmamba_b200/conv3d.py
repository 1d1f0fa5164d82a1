"""Dense 3x3x3 convolutions (stride 1, padding 1, no bias) on the native implicit-GEMM kernel of libsegmamba_b200
(smb_conv3d / smb_conv3d_wgrad: TMA -> wgmma, no im2col), with a native backward.

``conv3d(conv, x)`` is the one place that decides between the native kernel and the library convolution (cuDNN), pass by
pass: see ``native_ok`` and ``NATIVE_PASSES``.  The weight is used in the channels-last storage the model keeps it in, (C_out, 3, 3, 3, C_in), so neither the
state_dict nor the parameter layout changes.

Backward: the data gradient is the same kernel on dY with the weight flipped in its three spatial axes and C_in / C_out
swapped (a 27 C_in C_out copy per call); it is skipped when the input needs no gradient.  The weight gradient contracts over
all voxels on the native kernel in fp32 (split over the SMs, fp32 atomics) and is cast to the weight's dtype.
"""
from __future__ import annotations

import ctypes

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.amp import custom_bwd, custom_fwd

from . import _lib

_CL = torch.channels_last_3d

# The passes ("f" forward, "d" data gradient, "w" weight gradient) that run natively, per (C_in, C_out, voxels per sample):
# those that tools/conv3d_bench.py measured to be at least 10 % faster than cuDNN's heuristic plan at batch 2 in bf16 on an
# H100 80GB HBM3 (700 W).  Every other pass of a routed convolution, and every other convolution, runs on cuDNN.
NATIVE_PASSES = {
    (48, 48, 128 ** 3): "fdw",
    (96, 48, 128 ** 3): "fw",
    (48, 48, 64 ** 3): "fdw",
    (48, 96, 64 ** 3): "fw",
    (96, 96, 64 ** 3): "fw",
    (192, 96, 64 ** 3): "w",
    (96, 96, 32 ** 3): "fw",
    (96, 192, 32 ** 3): "dw",
    (192, 192, 32 ** 3): "d",
    (192, 384, 16 ** 3): "f",
    (384, 384, 16 ** 3): "f",
    (768, 384, 16 ** 3): "f",
}


def _compute_dtype(x: torch.Tensor) -> torch.dtype:
    return torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled("cuda") else x.dtype


def native_ok(conv: nn.Conv3d, x: torch.Tensor) -> bool:
    """True when ``conv`` applied to ``x`` (bias aside) runs on the native kernel: a CUDA input and ``shape_ok``."""
    return x.is_cuda and shape_ok(conv, x, _compute_dtype(x))


def shape_ok(conv: nn.Module, x: torch.Tensor, compute_dtype: torch.dtype) -> bool:
    """16-bit compute, kernel 3 / stride 1 / padding 1 / dilation 1 / groups 1 (no transposed convolution), a shape with at
    least one native pass in NATIVE_PASSES and a channels-last contiguous input."""
    return (type(conv) is nn.Conv3d and x.dim() == 5 and compute_dtype in (torch.float16, torch.bfloat16)
            and conv.kernel_size == (3, 3, 3) and conv.stride == (1, 1, 1) and conv.padding == (1, 1, 1)
            and conv.dilation == (1, 1, 1) and conv.groups == 1 and conv.padding_mode == "zeros"
            and bool(_passes(conv.in_channels, conv.out_channels, x))
            and x.is_contiguous(memory_format=_CL))


def _passes(c_in: int, c_out: int, x: torch.Tensor) -> str:
    return NATIVE_PASSES.get((c_in, c_out, x.shape[2] * x.shape[3] * x.shape[4]), "")


def conv3d(conv: nn.Conv3d, x: torch.Tensor, bias: bool = True) -> torch.Tensor:
    """``conv(x)``, or ``conv(x)`` without its bias when ``bias`` is False; native where ``native_ok`` says so."""
    if native_ok(conv, x) and (conv.bias is None or not bias):
        return _Conv3d3.apply(x, conv.weight, _compute_dtype(x), _passes(conv.in_channels, conv.out_channels, x))
    if bias:
        return conv(x)
    return F.conv3d(x, conv.weight, None, conv.stride, conv.padding, conv.dilation, conv.groups)


def _args(x5: torch.Tensor, c_in: int, c_out: int) -> _lib.Conv3dArgs:
    a = _lib.Conv3dArgs()
    a.batch, a.d, a.h, a.w = x5.shape[0], x5.shape[1], x5.shape[2], x5.shape[3]
    a.c_in, a.c_out, a.dtype = c_in, c_out, _lib.dtype_code(x5.dtype)
    return a


def conv3d_fwd(x5: torch.Tensor, w5: torch.Tensor) -> torch.Tensor:
    """x5 (N, D, H, W, C_in), w5 (C_out, 3, 3, 3, C_in), both contiguous 16-bit -> y (N, D, H, W, C_out)."""
    c_out, c_in = w5.shape[0], w5.shape[4]
    y = torch.empty(*x5.shape[:4], c_out, dtype=x5.dtype, device=x5.device)
    a = _args(x5, c_in, c_out)
    a.x, a.weight, a.y = x5.data_ptr(), w5.data_ptr(), y.data_ptr()
    sp = _lib.stream_ptr(x5.device)
    _lib.call("conv3d_fwd", (*x5.shape[:4], c_in, c_out, x5.element_size()), lambda: _lib.lib().smb_conv3d(ctypes.byref(a), sp), x5.device)
    return y


def dgrad_weight(w5: torch.Tensor) -> torch.Tensor:
    """(C_out, 3, 3, 3, C_in) -> (C_in, 3, 3, 3, C_out) flipped in kd, kh, kw: the weight of the data gradient as a forward."""
    return w5.flip(1, 2, 3).permute(4, 1, 2, 3, 0).contiguous()


def conv3d_dgrad(dy5: torch.Tensor, w5: torch.Tensor) -> torch.Tensor:
    """dX (N, D, H, W, C_in) of y = conv3d_fwd(x, w5) from dy5 (N, D, H, W, C_out)."""
    wd = dgrad_weight(w5)
    c_in, c_out = wd.shape[4], wd.shape[0]
    dx = torch.empty(*dy5.shape[:4], c_out, dtype=dy5.dtype, device=dy5.device)
    a = _args(dy5, c_in, c_out)
    a.x, a.weight, a.y = dy5.data_ptr(), wd.data_ptr(), dx.data_ptr()
    sp = _lib.stream_ptr(dy5.device)
    _lib.call("conv3d_dgrad", (*dy5.shape[:4], c_in, c_out, dy5.element_size()), lambda: _lib.lib().smb_conv3d(ctypes.byref(a), sp), dy5.device)
    return dx


def conv3d_wgrad(x5: torch.Tensor, dy5: torch.Tensor) -> torch.Tensor:
    """dW (C_out, 3, 3, 3, C_in) in fp32 of y = conv3d_fwd(x5, w)."""
    c_in, c_out = x5.shape[4], dy5.shape[4]
    dw = torch.zeros(c_out, 3, 3, 3, c_in, dtype=torch.float32, device=x5.device)
    a = _args(x5, c_in, c_out)
    a.x, a.dy, a.dweight = x5.data_ptr(), dy5.data_ptr(), dw.data_ptr()
    sp = _lib.stream_ptr(x5.device)
    _lib.call("conv3d_wgrad", (*x5.shape[:4], c_in, c_out, x5.element_size()), lambda: _lib.lib().smb_conv3d_wgrad(ctypes.byref(a), sp), x5.device)
    return dw


def _cl5(t: torch.Tensor) -> torch.Tensor:
    """(N, C, D, H, W) channels-last -> its (N, D, H, W, C) storage view, contiguous"""
    v = t.permute(0, 2, 3, 4, 1)
    return v if v.is_contiguous() else v.contiguous()


def _library_grads(dy5, x5, w5, mask):
    """the passes of ``mask`` (dX, dW) from cuDNN, on the same channels-last 16-bit operands"""
    cl = lambda t: t.permute(0, 4, 1, 2, 3)
    dx, dw, _ = torch.ops.aten.convolution_backward(cl(dy5), cl(x5), cl(w5), None, [1, 1, 1], [1, 1, 1], [1, 1, 1], False,
                                                   [0, 0, 0], 1, [mask[0], mask[1], False])
    return dx, dw


class _Conv3d3(torch.autograd.Function):
    """3x3x3 convolution whose passes named in ``passes`` ("f", "d", "w") run natively and the others on cuDNN"""

    @staticmethod
    @custom_fwd(device_type="cuda", cast_inputs=None)
    def forward(ctx, x, weight, cd, passes):
        _lib.require_cuda(x, weight)
        xq = x if x.dtype == cd else x.to(cd)
        wq = weight if weight.dtype == cd else weight.to(cd)
        x5, w5 = _cl5(xq), _cl5(wq)
        ctx.save_for_backward(x5, w5)
        ctx.w_dtype, ctx.x_dtype, ctx.passes = weight.dtype, x.dtype, passes
        if "f" in passes:
            return conv3d_fwd(x5, w5).permute(0, 4, 1, 2, 3)
        return F.conv3d(xq, wq, None, 1, 1)

    @staticmethod
    @custom_bwd(device_type="cuda")
    def backward(ctx, dy):
        x5, w5 = ctx.saved_tensors
        dy5 = _cl5(dy if dy.dtype == x5.dtype else dy.to(x5.dtype))
        want_dx, want_dw = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        lib_dx = want_dx and "d" not in ctx.passes
        lib_dw = want_dw and "w" not in ctx.passes
        dx = dw = None
        if lib_dx or lib_dw:
            dx, dw = _library_grads(dy5, x5, w5, (lib_dx, lib_dw))
        if want_dx and not lib_dx:
            dx = conv3d_dgrad(dy5, w5).permute(0, 4, 1, 2, 3)
        if want_dw and not lib_dw:
            dw = conv3d_wgrad(x5, dy5).permute(0, 4, 1, 2, 3)
        return (dx.to(ctx.x_dtype) if dx is not None else None), (dw.to(ctx.w_dtype) if dw is not None else None), None, None
