"""Channel concatenation of channels-last activations on the native strided-copy kernel (smb_copy2d).

``cat_channels(a, b)`` == ``torch.cat((a, b), dim=1)`` for 5-D tensors stored channels-last (NDHWC): the (tokens, C) matrices of the two
operands are copied into the left / right column block of the (tokens, Ca + Cb) result with full 16-byte vectors; the backward copies the
two column blocks of the incoming gradient back out.  Replaces ``torch.cat((out, skip), dim=1)`` of UnetrUpBlock
(monai/networks/blocks/unetr_block.py:81-86), which ATen runs as generic strided elementwise copies (two forward and two
backward per up block and step).  Operands that do not meet the layout / alignment rules raise; the caller decides (segmamba.py
uses torch.cat for them).
"""
from __future__ import annotations

import torch

from . import _lib

_CL = torch.channels_last_3d


def supported(a: torch.Tensor, b: torch.Tensor) -> bool:
    es = a.element_size()
    return (a.is_cuda and b.is_cuda and a.dim() == 5 and b.dim() == 5 and a.dtype == b.dtype and a.shape[0] == b.shape[0]
            and a.shape[2:] == b.shape[2:] and a.is_contiguous(memory_format=_CL) and b.is_contiguous(memory_format=_CL)
            and (a.shape[1] * es) % 16 == 0 and (b.shape[1] * es) % 16 == 0 and a.data_ptr() % 16 == 0 and b.data_ptr() % 16 == 0)


def _copy2d(src_ptr, src_pitch, dst_ptr, dst_pitch, rows, row_bytes, dev):
    sp = _lib.stream_ptr(dev)
    _lib.call("copy2d", (rows, row_bytes), lambda: _lib.lib().smb_copy2d(src_ptr, src_pitch, dst_ptr, dst_pitch, rows, row_bytes, sp), dev)


class _CatChannels(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, b):
        Bz, Ca = a.shape[:2]
        Cb = b.shape[1]
        sp = a.shape[2:]
        es = a.element_size()
        rows = a.numel() // Ca
        dev = a.device
        with torch.cuda.device(dev):
            out = torch.empty((Bz, Ca + Cb) + tuple(sp), dtype=a.dtype, device=dev, memory_format=_CL)
            pitch = (Ca + Cb) * es
            _copy2d(a.data_ptr(), Ca * es, out.data_ptr(), pitch, rows, Ca * es, dev)
            _copy2d(b.data_ptr(), Cb * es, out.data_ptr() + Ca * es, pitch, rows, Cb * es, dev)
        ctx.ca, ctx.cb = Ca, Cb
        return out

    @staticmethod
    def backward(ctx, g):
        Ca, Cb = ctx.ca, ctx.cb
        if not g.is_contiguous(memory_format=_CL):
            g = g.contiguous(memory_format=_CL)
        Bz = g.shape[0]
        sp = g.shape[2:]
        es = g.element_size()
        rows = g.numel() // (Ca + Cb)
        dev = g.device
        ga = gb = None
        with torch.cuda.device(dev):
            pitch = (Ca + Cb) * es
            if ctx.needs_input_grad[0]:
                ga = torch.empty((Bz, Ca) + tuple(sp), dtype=g.dtype, device=dev, memory_format=_CL)
                _copy2d(g.data_ptr(), pitch, ga.data_ptr(), Ca * es, rows, Ca * es, dev)
            if ctx.needs_input_grad[1]:
                gb = torch.empty((Bz, Cb) + tuple(sp), dtype=g.dtype, device=dev, memory_format=_CL)
                _copy2d(g.data_ptr() + Ca * es, pitch, gb.data_ptr(), Cb * es, rows, Cb * es, dev)
        return ga, gb


def cat_channels(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    if not supported(a, b):
        raise RuntimeError(f"cat_channels: channels-last 5-D operands with 16-byte channel rows expected (got {tuple(a.shape)} {a.dtype}, "
                           f"{tuple(b.shape)} {b.dtype})")
    return _CatChannels.apply(a, b)
