"""Autograd ops of the SegMamba hot path on top of the native library.

Mirrors the reference's operator interface (same names, argument meaning and return conventions):

* ``selective_scan_fn``            <- mamba/mamba_ssm/ops/selective_scan_interface.py:14-83  (SelectiveScanFn)
* ``causal_conv1d_fn``             <- causal-conv1d/causal_conv1d/causal_conv1d_interface.py:10-46 (CausalConv1dFn)
* ``mamba_inner_fn_no_out_proj``   <- selective_scan_interface.py:155-289,627-633 (MambaInnerFnNoOutProj)

Differences that stay behind the interface: the native scan/conv kernels take a walk ``direction`` so the
reversed pass of the tri-directional block needs no ``flip`` copies, the forward saves 256-position states
instead of the pre-gate output so the backward neither re-reads ``out`` nor needs the 2048-chunk ``x``, and
dB/dC come back already reduced over channels.  There is no CPU path: non-CUDA tensors raise RuntimeError.
"""
from __future__ import annotations

import os

import torch
from torch.amp import custom_bwd, custom_fwd

from . import causal_conv1d_cuda, selective_scan_cuda
from . import gemm as _gemm

# keep conv1d_out and delta for the backward instead of recomputing them (SMB_RECOMPUTE=1 restores the reference's
# checkpoint_lvl=1 behaviour, ssi.py:216-219)
KEEP_CONV_DELTA = os.environ.get("SMB_RECOMPUTE", "0") != "1"
# zero-pad the dt block of x_proj / dt_proj to a multiple of 8 rows so that no GEMM of the mixer has a 3- or 6-element
# leading dimension (SMB_ALIGN_GEMMS=0 restores the reference's shapes)
ALIGN_GEMMS = os.environ.get("SMB_ALIGN_GEMMS", "1") != "0"


class SelectiveScanFn(torch.autograd.Function):
    """ssi.py:14-74."""

    @staticmethod
    def forward(ctx, u, delta, A, B, C, D=None, z=None, delta_bias=None, delta_softplus=False, return_last_state=False):
        if u.stride(-1) != 1:
            u = u.contiguous()
        if delta.stride(-1) != 1:
            delta = delta.contiguous()
        if D is not None:
            D = D.contiguous()
        if B.stride(-1) != 1:
            B = B.contiguous()
        if C.stride(-1) != 1:
            C = C.contiguous()
        if z is not None and z.stride(-1) != 1:
            z = z.contiguous()
        ctx.squeeze_B = B.dim() == 3
        ctx.squeeze_C = C.dim() == 3
        if ctx.squeeze_B:
            B = B.unsqueeze(1)
        if ctx.squeeze_C:
            C = C.unsqueeze(1)
        out, x, out_z, hst, hd = selective_scan_cuda.fwd_ex(u, delta, A, B, C, D, z, delta_bias, delta_softplus, want_out=z is None,
                                                            want_x=return_last_state, want_hstates=True, want_hdense=True)
        ctx.delta_softplus = delta_softplus
        ctx.has_z = z is not None
        ctx.save_for_backward(u, delta, A, B, C, D, z, delta_bias, hst, hd)
        res = out_z if ctx.has_z else out
        if not return_last_state:
            return res
        last_state = x[:, :, -1, 1::2]          # (batch, dim, dstate)  ssi.py:40
        return res, last_state

    @staticmethod
    def backward(ctx, dout, *args):
        u, delta, A, B, C, D, z, delta_bias, hst, hd = ctx.saved_tensors
        if dout.stride(-1) != 1:
            dout = dout.contiguous()
        du, ddelta, dA, dB, dC, dD, ddelta_bias, dz, _ = selective_scan_cuda.bwd_ex(
            u, delta, A, B, C, D, z, delta_bias, dout, None, ctx.delta_softplus, False, hstates=hst, hdense=hd)
        dB = dB.to(B.dtype)
        dC = dC.to(C.dtype)
        dB = dB.squeeze(1) if ctx.squeeze_B else dB
        dC = dC.squeeze(1) if ctx.squeeze_C else dC
        return (du, ddelta, dA, dB, dC, dD if D is not None else None, dz,
                ddelta_bias if delta_bias is not None else None, None, None)


def selective_scan_fn(u, delta, A, B, C, D=None, z=None, delta_bias=None, delta_softplus=False, return_last_state=False):
    """if return_last_state is True, returns (out, last_state); last_state has shape (batch, dim, dstate)
    and carries no gradient (ssi.py:77-83)."""
    return SelectiveScanFn.apply(u, delta, A, B, C, D, z, delta_bias, delta_softplus, return_last_state)


class CausalConv1dFn(torch.autograd.Function):
    """causal_conv1d_interface.py:10-34."""

    @staticmethod
    def forward(ctx, x, weight, bias=None, activation=None):
        if activation not in [None, "silu", "swish"]:
            raise NotImplementedError("activation must be None, silu, or swish")
        if x.stride(2) != 1:
            x = x.contiguous()
        bias = bias.contiguous() if bias is not None else None
        ctx.save_for_backward(x, weight, bias)
        ctx.activation = activation in ["silu", "swish"]
        return causal_conv1d_cuda.causal_conv1d_fwd(x, weight, bias, ctx.activation)

    @staticmethod
    def backward(ctx, dout):
        x, weight, bias = ctx.saved_tensors
        if dout.stride(2) != 1:
            dout = dout.contiguous()
        dx, dweight, dbias = causal_conv1d_cuda.causal_conv1d_bwd(x, weight, bias, dout, None, ctx.activation)
        return dx, dweight, dbias if bias is not None else None, None


def causal_conv1d_fn(x, weight, bias=None, activation=None):
    """x: (batch, dim, seqlen); weight: (dim, width); bias: (dim,); activation: None | "silu" | "swish"."""
    return CausalConv1dFn.apply(x, weight, bias, activation)


def _as_dbl(t):
    """(b, d, l) -> (d, b*l) matrix; a view for the channel-major ("HBL") layout the mixer produces, else one copy."""
    return t.permute(1, 0, 2).reshape(t.shape[1], t.shape[0] * t.shape[2])


class MambaInnerFnNoOutProj(torch.autograd.Function):
    """conv1d+SiLU -> x_proj -> dt_proj -> selective scan -> SiLU(z) gate, with recompute in backward
    (ssi.py:155-289, checkpoint_lvl=1).  ``direction`` = 1 walks L in descending order, which equals calling the
    reference op on ``xz.flip(-1)`` and flipping its result back (mamba_simple.py:230,264)."""

    @staticmethod
    @custom_fwd(device_type="cuda")
    def forward(ctx, xz, conv1d_weight, conv1d_bias, x_proj_weight, delta_proj_weight, A, B=None, C=None, D=None,
                delta_bias=None, B_proj_bias=None, C_proj_bias=None, delta_softplus=True, direction=0):
        if B is not None or C is not None or B_proj_bias is not None or C_proj_bias is not None:
            raise RuntimeError("segmamba_b200: only input-dependent B and C without projection bias are supported "
                               "(what Mamba.forward v3 passes, mamba_simple.py:217-260)")
        if A.is_complex():
            raise RuntimeError("segmamba_b200: complex A is out of scope")
        L = xz.shape[-1]
        delta_rank = delta_proj_weight.shape[1]
        d_state = A.shape[-1]
        if torch.is_autocast_enabled("cuda"):                                              # ssi.py:169-171
            x_proj_weight = x_proj_weight.to(dtype=torch.get_autocast_dtype("cuda"))
            delta_proj_weight = delta_proj_weight.to(dtype=torch.get_autocast_dtype("cuda"))
        if xz.stride(-1) != 1:
            xz = xz.contiguous()
        conv1d_weight = conv1d_weight.reshape(conv1d_weight.shape[0], conv1d_weight.shape[-1])   # "d 1 w -> d w"
        x, z = xz.chunk(2, dim=1)
        conv1d_bias = conv1d_bias.contiguous() if conv1d_bias is not None else None
        conv1d_out = causal_conv1d_cuda.causal_conv1d_fwd_ex(x, conv1d_weight, conv1d_bias, True, direction=direction)
        bsz, d_inner, _ = conv1d_out.shape
        # Everything below works on the channel-major (d, b*l) view of the activations ("HBL", ssi.py:178-182), which is
        # what conv1d_out already is in memory: x_proj / dt_proj become plain GEMMs on that view and B, C are strided
        # views of their result -- no 'b d l -> (b l) d' transpose copy (ssi.py:181) and no .contiguous() of B / C (:187-207).
        conv2 = _as_dbl(conv1d_out)                                                     # (d_inner, b*l)
        # dt_rank = ceil(d_model / 16) is 3 / 6 / 12 at the first three stages: GEMMs with a 3- or 6-element leading dimension
        # fall back to cuBLAS's unaligned legacy kernels (cutlass_75_*_align1).  The two small weights are therefore zero-padded so that the dt block of x_dbl has R8 =
        # 8 / 8 / 16 rows and B, C start on 8-row boundaries; the padding rows / columns are exact zeros everywhere.
        R8 = -(-delta_rank // 8) * 8 if ALIGN_GEMMS else delta_rank
        if R8 != delta_rank:
            x_proj_weight = torch.cat([x_proj_weight[:delta_rank], x_proj_weight.new_zeros(R8 - delta_rank, d_inner),
                                       x_proj_weight[delta_rank:]], dim=0)             # (R8+2N, d_inner)
            delta_proj_weight = torch.nn.functional.pad(delta_proj_weight, (0, R8 - delta_rank))   # (d_inner, R8)
        x_dblT = _gemm.product(x_proj_weight, conv2.t())                                # (R8+2N, b*l)  = x_dbl.t()   :181
        delta = _gemm.product(delta_proj_weight, x_dblT[:R8].t()).view(d_inner, bsz, L).permute(1, 0, 2)     # HBL          :182
        Bm = x_dblT[R8:R8 + d_state].view(d_state, bsz, L).permute(1, 0, 2).unsqueeze(1)                # (b,1,N,l) view
        Cm = x_dblT[R8 + d_state:].view(d_state, bsz, L).permute(1, 0, 2).unsqueeze(1)
        D = D.contiguous() if D is not None else None
        _, _, out_z, hst, hd = selective_scan_cuda.fwd_ex(conv1d_out, delta, A, Bm, Cm, D, z, delta_bias, delta_softplus, direction=direction,
                                                          want_out=False, want_x=False, want_hstates=True, want_hdense=True)
        ctx.delta_softplus = delta_softplus
        ctx.direction = direction
        ctx.delta_rank = delta_rank
        # checkpoint_lvl: the reference frees conv1d_out and delta and recomputes them in backward (ssi.py:216-219,238-241) to
        # fit 16-32 GB parts.  With 180 GB of HBM the two (b, d_inner, l) tensors are kept instead (1.6 GB per training step
        # of the default model at batch 2), which removes one conv1d launch and one GEMM per direction from the backward.
        keep = (conv1d_out, delta) if KEEP_CONV_DELTA else (None, None)
        ctx.save_for_backward(xz, conv1d_weight, conv1d_bias, x_dblT, x_proj_weight, delta_proj_weight, A, D, delta_bias, hst, hd, *keep)
        return out_z

    @staticmethod
    @custom_bwd(device_type="cuda")
    def backward(ctx, dout):
        (xz, conv1d_weight, conv1d_bias, x_dblT, x_proj_weight, delta_proj_weight, A, D, delta_bias, hst, hd,
         conv1d_out, delta) = ctx.saved_tensors
        L = xz.shape[-1]
        delta_rank, R8 = ctx.delta_rank, delta_proj_weight.shape[1]     # the saved weights carry the zero padding (see forward)
        d_state = A.shape[-1]
        direction = ctx.direction
        x, z = xz.chunk(2, dim=1)
        if dout.stride(-1) != 1:
            dout = dout.contiguous()
        if conv1d_out is None:                          # recompute conv1d_out and delta (ssi.py:238-241)
            conv1d_out = causal_conv1d_cuda.causal_conv1d_fwd_ex(x, conv1d_weight, conv1d_bias, True, direction=direction)
        bsz, d_inner, _ = conv1d_out.shape
        conv2 = _as_dbl(conv1d_out)
        if delta is None:
            delta = _gemm.product(delta_proj_weight, x_dblT[:R8].t()).view(d_inner, bsz, L).permute(1, 0, 2)
        Bm = x_dblT[R8:R8 + d_state].view(d_state, bsz, L).permute(1, 0, 2).unsqueeze(1)
        Cm = x_dblT[R8 + d_state:].view(d_state, bsz, L).permute(1, 0, 2).unsqueeze(1)
        dxz = torch.empty_like(xz)                      # dx and dz are written next to each other (ssi.py:244-245)
        dx, dz = dxz.chunk(2, dim=1)
        dconv1d_out, ddelta, dA, dB, dC, dD, ddelta_bias, dz, _ = selective_scan_cuda.bwd_ex(
            conv1d_out, delta, A, Bm, Cm, D, z, delta_bias, dout, dz, ctx.delta_softplus, False,
            direction=direction, hstates=hst, hdense=hd)
        dx_dblT = torch.empty_like(x_dblT)                                                                      # (R8+2N, b*l)
        dx_dblT[R8:R8 + d_state].view(d_state, bsz, L).copy_(dB.squeeze(1).permute(1, 0, 2))                    # :255-262
        dx_dblT[R8 + d_state:].view(d_state, bsz, L).copy_(dC.squeeze(1).permute(1, 0, 2))                      # :264-271
        ntok = bsz * L
        ddelta2 = _as_dbl(ddelta)                                                                               # :272
        ddelta_proj_weight = _gemm.product(ddelta2, x_dblT[:R8], ntok)                                          # :273
        # (R8, d) copy of the small weight: as a transposed VIEW its rows would be 16 bytes long, a TMA box shape that crawls
        _gemm.product(delta_proj_weight.t().contiguous(), ddelta2.t(), out=dx_dblT[:R8])   # rows delta_rank..R8 are exact zeros  :274
        dconv2 = _as_dbl(dconv1d_out)                                                                           # :275
        dx_proj_weight = _gemm.product(dx_dblT, conv2, ntok)                                                    # :276
        dconv2 = _gemm.product(x_proj_weight.t(), dx_dblT.t(), out=dconv2, accumulate=True)                     # :277
        if R8 != delta_rank:                                          # gradients of the un-padded parameters
            ddelta_proj_weight = ddelta_proj_weight[:, :delta_rank]
            dx_proj_weight = torch.cat([dx_proj_weight[:delta_rank], dx_proj_weight[R8:]], dim=0)
        dconv1d_out = dconv2.view(d_inner, bsz, L).permute(1, 0, 2)                                             # :278
        dx, dconv1d_weight, dconv1d_bias = causal_conv1d_cuda.causal_conv1d_bwd_ex(
            x, conv1d_weight, conv1d_bias, dconv1d_out, dx, True, direction=direction)                          # :281-283
        dconv1d_weight = dconv1d_weight.to(conv1d_weight.dtype).unsqueeze(1)                                    # "d w -> d 1 w"
        dconv1d_bias = dconv1d_bias.to(conv1d_bias.dtype) if conv1d_bias is not None else None
        return (dxz, dconv1d_weight, dconv1d_bias, dx_proj_weight, ddelta_proj_weight, dA, None, None,
                dD if D is not None else None, ddelta_bias if delta_bias is not None else None, None, None, None, None)


def mamba_inner_fn_no_out_proj(xz, conv1d_weight, conv1d_bias, x_proj_weight, delta_proj_weight, A, B=None, C=None,
                               D=None, delta_bias=None, B_proj_bias=None, C_proj_bias=None, delta_softplus=True,
                               direction=0):
    """ssi.py:627-633 plus the native ``direction`` extension (0 = the reference op)."""
    return MambaInnerFnNoOutProj.apply(xz, conv1d_weight, conv1d_bias, x_proj_weight, delta_proj_weight, A, B, C, D,
                                       delta_bias, B_proj_bias, C_proj_bias, delta_softplus, direction)
