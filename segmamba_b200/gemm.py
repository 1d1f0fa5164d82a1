"""Pointwise contractions on the tensor-core GEMM of libsegmamba_b200 (smb_gemm: TMA -> wgmma, accumulator in registers).

``gemm(a, b, ...)`` computes  D[M, N] = epilogue(A[M, K] . B[N, K]^T)  from 2-D views of 16-bit tensors: an operand whose
last axis is contiguous is passed K-major, an operand whose FIRST axis is contiguous (a transposed view) is passed MN-major,
so no operand is ever copied.  ``linear`` is ``F.linear`` (y = x W^T + b, optional exact GELU) with a native backward:
dx = dy . W (the weight as an MN-major operand), dW = dy^T . x (both operands MN-major, K = tokens split over CTAs, fp32
atomics), db = column sums from the same kernel with a ones operand folded in by the caller -- here a plain fp32 reduction.
Replaces cuBLAS / cuDNN behind Mamba.in_proj / out_proj (mamba_simple.py:204-208,264), MlpChannel (segmamba.py:81-89),
GSC.proj3 / proj4 (segmamba.py:103-107) and UnetResBlock.conv3 (dynunet_block.py:66-69).  No fallback: unsupported operands raise.
"""
from __future__ import annotations

import ctypes
import os

import torch
from torch.amp import custom_bwd, custom_fwd

from . import _lib

EPI_NONE, EPI_BIAS_N, EPI_BIAS_N_GELU, EPI_BIAS_M = 0, 1, 2, 3

# Which products of the model run on the native kernel (the split is not re-measured per shape on H100):
#   "auto" (default)  the products that contract over the token axis -- every weight gradient of the mixer (dW of in_proj /
#                     x_proj / dt_proj / out_proj; K = 65 536 ... 524 288 tokens split over the SMs with fp32 atomics); the
#                     activation-sized products (output = tokens x channels) stay library calls, as in the reference;
#   "all"             every pointwise contraction and 1x1x1 convolution;      "off"  none.
MODE = os.environ.get("SMB_GEMM", "auto")
SPLIT_TOKENS = 16384     # contraction length from which the split-K path is used (and wins)


def _operand(t: torch.Tensor, what: str):
    """(major, ld) of a 2-D (rows = M or N, cols = K) view; raises if neither axis is contiguous."""
    if t.dim() != 2:
        raise RuntimeError(f"gemm: {what} must be 2-D")
    if t.stride(1) == 1 and (t.stride(0) >= t.shape[1] or t.shape[0] == 1):
        major, ld = 0, (t.stride(0) if t.shape[0] > 1 else max(t.shape[1], 8))
    elif t.stride(0) == 1 and (t.stride(1) >= t.shape[0] or t.shape[1] == 1):
        major, ld = 1, (t.stride(1) if t.shape[1] > 1 else max(t.shape[0], 8))
    else:
        raise RuntimeError(f"gemm: {what} needs one contiguous axis (strides {t.stride()})")
    if ld % 8 or t.data_ptr() % 16:
        raise RuntimeError(f"gemm: {what} needs 16-byte aligned rows (ld {ld}, ptr % 16 = {t.data_ptr() % 16})")
    return major, ld


def supported(a: torch.Tensor, b: torch.Tensor) -> bool:
    try:
        if a.dtype != b.dtype or a.dtype not in (torch.float16, torch.bfloat16) or not a.is_cuda:
            return False
        _operand(a, "A"), _operand(b, "B")
        return True
    except RuntimeError:
        return False


def gemm(a: torch.Tensor, b: torch.Tensor, bias: torch.Tensor | None = None, epilogue: int = EPI_NONE,
         out_dtype: torch.dtype | None = None, out: torch.Tensor | None = None, split_k: int = 1, accumulate: bool = False):
    """D[M, N] = epilogue(a[M, K] @ b[N, K].T); a, b: fp16 / bf16 2-D views (see module docstring)."""
    _lib.require_cuda(a, b, bias, out)
    if a.dtype != b.dtype or a.dtype not in (torch.float16, torch.bfloat16):
        raise RuntimeError(f"gemm: operands must both be fp16 or bf16 (got {a.dtype}, {b.dtype})")
    M, K = a.shape
    N, Kb = b.shape
    if K != Kb:
        raise RuntimeError(f"gemm: inner dimensions differ ({K} vs {Kb})")
    am, lda = _operand(a, "A")
    bm, ldb = _operand(b, "B")
    od = out_dtype or a.dtype
    dev = a.device
    with torch.cuda.device(dev):
        if out is None:
            out = (torch.zeros if (split_k > 1 or accumulate) else torch.empty)((M, N), dtype=od, device=dev)
        elif out.shape != (M, N) or out.stride(1) != 1 or out.dtype != od:
            raise RuntimeError("gemm: out must be (M, N) with unit column stride in out_dtype")
        if bias is not None:
            bias = bias.float().contiguous()
        g = _lib.GemmArgs()
        g.M, g.N, g.K = M, N, K
        g.dtype, g.out_dtype = _lib.dtype_code(a.dtype), _lib.dtype_code(od)
        g.a_major, g.b_major, g.epilogue, g.split_k, g.accumulate = am, bm, epilogue, int(split_k), int(bool(accumulate))
        g.A, g.B, g.bias, g.D = _lib.ptr(a), _lib.ptr(b), _lib.ptr(bias), _lib.ptr(out)
        g.lda, g.ldb, g.ldd = lda, ldb, (out.stride(0) if M > 1 else N)
        sp = _lib.stream_ptr(dev)
        _lib.call("gemm", (M, N, K, am, bm, epilogue, split_k, a.element_size()), lambda: _lib.lib().smb_gemm(ctypes.byref(g), sp), dev)
    return out


def _split_k_for(tokens: int) -> int:
    """weight-gradient products contract over the token axis: one K slice per ~SM, at least 512 tokens each."""
    return max(1, min(132, tokens // 512))


class _Linear(torch.autograd.Function):
    """y = act(x W^T + b) over the last axis of x (any leading shape, last axis contiguous)."""

    @staticmethod
    @custom_fwd(device_type="cuda", cast_inputs=None)
    def forward(ctx, x, weight, bias, gelu, compute_dtype):
        cd = compute_dtype
        x2 = x.reshape(-1, x.shape[-1])
        xq = x2 if x2.dtype == cd else x2.to(cd)
        wq = weight if weight.dtype == cd else weight.to(cd)
        wq = wq.reshape(weight.shape[0], -1)
        epi = EPI_NONE if bias is None else (EPI_BIAS_N_GELU if gelu else EPI_BIAS_N)
        if gelu and bias is None:
            raise RuntimeError("linear: gelu epilogue needs a bias (pass zeros)")
        if MODE == "all":
            y = gemm(xq, wq, bias, epi)                       # bias (+ exact GELU) applied in the accumulator epilogue
        else:
            y = torch.nn.functional.linear(xq, wq, bias.to(cd) if bias is not None else None)
            if gelu:
                y = torch.nn.functional.gelu(y)
        ctx.save_for_backward(xq, wq, bias if gelu else None)   # the pre-activation is recomputed in the backward
        ctx.gelu, ctx.has_bias = gelu, bias is not None
        ctx.x_dtype, ctx.w_dtype, ctx.w_shape = x.dtype, weight.dtype, weight.shape
        ctx.b_dtype = bias.dtype if bias is not None else None
        return y.reshape(*x.shape[:-1], weight.shape[0])

    @staticmethod
    @custom_bwd(device_type="cuda")
    def backward(ctx, dy):
        xq, wq, bias = ctx.saved_tensors
        dy2 = dy.reshape(-1, dy.shape[-1])
        if dy2.dtype != xq.dtype:
            dy2 = dy2.to(xq.dtype)
        if not dy2.is_contiguous():
            dy2 = dy2.contiguous()
        if ctx.gelu:
            p32 = (gemm(xq, wq, bias, EPI_BIAS_N, out_dtype=torch.float32) if MODE == "all"
                   else torch.nn.functional.linear(xq, wq, bias.to(xq.dtype)).float())
            cdf = 0.5 * (1 + torch.erf(p32 * 0.7071067811865476))
            pdf = torch.exp(-0.5 * p32 * p32) * 0.3989422804014327
            dy2 = (dy2.float() * (cdf + p32 * pdf)).to(xq.dtype)
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = (gemm(dy2, wq.t()) if MODE == "all" else dy2 @ wq)                            # (tokens, N) x (C_in, N)^T
            dx = dx.reshape(*dy.shape[:-1], wq.shape[1]).to(ctx.x_dtype)
        if ctx.needs_input_grad[1]:
            if MODE == "all" or (MODE == "auto" and dy2.shape[0] >= SPLIT_TOKENS and supported(dy2.t(), xq.t())):
                dw = gemm(dy2.t(), xq.t(), out_dtype=torch.float32, split_k=_split_k_for(dy2.shape[0]))   # (N, tokens) x (C_in, tokens)^T
            else:
                dw = dy2.t() @ xq
            dw = dw.reshape(ctx.w_shape).to(ctx.w_dtype)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = dy2.float().sum(0).to(ctx.b_dtype)
        return dx, dw, db, None, None


def _is_mn(t: torch.Tensor) -> bool:
    return t.stride(0) == 1 and t.stride(1) != 1


class _MatmulNT(torch.autograd.Function):
    """D = a @ b.T for 2-D operands of either major (a: (M, K), b: (N, K)), 16-bit arithmetic operands, fp32 accumulation.
    Gradients on the same kernel: da = dD @ b (B operand = b.T view), db = dD.T @ a (both operands transposed views)."""

    @staticmethod
    @custom_fwd(device_type="cuda", cast_inputs=None)
    def forward(ctx, a, b, compute_dtype, out_dtype):
        aq = a if a.dtype == compute_dtype else a.to(compute_dtype)
        bq = b if b.dtype == compute_dtype else b.to(compute_dtype)
        ctx.save_for_backward(aq, bq)
        ctx.a_dtype, ctx.b_dtype = a.dtype, b.dtype
        if MODE != "all":
            return (aq @ bq.t()).to(out_dtype or compute_dtype)
        return gemm(aq, bq, out_dtype=out_dtype or compute_dtype)

    @staticmethod
    @custom_bwd(device_type="cuda")
    def backward(ctx, dD):
        aq, bq = ctx.saved_tensors
        if dD.dtype != aq.dtype:
            dD = dD.to(aq.dtype)
        if not (dD.stride(1) == 1 or dD.stride(0) == 1):
            dD = dD.contiguous()
        da = db = None
        M, N = dD.shape
        K = aq.shape[1]
        # each gradient is produced in the storage layout of its operand (an MN-major operand gets the transposed product),
        # so no transpose copy follows: e.g. out_proj's activation gradient comes out channel-major, as the scans want it
        def prod(x, y, big, contraction):
            """x @ y.T; native when the routing says so (see MODE)"""
            if MODE == "all" or (MODE == "auto" and big and supported(x, y)):
                return gemm(x, y, out_dtype=torch.float32 if big else None, split_k=_split_k_for(contraction) if big else 1)
            return x @ y.t()
        if ctx.needs_input_grad[0]:          # da = dD @ b: contraction over N
            big = N >= SPLIT_TOKENS and M * K <= 1 << 21
            da = prod(bq.t(), dD, big, N).t() if _is_mn(aq) else prod(dD, bq.t(), big, N)
            da = da.to(ctx.a_dtype)
        if ctx.needs_input_grad[1]:          # db = dD.T @ a: contraction over M
            big = M >= SPLIT_TOKENS and N * K <= 1 << 21
            db = prod(aq.t(), dD.t(), big, M).t() if _is_mn(bq) else prod(dD.t(), aq.t(), big, M)
            db = db.to(ctx.b_dtype)
        return da, db, None, None


def matmul_nt(a: torch.Tensor, b: torch.Tensor, compute_dtype: torch.dtype | None = None, out_dtype: torch.dtype | None = None):
    """a @ b.T on the native GEMM (differentiable).  a: (M, K), b: (N, K); each needs one contiguous axis."""
    if compute_dtype is None:
        if torch.is_autocast_enabled("cuda"):
            compute_dtype = torch.get_autocast_dtype("cuda")
        else:
            compute_dtype = a.dtype if a.dtype in (torch.float16, torch.bfloat16) else b.dtype
    if compute_dtype not in (torch.float16, torch.bfloat16):
        raise RuntimeError("gemm.matmul_nt: 16-bit operands only (fp32 inputs need autocast or compute_dtype)")
    return _MatmulNT.apply(a, b, compute_dtype, out_dtype)


def conv1x1(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor | None = None, gelu: bool = False) -> torch.Tensor:
    """nn.Conv3d(kernel_size=1) on a channels-last (NDHWC storage) activation: one (tokens, C_in) x (C_out, C_in)^T product.
    Returns a channels-last tensor of logical shape (B, C_out, D, H, W)."""
    Bz, C = x.shape[:2]
    sp = x.shape[2:]
    xt = x.permute(0, 2, 3, 4, 1)
    if not xt.is_contiguous():
        raise RuntimeError("gemm.conv1x1: channels-last activation expected")
    y = linear(xt.reshape(-1, C), weight.reshape(weight.shape[0], C), bias, gelu=gelu)
    return y.reshape(Bz, *sp, weight.shape[0]).permute(0, 4, 1, 2, 3)


def linear(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor | None = None, gelu: bool = False,
           compute_dtype: torch.dtype | None = None) -> torch.Tensor:
    """F.linear on the native GEMM.  compute_dtype: operand dtype (default: the autocast dtype when autocast is on, else
    x.dtype, which must then be fp16 / bf16)."""
    if compute_dtype is None:
        compute_dtype = torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled("cuda") else x.dtype
    if compute_dtype not in (torch.float16, torch.bfloat16):
        raise RuntimeError("gemm.linear: 16-bit operands only (fp32 inputs need autocast or compute_dtype)")
    return _Linear.apply(x, weight, bias, gelu, compute_dtype)
