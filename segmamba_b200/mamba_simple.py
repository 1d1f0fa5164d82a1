"""Tri-directional Mamba mixer (``bimamba_type="v3"``) on the native kernels.

Same constructor arguments, parameter names/shapes/initialisation and forward contract as the reference's
``mamba_ssm.Mamba`` (mamba/mamba_ssm/modules/mamba_simple.py:34-264), restricted to what SegMamba uses: the v3
fast path.  The decode-time ``step``, the v2/none branches and ``Block`` are out of scope (never reached by
``MambaLayer``, SURVEY.md section 2.1 #2).
"""
from __future__ import annotations

import math
import os

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import causal_conv1d_cuda
from ._lib import DIR_FORWARD, DIR_REVERSE
from . import gemm as _gemm
from .selective_scan_interface import mamba_inner_fn_no_out_proj


# opt-in: run the three directional passes of a mixer on separate CUDA streams (see Mamba.forward)
def _tc_ok(x2d, weight):
    """the native GEMM takes 16-bit operands: autocast on, or 16-bit activations; rows must be 16-byte multiples"""
    cd = torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled("cuda") else x2d.dtype
    return (_gemm.MODE != "off" and x2d.is_cuda and cd in (torch.float16, torch.bfloat16) and x2d.shape[1] % 8 == 0 and weight.shape[0] % 8 == 0
            and x2d.shape[0] % 8 == 0)


DIRECTION_STREAMS = os.environ.get("SMB_DIR_STREAMS", "0") == "1"
_SIDE_STREAMS = {}


def _side_streams(device):
    key = (device.type, device.index)
    if key not in _SIDE_STREAMS:
        _SIDE_STREAMS[key] = (torch.cuda.Stream(device=device), torch.cuda.Stream(device=device))
    return _SIDE_STREAMS[key]


class Mamba(nn.Module):
    def __init__(self, d_model, d_state=16, d_conv=4, expand=2, dt_rank="auto", dt_min=0.001, dt_max=0.1,
                 dt_init="random", dt_scale=1.0, dt_init_floor=1e-4, conv_bias=True, bias=False, use_fast_path=True,
                 layer_idx=None, device=None, dtype=None, bimamba_type="v3", nslices=5):
        factory_kwargs = {"device": device, "dtype": dtype}
        super().__init__()
        if bimamba_type != "v3":
            raise ValueError('segmamba_b200.Mamba implements bimamba_type="v3" only (mamba_simple.py:125 asserts the same)')
        self.d_model = d_model
        self.d_state = d_state
        self.d_conv = d_conv
        self.expand = expand
        self.d_inner = int(self.expand * self.d_model)
        self.dt_rank = math.ceil(self.d_model / 16) if dt_rank == "auto" else dt_rank
        self.use_fast_path = use_fast_path
        self.layer_idx = layer_idx
        self.bimamba_type = bimamba_type
        self.nslices = nslices

        # registration order follows mamba_simple.py:69-186 so that state_dict() key order is identical
        self.in_proj = nn.Linear(self.d_model, self.d_inner * 2, bias=bias, **factory_kwargs)
        self.conv1d = self._make_conv(conv_bias, factory_kwargs)
        self.activation = "silu"
        self.act = nn.SiLU()
        self.x_proj = nn.Linear(self.d_inner, self.dt_rank + self.d_state * 2, bias=False, **factory_kwargs)
        self.dt_proj = nn.Linear(self.dt_rank, self.d_inner, bias=True, **factory_kwargs)

        # dt projection init of the forward direction only (mamba_simple.py:89-108; the _b/_s twins keep nn.Linear's default)
        dt_init_std = self.dt_rank ** -0.5 * dt_scale
        if dt_init == "constant":
            nn.init.constant_(self.dt_proj.weight, dt_init_std)
        elif dt_init == "random":
            nn.init.uniform_(self.dt_proj.weight, -dt_init_std, dt_init_std)
        else:
            raise NotImplementedError
        dt = torch.exp(torch.rand(self.d_inner, **factory_kwargs) * (math.log(dt_max) - math.log(dt_min))
                       + math.log(dt_min)).clamp(min=dt_init_floor)
        inv_dt = dt + torch.log(-torch.expm1(-dt))
        with torch.no_grad():
            self.dt_proj.bias.copy_(inv_dt)
        self.dt_proj.bias._no_reinit = True

        self.A_log = self._make_A_log(device)
        self.D = self._make_D(device)

        self.A_b_log = self._make_A_log(device)
        self.conv1d_b = self._make_conv(conv_bias, factory_kwargs)
        self.x_proj_b = nn.Linear(self.d_inner, self.dt_rank + self.d_state * 2, bias=False, **factory_kwargs)
        self.dt_proj_b = nn.Linear(self.dt_rank, self.d_inner, bias=True, **factory_kwargs)
        self.D_b = self._make_D(device)

        self.A_s_log = self._make_A_log(device)
        self.conv1d_s = self._make_conv(conv_bias, factory_kwargs)
        self.x_proj_s = nn.Linear(self.d_inner, self.dt_rank + self.d_state * 2, bias=False, **factory_kwargs)
        self.dt_proj_s = nn.Linear(self.dt_rank, self.d_inner, bias=True, **factory_kwargs)
        self.D_s = self._make_D(device)

        self.out_proj = nn.Linear(self.d_inner, self.d_model, bias=bias, **factory_kwargs)

    def _make_conv(self, conv_bias, factory_kwargs):
        return nn.Conv1d(in_channels=self.d_inner, out_channels=self.d_inner, bias=conv_bias, kernel_size=self.d_conv,
                         groups=self.d_inner, padding=self.d_conv - 1, **factory_kwargs)

    def _make_A_log(self, device):
        A = torch.arange(1, self.d_state + 1, dtype=torch.float32, device=device).repeat(self.d_inner, 1).contiguous()
        p = nn.Parameter(torch.log(A))          # S4D-real init, kept in fp32 (mamba_simple.py:111-118)
        p._no_weight_decay = True
        return p

    def _make_D(self, device):
        p = nn.Parameter(torch.ones(self.d_inner, device=device))
        p._no_weight_decay = True
        return p

    def forward(self, hidden_states, inference_params=None):
        """hidden_states: (B, L, D) -> (B, L, D)   (mamba_simple.py:188-264, v3 branch)."""
        if inference_params is not None:
            raise RuntimeError("segmamba_b200.Mamba: decoding with inference_params is out of scope")
        batch, seqlen, _ = hidden_states.shape
        if seqlen % self.nslices != 0:
            raise RuntimeError(f"Mamba v3: seqlen {seqlen} is not divisible by nslices {self.nslices}")
        # matmul and transpose BLH -> HBL at the same time (mamba_simple.py:204-208)
        x2d = hidden_states.reshape(batch * seqlen, -1)
        tc = _tc_ok(x2d, self.in_proj.weight)                 # 16-bit arithmetic (autocast): the native tensor-core GEMM
        if tc:
            xz = _gemm.matmul_nt(self.in_proj.weight, x2d).view(-1, batch, seqlen).permute(1, 0, 2)
        else:
            xz = (self.in_proj.weight @ x2d.t()).view(-1, batch, seqlen).permute(1, 0, 2)
        if self.in_proj.bias is not None:
            xz = xz + self.in_proj.bias.to(dtype=xz.dtype)[None, :, None]

        def inner(xz_dir, sfx, direction):
            A = -torch.exp(getattr(self, f"A{sfx}_log").float())
            return mamba_inner_fn_no_out_proj(
                xz_dir, getattr(self, f"conv1d{sfx}").weight, getattr(self, f"conv1d{sfx}").bias,
                getattr(self, f"x_proj{sfx}").weight, getattr(self, f"dt_proj{sfx}").weight, A, None, None,
                getattr(self, f"D{sfx}").float(), delta_bias=getattr(self, f"dt_proj{sfx}").bias.float(),
                delta_softplus=True, direction=direction)

        def slice_pass():
            xz_s = _SeqPermute.apply(xz, self.nslices, False)              # :245-247
            return _SeqPermute.apply(inner(xz_s, "_s", DIR_FORWARD), self.nslices, True)    # :248-261

        if DIRECTION_STREAMS and xz.is_cuda:
            # The three directional passes are independent until the sum below.  At the deep stages (L = 4096 / 512) one pass
            # cannot fill 132 SMs, so the reversed and the inter-slice pass are enqueued on two side streams (forked from and
            # joined to the caller's stream; inside a CUDA-graph capture these become parallel branches).  Autograd replays
            # each branch's backward on the stream its forward ran on.  Opt-in until measured (SMB_DIR_STREAMS=1).
            cur = torch.cuda.current_stream()
            s_b, s_s = _side_streams(xz.device)
            s_b.wait_stream(cur)
            s_s.wait_stream(cur)
            xz.record_stream(s_b)
            xz.record_stream(s_s)
            with torch.cuda.stream(s_b):
                out_b = inner(xz, "_b", DIR_REVERSE)
            with torch.cuda.stream(s_s):
                out_s = slice_pass()
            out = inner(xz, "", DIR_FORWARD)
            cur.wait_stream(s_b)
            cur.wait_stream(s_s)
            out_b.record_stream(cur)
            out_s.record_stream(cur)
        else:
            out = inner(xz, "", DIR_FORWARD)                               # :217-229
            out_b = inner(xz, "_b", DIR_REVERSE)                           # :230-242 without the flip copies
            out_s = slice_pass()
        y = out + out_b + out_s
        if tc and self.out_proj.bias is None:
            # (b l, d) x (C, d)^T: y stays in its channel-major storage, it enters the GEMM as an MN-major operand
            y2d = y.permute(1, 0, 2).reshape(y.shape[1], batch * seqlen)
            return _gemm.matmul_nt(y2d.t(), self.out_proj.weight).view(batch, seqlen, -1)
        return F.linear(y.permute(0, 2, 1), self.out_proj.weight, self.out_proj.bias)     # :264


class _SeqPermute(torch.autograd.Function):
    """inter-slice re-ordering of the token axis (smb_seq_permute); its adjoint is the inverse permutation."""

    @staticmethod
    def forward(ctx, x, nslices, inverse):
        ctx.nslices, ctx.inverse = nslices, inverse
        return causal_conv1d_cuda.seq_permute(x, nslices, inverse=inverse)

    @staticmethod
    def backward(ctx, g):
        return causal_conv1d_cuda.seq_permute(g, ctx.nslices, inverse=not ctx.inverse), None, None
