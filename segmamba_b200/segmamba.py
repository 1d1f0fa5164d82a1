"""SegMamba on the native hot path: same constructor, forward contract and state_dict surface as the reference's
``model_segmamba.segmamba.SegMamba`` (model_segmamba/segmamba.py:195-343), so checkpoints written by the reference's
3_train.py load with ``strict=True`` and the module drops into 3_train.py / 4_predict.py.

Module / attribute names reproduce the reference's 291 state_dict keys (SURVEY.md Appendix A):
``vit.{downsample_layers,stages,gscs,mlps}``, ``encoder{1..5}.layer.conv{1,2,3}.conv``,
``decoder{5..2}.{transp_conv.conv,conv_block.conv{1,2,3}.conv}``, ``decoder1.layer.conv{1,2}.conv``, ``out.conv.conv``.
The MONAI blocks are restated minimally (monai/networks/blocks/dynunet_block.py:25-111,247-267,
unetr_block.py:22-86,209-259, convolutions.py:25): dense Conv3d / ConvTranspose3d(k2,s2) without bias,
InstanceNorm3d(affine=False, eps=1e-5), LeakyReLU(0.01).  The dense 3x3x3 convolutions of UnetResBlock and GSC run on the
native implicit-GEMM kernel where conv3d.native_ok allows it (16-bit compute, large volumes); the other dense convolutions
are library (cuDNN) calls, as in the reference.  The TSMamba token mixer and every InstanceNorm(+activation+residual) chain
are native kernels.

Data layout: activations are kept channels-last (NDHWC) end to end, so (i) cuDNN's tensor-core convolutions need
no NCHW<->NHWC conversion kernels, (ii) the (B, L, C) token view that MambaLayer needs is free (the reference pays a
transpose copy each way, segmamba.py:69,74), and (iii) the fused instance-norm kernels stream full rows.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import gemm as _gemm
from . import conv3d as _conv3d
from . import layer_norm
from . import layout as _layout
from .instance_norm import fused_instance_norm
from .mamba_simple import Mamba

_CL = torch.channels_last_3d


class _ZeroGradBias(torch.autograd.Function):
    """identity on ``y`` that keeps ``bias`` in the graph with an exact zero gradient (see ``_conv_before_norm``)."""

    @staticmethod
    def forward(ctx, y, bias):
        ctx.bias_meta = (bias.shape, bias.dtype, bias.device)
        return y.view_as(y)

    @staticmethod
    def backward(ctx, g):
        shape, dtype, device = ctx.bias_meta
        return g, torch.zeros(shape, dtype=dtype, device=device)


def _conv_before_norm(conv: nn.Conv3d, x: torch.Tensor) -> torch.Tensor:
    """``conv(x)`` for a convolution whose output goes straight into an InstanceNorm (GSC, segmamba.py:111-128): its bias is a
    per-channel constant that the normalisation subtracts again, and the bias gradient -- the per-channel sum of a gradient that
    has passed through the norm -- is analytically zero.  So the bias is neither added (one full-tensor ATen kernel per
    convolution) nor reduced in the backward (one reduction per convolution); the parameter stays in the graph with an exact
    zero gradient, so weight decay acts on it exactly as in the reference and the state_dict surface is unchanged."""
    entry = _gemm.pointwise_conv if conv.kernel_size == (1, 1, 1) else _conv3d.conv3d
    if conv.bias is None:
        return entry(conv, x)
    return _ZeroGradBias.apply(entry(conv, x, bias=False), conv.bias)


class _Conv(nn.Sequential):
    """stand-in for monai Convolution(conv_only-like: act=None, norm=None): a Sequential with one child `conv`."""

    def __init__(self, cin, cout, kernel_size, stride=1, bias=False, transposed=False):
        super().__init__()
        if transposed:
            conv = nn.ConvTranspose3d(cin, cout, kernel_size=kernel_size, stride=stride, padding=0, output_padding=0, bias=bias)
        else:
            pad = (kernel_size - stride + 1) // 2            # get_padding(), dynunet_block.py:303-312
            conv = nn.Conv3d(cin, cout, kernel_size=kernel_size, stride=stride, padding=pad, bias=bias)
        self.add_module("conv", conv)


class UnetResBlock(nn.Module):
    """dynunet_block.py:25-111 with norm_name="instance" and the default leaky-relu."""

    def __init__(self, in_channels, out_channels, kernel_size=3, stride=1):
        super().__init__()
        self.conv1 = _Conv(in_channels, out_channels, kernel_size, stride)
        self.conv2 = _Conv(out_channels, out_channels, kernel_size, 1)
        self.lrelu = nn.LeakyReLU(negative_slope=0.01, inplace=True)
        self.norm1 = nn.InstanceNorm3d(out_channels)
        self.norm2 = nn.InstanceNorm3d(out_channels)
        self.downsample = in_channels != out_channels or stride != 1
        if self.downsample:
            self.conv3 = _Conv(in_channels, out_channels, 1, stride)
            self.norm3 = nn.InstanceNorm3d(out_channels)

    def forward(self, inp):
        # norm1/norm2/norm3/lrelu stay registered for structural parity; the math runs in the fused kernels
        out = fused_instance_norm(_conv3d.conv3d(self.conv1.conv, inp), "leaky_relu", 0.01)   # dynunet_block.py:100-102
        out = _conv3d.conv3d(self.conv2.conv, out)
        if self.downsample:                                                               # :105-110
            return fused_instance_norm(out, "leaky_relu", 0.01, add=_gemm.pointwise_conv(self.conv3.conv, inp), add_norm=True)
        return fused_instance_norm(out, "leaky_relu", 0.01, add=inp)


class UnetrBasicBlock(nn.Module):
    """unetr_block.py:209-259 with res_block=True."""

    def __init__(self, spatial_dims, in_channels, out_channels, kernel_size, stride, norm_name="instance", res_block=True):
        super().__init__()
        assert spatial_dims == 3 and res_block and norm_name == "instance"
        self.layer = UnetResBlock(in_channels, out_channels, kernel_size, stride)

    def forward(self, inp):
        return self.layer(inp)


class UnetrUpBlock(nn.Module):
    """unetr_block.py:22-86 with res_block=True."""

    def __init__(self, spatial_dims, in_channels, out_channels, kernel_size, upsample_kernel_size, norm_name="instance",
                 res_block=True):
        super().__init__()
        assert spatial_dims == 3 and res_block and norm_name == "instance"
        self.transp_conv = _Conv(in_channels, out_channels, upsample_kernel_size, upsample_kernel_size, transposed=True)
        self.conv_block = UnetResBlock(out_channels + out_channels, out_channels, kernel_size, 1)

    def forward(self, inp, skip):
        out = self.transp_conv(inp)
        if _layout.supported(out, skip):                    # channels-last, 16-bit or fp32 rows of 16-byte multiples: native copies
            out = _layout.cat_channels(out, skip)
        else:
            out = torch.cat((out, skip), dim=1)
        return self.conv_block(out)


class UnetOutBlock(nn.Module):
    """dynunet_block.py:247-267."""

    def __init__(self, spatial_dims, in_channels, out_channels):
        super().__init__()
        self.conv = _Conv(in_channels, out_channels, 1, 1, bias=True)

    def forward(self, inp):
        return self.conv(inp)


class MambaLayer(nn.Module):
    """segmamba.py:49-76."""

    def __init__(self, dim, d_state=16, d_conv=4, expand=2, num_slices=None):
        super().__init__()
        self.dim = dim
        self.norm = nn.LayerNorm(dim)
        self.mamba = Mamba(d_model=dim, d_state=d_state, d_conv=d_conv, expand=expand, bimamba_type="v3", nslices=num_slices)

    def forward(self, x):
        B, C = x.shape[:2]
        assert C == self.dim
        img_dims = x.shape[2:]
        n_tokens = img_dims.numel()
        if x.is_contiguous(memory_format=_CL):
            # channels-last storage IS the (B, L, C) token matrix: both reshapes are views
            x_flat = x.permute(0, 2, 3, 4, 1).reshape(B, n_tokens, C)
            if layer_norm.ENABLED and layer_norm.supported(x_flat, C):
                x_norm = layer_norm.fused_layer_norm(x_flat, self.norm.weight, self.norm.bias, self.norm.eps)
            else:
                x_norm = self.norm(x_flat)
            x_mamba = self.mamba(x_norm)
            out = x_mamba.reshape(B, *img_dims, C).permute(0, 4, 1, 2, 3)
            return out + x
        x_flat = x.reshape(B, C, n_tokens).transpose(-1, -2)
        x_norm = self.norm(x_flat)
        x_mamba = self.mamba(x_norm)
        out = x_mamba.transpose(-1, -2).reshape(B, C, *img_dims)
        return out + x


class MlpChannel(nn.Module):
    """segmamba.py:78-89."""

    def __init__(self, hidden_size, mlp_dim):
        super().__init__()
        self.fc1 = nn.Conv3d(hidden_size, mlp_dim, 1)
        self.act = nn.GELU()
        self.fc2 = nn.Conv3d(mlp_dim, hidden_size, 1)

    def forward(self, x):
        return _gemm.pointwise_conv(self.fc2, _gemm.pointwise_conv(self.fc1, x, gelu=True))   # act = exact-erf nn.GELU(), fused into fc1's epilogue


class GSC(nn.Module):
    """segmamba.py:91-132 (the two branches are summed, :127)."""

    def __init__(self, in_channles):
        super().__init__()
        self.proj = nn.Conv3d(in_channles, in_channles, 3, 1, 1)
        self.norm = nn.InstanceNorm3d(in_channles)
        self.nonliner = nn.ReLU()
        self.proj2 = nn.Conv3d(in_channles, in_channles, 3, 1, 1)
        self.norm2 = nn.InstanceNorm3d(in_channles)
        self.nonliner2 = nn.ReLU()
        self.proj3 = nn.Conv3d(in_channles, in_channles, 1, 1, 0)
        self.norm3 = nn.InstanceNorm3d(in_channles)
        self.nonliner3 = nn.ReLU()
        self.proj4 = nn.Conv3d(in_channles, in_channles, 1, 1, 0)
        self.norm4 = nn.InstanceNorm3d(in_channles)
        self.nonliner4 = nn.ReLU()

    def forward(self, x):
        x_residual = x
        x1 = fused_instance_norm(_conv_before_norm(self.proj, x), "relu")
        x1 = fused_instance_norm(_conv_before_norm(self.proj2, x1), "relu")
        x2 = fused_instance_norm(_conv_before_norm(self.proj3, x), "relu")
        x = fused_instance_norm(_conv_before_norm(self.proj4, x1 + x2), "relu")
        return x + x_residual


class MambaEncoder(nn.Module):
    """segmamba.py:134-193."""

    def __init__(self, in_chans=1, depths=[2, 2, 2, 2], dims=[48, 96, 192, 384], drop_path_rate=0.,
                 layer_scale_init_value=1e-6, out_indices=[0, 1, 2, 3]):
        super().__init__()
        self.downsample_layers = nn.ModuleList()
        self.downsample_layers.append(nn.Sequential(nn.Conv3d(in_chans, dims[0], kernel_size=7, stride=2, padding=3)))
        for i in range(3):
            self.downsample_layers.append(nn.Sequential(nn.InstanceNorm3d(dims[i]),
                                                        nn.Conv3d(dims[i], dims[i + 1], kernel_size=2, stride=2)))
        self.stages = nn.ModuleList()
        self.gscs = nn.ModuleList()
        num_slices_list = [64, 32, 16, 8]
        for i in range(4):
            self.stages.append(nn.Sequential(*[MambaLayer(dim=dims[i], num_slices=num_slices_list[i]) for _ in range(depths[i])]))
            self.gscs.append(GSC(dims[i]))
        self.out_indices = out_indices
        self.mlps = nn.ModuleList()
        for i_layer in range(4):
            self.add_module(f"norm{i_layer}", nn.InstanceNorm3d(dims[i_layer]))
            self.mlps.append(MlpChannel(dims[i_layer], 2 * dims[i_layer]))

    def forward_features(self, x):
        outs = []
        for i in range(4):
            if i == 0:
                x = self.downsample_layers[0][0](x)
            else:                                       # Sequential(InstanceNorm3d, Conv3d), segmamba.py:145-149
                x = self.downsample_layers[i][1](fused_instance_norm(x))
            x = self.gscs[i](x)
            x = self.stages[i](x)
            if i in self.out_indices:
                outs.append(self.mlps[i](fused_instance_norm(x)))          # norm{i} then MlpChannel, :183-187
        return tuple(outs)

    def forward(self, x):
        return self.forward_features(x)


class SegMamba(nn.Module):
    """segmamba.py:195-343."""

    def __init__(self, in_chans=1, out_chans=13, depths=[2, 2, 2, 2], feat_size=[48, 96, 192, 384], drop_path_rate=0,
                 layer_scale_init_value=1e-6, hidden_size: int = 768, norm_name="instance", conv_block: bool = True,
                 res_block: bool = True, spatial_dims=3) -> None:
        super().__init__()
        self.hidden_size = hidden_size
        self.in_chans = in_chans
        self.out_chans = out_chans
        self.depths = depths
        self.drop_path_rate = drop_path_rate
        self.feat_size = feat_size
        self.layer_scale_init_value = layer_scale_init_value
        self.spatial_dims = spatial_dims
        self.vit = MambaEncoder(in_chans, depths=depths, dims=feat_size, drop_path_rate=drop_path_rate,
                                layer_scale_init_value=layer_scale_init_value)
        kw = dict(spatial_dims=spatial_dims, norm_name=norm_name, res_block=res_block)
        self.encoder1 = UnetrBasicBlock(in_channels=in_chans, out_channels=feat_size[0], kernel_size=3, stride=1, **kw)
        self.encoder2 = UnetrBasicBlock(in_channels=feat_size[0], out_channels=feat_size[1], kernel_size=3, stride=1, **kw)
        self.encoder3 = UnetrBasicBlock(in_channels=feat_size[1], out_channels=feat_size[2], kernel_size=3, stride=1, **kw)
        self.encoder4 = UnetrBasicBlock(in_channels=feat_size[2], out_channels=feat_size[3], kernel_size=3, stride=1, **kw)
        self.encoder5 = UnetrBasicBlock(in_channels=feat_size[3], out_channels=hidden_size, kernel_size=3, stride=1, **kw)
        self.decoder5 = UnetrUpBlock(in_channels=hidden_size, out_channels=feat_size[3], kernel_size=3, upsample_kernel_size=2, **kw)
        self.decoder4 = UnetrUpBlock(in_channels=feat_size[3], out_channels=feat_size[2], kernel_size=3, upsample_kernel_size=2, **kw)
        self.decoder3 = UnetrUpBlock(in_channels=feat_size[2], out_channels=feat_size[1], kernel_size=3, upsample_kernel_size=2, **kw)
        self.decoder2 = UnetrUpBlock(in_channels=feat_size[1], out_channels=feat_size[0], kernel_size=3, upsample_kernel_size=2, **kw)
        self.decoder1 = UnetrBasicBlock(in_channels=feat_size[0], out_channels=feat_size[0], kernel_size=3, stride=1, **kw)
        # the reference hard-codes in_channels=48 here (segmamba.py:319)
        self.out = UnetOutBlock(spatial_dims=spatial_dims, in_channels=48, out_channels=out_chans)
        # conv weights in channels-last storage (values / state_dict unchanged)
        self.to(memory_format=_CL)

    def forward(self, x_in):
        x_in = x_in.contiguous(memory_format=_CL)
        outs = self.vit(x_in)
        enc1 = self.encoder1(x_in)
        enc2 = self.encoder2(outs[0])
        enc3 = self.encoder3(outs[1])
        enc4 = self.encoder4(outs[2])
        enc_hidden = self.encoder5(outs[3])
        dec3 = self.decoder5(enc_hidden, enc4)
        dec2 = self.decoder4(dec3, enc3)
        dec1 = self.decoder3(dec2, enc2)
        dec0 = self.decoder2(dec1, enc1)
        out = self.decoder1(dec0)
        return self.out(out).contiguous()
