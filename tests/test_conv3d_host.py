"""Host-side checks of the native 3x3x3 convolution (segmamba_b200/conv3d.py): the routing predicate, the data-gradient
weight re-layout and the ctypes layout of smb_conv3d_args."""
import ctypes

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from segmamba_b200 import _lib
from segmamba_b200 import conv3d as C

CL = torch.channels_last_3d


def _x(c, edge, layout=CL):
    return torch.empty(2, c, edge, edge, edge, device="meta").contiguous(memory_format=layout)


def test_routes_measured_shapes_native():
    for (ci, co, vox), passes in C.NATIVE_PASSES.items():
        edge = round(vox ** (1 / 3))
        assert edge ** 3 == vox and passes and set(passes) <= set("fdw")
        conv = nn.Conv3d(ci, co, 3, 1, 1, bias=False)
        for cd in (torch.bfloat16, torch.float16):
            assert C.shape_ok(conv, _x(ci, edge), cd), (ci, co, edge, cd)


@pytest.mark.parametrize("case", ["fp32", "c_in_4", "stem_7", "down_2", "transposed", "pointwise", "unmeasured_shape", "ncdhw",
                                  "dilated", "grouped", "cpu"])
def test_routes_everything_else_to_library(case):
    conv, x, cd = nn.Conv3d(48, 48, 3, 1, 1, bias=False), _x(48, 128), torch.bfloat16
    if case == "fp32":
        cd = torch.float32
    elif case == "c_in_4":                           # encoder1.conv1
        conv, x = nn.Conv3d(4, 48, 3, 1, 1, bias=False), _x(4, 128)
    elif case == "stem_7":
        conv, x = nn.Conv3d(4, 48, 7, 2, 3), _x(4, 128)
    elif case == "down_2":
        conv, x = nn.Conv3d(48, 96, 2, 2), _x(48, 64)
    elif case == "transposed":
        conv, x = nn.ConvTranspose3d(96, 48, 2, 2, bias=False), _x(96, 64)
    elif case == "pointwise":
        conv = nn.Conv3d(48, 48, 1)
    elif case == "unmeasured_shape":                  # a shape where cuDNN was as fast or faster in every pass
        conv, x = nn.Conv3d(384, 192, 3, 1, 1, bias=False), _x(384, 32)
    elif case == "ncdhw":
        x = _x(48, 128, torch.contiguous_format)
    elif case == "dilated":
        conv = nn.Conv3d(48, 48, 3, 1, 2, dilation=2, bias=False)
    elif case == "grouped":
        conv = nn.Conv3d(48, 48, 3, 1, 1, groups=2, bias=False)
    if case == "cpu":
        assert not C.native_ok(conv, torch.empty(1, 48, 64, 64, 64).contiguous(memory_format=CL))
    else:
        assert not C.shape_ok(conv, x, cd)


def test_library_path_unchanged_on_cpu():
    torch.manual_seed(0)
    conv = nn.Conv3d(8, 16, 3, 1, 1)
    x = torch.randn(1, 8, 5, 6, 7)
    assert torch.equal(C.conv3d(conv, x), conv(x))
    assert torch.equal(C.conv3d(conv, x, bias=False), F.conv3d(x, conv.weight, None, 1, 1))


@pytest.mark.parametrize("ci,co", [(8, 16), (16, 8), (24, 24)])
def test_dgrad_weight_relayout(ci, co):
    """the data gradient is a forward convolution of dY with dgrad_weight(W)"""
    torch.manual_seed(1)
    x = torch.randn(2, ci, 5, 6, 7, dtype=torch.float64, requires_grad=True)
    w = torch.randn(co, ci, 3, 3, 3, dtype=torch.float64)
    dy = torch.randn(2, co, 5, 6, 7, dtype=torch.float64)
    (gx,) = torch.autograd.grad(F.conv3d(x, w, None, 1, 1), x, dy)
    wd = C.dgrad_weight(w.permute(0, 2, 3, 4, 1))            # (C_in, 3, 3, 3, C_out) storage of the flipped weight
    assert wd.shape == (ci, 3, 3, 3, co) and wd.is_contiguous()
    gx2 = F.conv3d(dy, wd.permute(0, 4, 1, 2, 3), None, 1, 1)
    torch.testing.assert_close(gx2, gx, rtol=1e-12, atol=1e-12)


def test_ctypes_layout():
    a = _lib.Conv3dArgs
    assert [f[0] for f in a._fields_] == ["batch", "d", "h", "w", "c_in", "c_out", "dtype", "x", "weight", "y", "dy", "dweight"]
    assert a.x.offset == 32 and a.dweight.offset == 64 and ctypes.sizeof(a) == 72
    assert _lib.EXPORTS["smb_conv3d"][1][0]._type_ is a and _lib.EXPORTS["smb_conv3d_wgrad"][1][0]._type_ is a
