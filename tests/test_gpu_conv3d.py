"""Implicit-GEMM 3x3x3 convolution (smb_conv3d / smb_conv3d_wgrad) against an fp32 F.conv3d and its autograd on the same
16-bit-rounded operands: every 3x3x3 shape of the default model at 128^3 and 64^3 (batch 2), ragged shapes, a batch whose
samples differ by orders of magnitude (leakage across the sample boundary), the autograd wrapper under autocast against
nn.Conv3d, bitwise reruns, freedom from host synchronisation and CUDA-graph capture."""
import pytest
import torch
import torch.nn.functional as F

from util import assert_close

pytestmark = pytest.mark.gpu

# (C_in, C_out, edge): the 3x3x3 convolutions of the default model at 128^3 and 64^3 (UnetResBlock conv1 / conv2, GSC proj / proj2)
MODEL = [(48, 48, 128), (96, 48, 128), (48, 48, 64), (48, 96, 64), (96, 96, 64), (192, 96, 64)]
# (batch, C_in, C_out, D, H, W)
RAGGED = [(1, 16, 16, 8, 9, 130), (2, 48, 48, 13, 17, 19), (1, 96, 192, 13, 17, 19), (1, 192, 48, 5, 6, 7), (2, 16, 96, 3, 4, 40),
          (1, 48, 384, 8, 8, 8)]


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = old


def _inputs(b, ci, co, d, h, w, dtype, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(b, ci, d, h, w, device="cuda", generator=g).to(dtype)
    wt = (torch.randn(co, ci, 3, 3, 3, device="cuda", generator=g) / (27 * ci) ** 0.5).to(dtype)
    dy = torch.randn(b, co, d, h, w, device="cuda", generator=g).to(dtype)
    return x, wt, dy


def _reference(x, wt, dy):
    xr, wr = x.float().requires_grad_(), wt.float().requires_grad_()
    y = F.conv3d(xr, wr, None, 1, 1)
    gx, gw = torch.autograd.grad(y, (xr, wr), dy.float())
    return y, gx, gw


def _cl5(t):
    return t.permute(0, 2, 3, 4, 1).contiguous()


def _check(x, wt, dy, wgrad_tol=1e-3):
    from segmamba_b200 import conv3d as C
    y, gx, gw = _reference(x, wt, dy)
    x5, w5, dy5 = _cl5(x), _cl5(wt), _cl5(dy)
    yn = C.conv3d_fwd(x5, w5).permute(0, 4, 1, 2, 3)
    dxn = C.conv3d_dgrad(dy5, w5).permute(0, 4, 1, 2, 3)
    dwn = C.conv3d_wgrad(x5, dy5).permute(0, 4, 1, 2, 3)
    assert yn.dtype == x.dtype and dwn.dtype == torch.float32
    assert_close(yn, y, 1e-2, "y")
    assert_close(dxn, gx, 1e-2, "dx")
    assert_close(dwn, gw, wgrad_tol, "dW")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("ci,co,edge", MODEL)
def test_model_shapes(ci, co, edge, dtype):
    _check(*_inputs(2, ci, co, edge, edge, edge, dtype))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("b,ci,co,d,h,w", RAGGED)
def test_ragged(b, ci, co, d, h, w, dtype):
    _check(*_inputs(b, ci, co, d, h, w, dtype, seed=1))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_sample_boundary(dtype):
    """sample 0 all zero, sample 1 large: any read across the batch boundary shows up in sample 0's outputs"""
    from segmamba_b200 import conv3d as C
    x, wt, dy = _inputs(2, 48, 48, 16, 16, 64, dtype, seed=2)
    x[0].zero_()
    dy[0].zero_()
    x[1] *= 100
    dy[1] *= 100
    _check(x, wt, dy)
    y0 = C.conv3d_fwd(_cl5(x), _cl5(wt))[0]
    dx0 = C.conv3d_dgrad(_cl5(dy), _cl5(wt))[0]
    assert int(torch.count_nonzero(y0)) == 0 and int(torch.count_nonzero(dx0)) == 0


@pytest.mark.parametrize("ci,co,edge", [(48, 96, 64), (192, 96, 64), (96, 192, 32)])
def test_autograd_autocast_matches_conv3d(ci, co, edge):
    """routed shapes whose native passes differ: forward only, weight gradient only, data gradient only"""
    from segmamba_b200 import conv3d as C
    torch.manual_seed(3)
    conv = torch.nn.Conv3d(ci, co, 3, 1, 1, bias=False).cuda().to(memory_format=torch.channels_last_3d)
    x = torch.randn(2, ci, edge, edge, edge, device="cuda").contiguous(memory_format=torch.channels_last_3d).requires_grad_()
    dy = torch.randn(2, co, edge, edge, edge, device="cuda")
    with torch.autocast("cuda", dtype=torch.bfloat16):
        assert C.native_ok(conv, x)
        y = C.conv3d(conv, x)
    assert y.dtype == torch.bfloat16 and y.is_contiguous(memory_format=torch.channels_last_3d)
    gx, gw = torch.autograd.grad(y, (x, conv.weight), dy)
    assert gx.dtype == torch.float32 and gw.dtype == torch.float32 and gw.shape == conv.weight.shape
    # the reference: the library convolution of the same bf16-rounded operands in fp32
    y_ref, gx_ref, gw_ref = _reference(x.detach().bfloat16(), conv.weight.detach().bfloat16(), dy.bfloat16())
    assert_close(y, y_ref, 1e-2, "y")
    assert_close(gx, gx_ref, 1e-2, "dx")
    # the native weight gradient is fp32; cuDNN's comes out in the 16-bit compute dtype
    assert_close(gw, gw_ref, 1e-3 if "w" in C.NATIVE_PASSES[(ci, co, edge ** 3)] else 1e-2, "dW")
    with torch.autocast("cuda", dtype=torch.bfloat16):
        y_lib = conv(x)
    assert_close(y, y_lib.float(), 1e-2, "y vs nn.Conv3d")


def test_rerun_bitwise_and_no_sync():
    from segmamba_b200 import conv3d as C
    x, wt, dy = _inputs(2, 48, 48, 64, 64, 64, torch.bfloat16, seed=4)
    x5, w5, dy5 = _cl5(x), _cl5(wt), _cl5(dy)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        y1, d1 = C.conv3d_fwd(x5, w5), C.conv3d_dgrad(dy5, w5)
        y2, d2 = C.conv3d_fwd(x5, w5), C.conv3d_dgrad(dy5, w5)
        w1 = C.conv3d_wgrad(x5, dy5)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(y1, y2) and torch.equal(d1, d2)
    assert torch.isfinite(w1).all()


def test_cuda_graph_capture():
    from segmamba_b200 import conv3d as C
    x, wt, dy = _inputs(2, 96, 48, 32, 32, 32, torch.bfloat16, seed=5)
    x5, w5, dy5 = _cl5(x), _cl5(wt), _cl5(dy)
    ref = (C.conv3d_fwd(x5, w5), C.conv3d_dgrad(dy5, w5), C.conv3d_wgrad(x5, dy5))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        C.conv3d_fwd(x5, w5)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = (C.conv3d_fwd(x5, w5), C.conv3d_dgrad(dy5, w5), C.conv3d_wgrad(x5, dy5))
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out[0], ref[0]) and torch.equal(out[1], ref[1])
    assert_close(out[2], ref[2], 1e-5, "dW")
