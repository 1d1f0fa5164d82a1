"""3x3x3 weight gradient (smb_conv3d_wgrad) against an fp64 sum over the 27 taps of the same 16-bit operands, at shapes that
stress its geometry: nine taps of one kd per work item, K blocks of one 8 x 8 x 1 brick, one dY box
per kw shared by the three kh taps, C_in tiles of at most 64 channels, and the K range split over the SMs."""
import pytest
import torch
import torch.nn.functional as F

from util import assert_close

pytestmark = pytest.mark.gpu

# (batch, C_in, C_out, D, H, W)
SHAPES = [
    (2, 48, 48, 5, 12, 7),       # W smaller than the brick
    (1, 16, 40, 4, 8, 12),       # W < 16, not a multiple of 8
    (2, 32, 48, 3, 8, 16),       # a 32-channel C_in tile
    (1, 48, 48, 3, 8, 20),       # W not a multiple of 16 or 8
    (2, 40, 16, 4, 9, 32),       # H not a multiple of 8
    (1, 96, 48, 3, 13, 16),      # H ragged, two 48-channel C_in tiles
    (2, 48, 96, 1, 16, 16),      # D = 1
    (1, 192, 16, 2, 8, 16),      # three 64-channel C_in tiles
    (1, 16, 192, 2, 8, 16),      # three 64-channel C_out blocks
    (1, 96, 96, 3, 10, 18),
    (1, 40, 192, 2, 9, 17),
    # 127 bricks, a prime: a split of the K range into 2..126 slices cannot make them equal, so the last one is short.  The
    # launcher splits this shape's 3 work items whenever the GPU has 6 SMs or more.
    (1, 48, 48, 127, 8, 8),
    (1, 96, 48, 61, 8, 16),
]


def _inputs(b, ci, co, d, h, w, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(b, d, h, w, ci, device="cuda", generator=g).to(dtype)
    dy = torch.randn(b, d, h, w, co, device="cuda", generator=g).to(dtype)
    return x, dy


def _reference(x5, dy5):
    """dW (C_out, 3, 3, 3, C_in) in fp64: dW[tap] = sum_v dY(v) . X(v + tap - 1), X zero-padded"""
    _, D, H, W, ci = x5.shape
    co = dy5.shape[4]
    xp = F.pad(x5.double(), (0, 0, 1, 1, 1, 1, 1, 1))
    dy = dy5.double()
    dw = torch.empty(co, 3, 3, 3, ci, dtype=torch.float64, device=x5.device)
    for kd in range(3):
        for kh in range(3):
            for kw in range(3):
                dw[:, kd, kh, kw] = torch.einsum("ndhwo,ndhwi->oi", dy, xp[:, kd:kd + D, kh:kh + H, kw:kw + W])
    return dw


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "f16"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "b%d_%dto%d_%dx%dx%d" % s)
def test_wgrad_matches_fp64(dtype, shape):
    from segmamba_b200 import conv3d as C
    x5, dy5 = _inputs(*shape, dtype, seed=sum(shape))
    dw = C.conv3d_wgrad(x5, dy5)
    assert dw.dtype == torch.float32 and dw.shape == (shape[2], 3, 3, 3, shape[1])
    assert_close(dw, _reference(x5, dy5), 1e-3, "dW")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "f16"])
@pytest.mark.parametrize("big", ["x", "dy"])
def test_wgrad_batch_boundary(dtype, big):
    """batch 3: sample 1 holds large values in one operand and zeros in the other, so its true contribution is zero and any
    pairing across a sample boundary (a d shift that reads the neighbouring sample) would dominate dW"""
    from segmamba_b200 import conv3d as C
    x5, dy5 = _inputs(3, 48, 48, 4, 10, 20, dtype, seed=7)
    scale = 1000.0 if dtype == torch.bfloat16 else 100.0
    if big == "x":
        x5[1] = (x5[1].float() * scale).to(dtype)
        dy5[1] = 0
    else:
        dy5[1] = (dy5[1].float() * scale).to(dtype)
        x5[1] = 0
    assert_close(C.conv3d_wgrad(x5, dy5), _reference(x5, dy5), 1e-3, "dW")
