"""Tensor-core GEMM (smb_gemm: TMA + wgmma) against a plain fp32 torch product of the same 16-bit
operands, at the shapes of the model's pointwise contractions (SURVEY.md section 8d) and at ragged ones; every operand-major
combination, every epilogue, split-K accumulation, and the autograd wrapper ``gemm.linear`` against F.linear."""
import pytest
import torch

from util import assert_close

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True, params=["all", "auto"])
def _gemm_mode(request, monkeypatch):
    """every autograd-level test runs with all products on the native kernel and with the default routing (token-axis
    contractions native, the rest library); the raw gemm() tests do not depend on it."""
    from segmamba_b200 import gemm as G
    monkeypatch.setattr(G, "MODE", request.param)
    yield


def _mk(rows, cols, major, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if major == "k":
        return (torch.randn(rows, cols, device="cuda", generator=g) / cols ** 0.25).to(dtype)
    return (torch.randn(cols, rows, device="cuda", generator=g) / cols ** 0.25).to(dtype).t()     # MN-major view


SHAPES = [(524288, 192, 48), (65536, 384, 96), (8192, 768, 192), (1024, 1536, 384), (524288, 48, 96), (1024, 384, 768),
          (300, 40, 72), (129, 16, 8), (4096, 96, 200), (77, 264, 1000)]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "f16"])
@pytest.mark.parametrize("am,bm", [("k", "k"), ("k", "mn"), ("mn", "k"), ("mn", "mn")])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "M%d_N%d_K%d" % s)
def test_gemm_vs_fp32(dtype, am, bm, shape):
    from segmamba_b200 import gemm as G
    M, N, K = shape
    if dtype == torch.float16 and M > 100000:
        pytest.skip("large shapes: bf16 only")
    for t, ext in (("mn" == am, M), ("mn" == bm, N)):
        if t and ext % 8:
            pytest.skip("MN-major operand needs a 16-byte aligned contiguous extent")
    if (am == "k" or bm == "k") and K % 8:
        pytest.skip("K-major operand needs K % 8 == 0")
    a, b = _mk(M, K, am, dtype, 1), _mk(N, K, bm, dtype, 2)
    d = G.gemm(a, b)
    ref = a.float() @ b.float().t()
    assert d.shape == (M, N) and d.dtype == dtype
    assert_close(d, ref, 1e-2, "D")
    d32 = G.gemm(a, b, out_dtype=torch.float32)
    assert_close(d32, ref, 2e-5 if K <= 1024 else 1e-4, "D fp32")     # fp32 accumulation of exact 16-bit products


@pytest.mark.parametrize("epi", ["bias_n", "bias_n_gelu", "bias_m"])
@pytest.mark.parametrize("shape", [(65536, 96, 48), (1000, 200, 136), (4096, 768, 384)], ids=lambda s: "M%d_N%d_K%d" % s)
def test_gemm_epilogues(epi, shape):
    from segmamba_b200 import gemm as G
    M, N, K = shape
    a, b = _mk(M, K, "k", torch.bfloat16, 3), _mk(N, K, "k", torch.bfloat16, 4)
    ref = a.float() @ b.float().t()
    if epi == "bias_m":
        bias = torch.randn(M, device="cuda")
        d = G.gemm(a, b, bias, G.EPI_BIAS_M, out_dtype=torch.float32)
        ref = ref + bias[:, None]
    else:
        bias = torch.randn(N, device="cuda")
        d = G.gemm(a, b, bias, G.EPI_BIAS_N_GELU if epi == "bias_n_gelu" else G.EPI_BIAS_N, out_dtype=torch.float32)
        ref = ref + bias[None]
        if epi == "bias_n_gelu":
            ref = torch.nn.functional.gelu(ref)
    assert_close(d, ref, 1e-4, epi)


@pytest.mark.parametrize("split", [2, 7, 148])
def test_gemm_split_k_accumulates(split):
    """weight-gradient shape: K = tokens, both operands MN-major, fp32 atomics into a zero-initialised D."""
    from segmamba_b200 import gemm as G
    tokens, n_out, c_in = 70000, 96, 48
    dy, x = _mk(n_out, tokens, "mn", torch.bfloat16, 5), _mk(c_in, tokens, "mn", torch.bfloat16, 6)
    d = G.gemm(dy, x, out_dtype=torch.float32, split_k=split)
    ref = dy.float() @ x.float().t()
    assert_close(d, ref, 1e-4, "dW")
    d2 = G.gemm(dy, x, out_dtype=torch.float32, out=d.clone(), accumulate=True)
    assert_close(d2, 2 * ref, 1e-4, "accumulate")


@pytest.mark.parametrize("gelu", [False, True], ids=["plain", "gelu"])
@pytest.mark.parametrize("shape", [(2, 4096, 48, 96), (1, 333, 192, 384), (2, 512, 384, 48)], ids=lambda s: "b%d_l%d_c%d_n%d" % s)
def test_linear_autograd_vs_torch(gelu, shape):
    from segmamba_b200 import gemm as G
    Bz, L, C, N = shape
    torch.manual_seed(0)
    x = torch.randn(Bz, L, C, device="cuda").bfloat16().requires_grad_()
    w = (torch.randn(N, C, device="cuda") / C ** 0.5).requires_grad_()
    b = torch.randn(N, device="cuda").requires_grad_()
    dy = torch.randn(Bz, L, N, device="cuda").bfloat16()
    y = G.linear(x, w, b, gelu=gelu, compute_dtype=torch.bfloat16)
    gx, gw, gb = torch.autograd.grad(y, [x, w, b], dy)
    xr = x.detach().float().requires_grad_()
    wr = w.detach().bfloat16().float().requires_grad_()
    br = b.detach().clone().requires_grad_()
    yr = torch.nn.functional.linear(xr, wr, br)
    if gelu:
        yr = torch.nn.functional.gelu(yr)
    rx, rw, rb = torch.autograd.grad(yr, [xr, wr, br], dy.float())
    assert_close(y, yr, 1e-2, "y")
    assert_close(gx, rx, 2e-2, "dx")
    assert_close(gw, rw, 2e-2, "dW")
    assert_close(gb, rb, 2e-2, "db")


def test_matmul_nt_autograd_transposed_output():
    """in_proj form: xz[2 d_inner, B L] = W[2 d_inner, C] @ X[B L, C]^T with gradients for both (mamba_simple.py:204-208)."""
    from segmamba_b200 import gemm as G
    torch.manual_seed(1)
    W = (torch.randn(192, 48, device="cuda") / 7).requires_grad_()
    X = torch.randn(2 * 20000, 48, device="cuda").bfloat16().requires_grad_()
    dD = torch.randn(192, 2 * 20000, device="cuda").bfloat16()
    D = G.matmul_nt(W, X, compute_dtype=torch.bfloat16)
    gW, gX = torch.autograd.grad(D, [W, X], dD)
    Wr, Xr = W.detach().bfloat16().float().requires_grad_(), X.detach().float().requires_grad_()
    Dr = Wr @ Xr.t()
    rW, rX = torch.autograd.grad(Dr, [Wr, Xr], dD.float())
    assert_close(D, Dr, 1e-2, "xz")
    assert_close(gW, rW, 2e-2, "dW")
    assert_close(gX, rX, 2e-2, "dX")


def test_conv1x1_vs_conv3d():
    from segmamba_b200 import gemm as G
    torch.manual_seed(2)
    conv = torch.nn.Conv3d(48, 96, 1).cuda()
    x = torch.randn(2, 48, 16, 12, 20, device="cuda").bfloat16().contiguous(memory_format=torch.channels_last_3d).requires_grad_()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        y = G.conv1x1(x, conv.weight, conv.bias)
        yr = conv(x)
    assert y.shape == yr.shape
    assert_close(y, yr.float(), 1e-2, "conv1x1")
    dy = torch.randn_like(yr)
    g = torch.autograd.grad(y, [x, conv.weight, conv.bias], dy)
    gr = torch.autograd.grad(yr, [x, conv.weight, conv.bias], dy)
    for a, b, n in zip(g, gr, ("dx", "dW", "db")):
        assert_close(a, b.float(), 3e-2, n)
