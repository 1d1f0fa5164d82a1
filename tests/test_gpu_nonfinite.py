"""Non-finite locality and poisoned memory (tests/nonfinite_checks.py) on the H100: the emulator's checks in all three dtypes
and at full model sizes (stage-0 scan, instance norm at 2 x 48 x 128^3), where the many-CTA Chan merge and the segment
carries run."""
import pytest
import torch

import nonfinite_checks as nf
from util import GRAD_TOL

pytestmark = pytest.mark.gpu

NAN, INF = nf.NAN, nf.INF
DTYPES = [torch.float32, torch.bfloat16, torch.float16]
IDS = ["f32", "bf16", "f16"]


@pytest.fixture
def poison():
    """poisoned torch.empty / torch.empty_like (checked to poison before it is used)"""
    nf.check_poison_works("cuda")
    return nf.poisoned


def test_poison_fixture(poison):
    with poison():
        assert bool(torch.empty(1 << 20, device="cuda").isnan().all())


# ------------------------------------------------------------------------------------------------------- instance norm
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_instnorm_relu_propagates_nan(dtype):
    nf.relu_nan_semantics("cuda", dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("mode", ["plain", "add", "addnorm"])
@pytest.mark.parametrize("act", [None, "relu", "leaky_relu"])
def test_instnorm_locality(dtype, mode, act):
    C = 44 if dtype == torch.float32 else 48
    shape = (2, C, 9, 7, 5)
    x, add, dy = nf.in_inputs(shape, dtype, mode, "cuda", seed=1)
    sites = [("x", (0, 0, 0, 0, 0), NAN), ("x", (1, C - 1, 8, 6, 4), INF), ("x", (1, 0, 0, 0, 0), NAN),
             ("dy", (0, C - 5, 2, 1, 1), NAN)]
    if mode != "plain":
        sites.append(("add", (1, 7, 0, 0, 1), NAN))
    nf.in_locality(x, add, dy, act, mode, sites)


def test_instnorm_locality_full_size():
    x, add, dy = nf.in_inputs((2, 48, 128, 128, 128), torch.bfloat16, "add", "cuda", seed=2)
    nf.in_locality(x, add, dy, "relu", "add", [("x", (1, 47, 127, 127, 127), NAN), ("add", (0, 5, 64, 0, 3), NAN)],
                   use_rule=True)


@pytest.mark.parametrize("mode", ["plain", "add", "addnorm"])
def test_instnorm_fp16_headroom(mode):
    x, add, dy = nf.in_inputs((2, 48, 16, 16, 16), torch.float16, mode, "cuda", seed=7)
    lead = ("dx",) if mode == "plain" else ("dx", "dadd")
    top = max(float(nf.in_reference(x, add, dy, "relu", mode)[k].abs().max()) for k in lead)
    dy = (dy.float() * nf.headroom_scale(top)).half()
    got, ref = nf.in_run(x, add, dy, "relu", mode), nf.in_reference(x, add, dy, "relu", mode)
    nf.check_headroom({k: got[k] for k in lead}, {k: ref[k] for k in lead}, lead, 3e-2, f"[mode={mode}] ")


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_instnorm_poisoned(poison, dtype):
    for mode in ("plain", "add", "addnorm"):
        for shape in ((2, 48, 16, 16, 16), (1, 96, 9, 7, 5)):
            nf.in_poison(*nf.in_inputs(shape, dtype, mode, "cuda", seed=3), "leaky_relu", mode)


# ---------------------------------------------------------------------------------------------------------- layer norm
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("rows,C", [(4096, 48), (513, 192), (77, 384)], ids=lambda v: str(v))
def test_layernorm_locality(dtype, rows, C):
    x, w, b, dy = nf.ln_inputs(rows, C, dtype, "cuda", seed=4)
    sites = [("x", (0, 0), NAN), ("x", (rows - 1, C - 1), INF), ("dy", (rows // 2, C - 1), NAN), ("dy", (0, 7), NAN)]
    nf.ln_locality(x, w, b, dy, sites)
    nf.ln_locality(x, w, b, dy, [("x", (rows - 2, 3), NAN), ("dy", (1, C - 2), NAN)], use_rule=True)


def test_layernorm_locality_full_size():
    x, w, b, dy = nf.ln_inputs(524288, 48, torch.bfloat16, "cuda", seed=8)         # stage-0 tokens x 48 channels
    nf.ln_locality(x, w, b, dy, [("x", (524287, 47), NAN), ("dy", (262144, 0), INF), ("x", (0, 0), NAN)], use_rule=True)


def test_layernorm_fp16_headroom():
    x, w, b, dy = nf.ln_inputs(4096, 96, torch.float16, "cuda", seed=9)
    top = float(nf.ln_reference(x, w, b, dy)["dx"].abs().max())
    dy = (dy.float() * nf.headroom_scale(top)).half()
    nf.check_headroom(nf.ln_run(x, w, b, dy), nf.ln_reference(x, w, b, dy), ("dx",), 2e-2, "")


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_layernorm_poisoned(poison, dtype):
    nf.ln_poison(*nf.ln_inputs(65536, 96, dtype, "cuda", seed=5))
    nf.ln_poison(*nf.ln_inputs(333, 384, dtype, "cuda", seed=6))


# ------------------------------------------------------------------------------------------------------ selective scan
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("low_memory", [True, False], ids=["low_mem", "stash"])
@pytest.mark.parametrize("direction", [0, 1], ids=["fwd", "rev"])
def test_scan_locality_hbl(dtype, direction, low_memory):
    d = nf.scan_inputs(21, 2, 40, 2300, 16, 1, dtype, "cuda")
    sites = [("u", (0, 39, 2299), NAN), ("u", (1, 39, 0), NAN), ("B", (1, 0, 3, 32), NAN), ("C", (0, 0, 15, 255), NAN),
             ("z", (1, 8, 256), INF), ("dout", (0, 17, 2047), NAN), ("dout", (1, 2, 2048), NAN), ("u", (0, 0, 31), NAN),
             ("delta", (0, 5, 101), NAN), ("delta", (1, 33, 1029), NAN), ("dout", (1, 7, 0 if direction == 0 else 2299), NAN)]
    nf.scan_locality(d, sites, direction, low_memory, hbl=True)


@pytest.mark.parametrize("hbl", [False, True], ids=["contig", "hbl"])
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_scan_poisoned(poison, dtype, hbl):
    d = nf.scan_inputs(23, 2, 96, 5000, 16, 1, dtype, "cuda")
    for direction in (0, 1):
        for low in (True, False):
            nf.scan_poison(d, direction, low, hbl)


def test_scan_locality_full_size_stage0():
    """D = 96, L = 262144 (segment carries, many chunks): a NaN in u / delta reaches out / out_z from its position to the end
    of the walk and the last state; a NaN in dout reaches the gradients the rule names; nothing else changes."""
    d = nf.scan_inputs(5, 1, 96, 262144, 16, 1, torch.bfloat16, "cuda")
    for direction in (0, 1):
        nf.scan_locality(d, [("u", (0, 95, 131071), NAN), ("delta", (0, 32, 2053), NAN)], direction, True, hbl=False,
                         expect_fn=lambda e, site: nf.scan_fwd_rule(e, site, direction))
        for low in (True, False):
            nf.scan_locality(d, [("dout", (0, 40, 200001), NAN)], direction, low, hbl=False,
                             expect_fn=lambda e, site: nf.scan_bwd_rule(e, site, direction))


@pytest.mark.parametrize("low_memory", [True, False], ids=["low_mem", "stash"])
def test_scan_fp16_headroom(low_memory):
    d = nf.scan_inputs(41, 2, 40, 2300, 16, 1, torch.float16, "cuda")
    lead = ("du", "ddelta", "dz")
    grads = lead + ("dA", "dB", "dC", "dD", "ddelta_bias")
    top = max(float(nf.scan_reference(d, 0)[k].abs().max()) for k in lead)
    d["dout"] = (d["dout"].float() * nf.headroom_scale(top)).half()
    for direction in (0, 1):
        got, _ = nf.scan_run(d, direction, low_memory, hbl=True)
        ref = nf.scan_reference(d, direction)
        nf.check_headroom({k: got[k] for k in grads}, {k: ref[k] for k in grads}, lead, GRAD_TOL[torch.float16],
                          f"[dir={direction}] ")


# -------------------------------------------------------------------------------------------------- conv1d and permute
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("direction", [0, 1], ids=["fwd", "rev"])
def test_conv1d_locality_hbl(dtype, direction):
    import golden_inputs as gi
    g = gi.conv_inputs(31, 2, 40, 1300, 4)
    x, dout = g["x"].to(dtype).cuda(), g["dout"].to(dtype).cuda()
    w, b = g["weight"].cuda(), g["bias"].cuda()
    first, last = (0, 1299) if direction == 0 else (1299, 0)
    sites = [("x", (0, 39, last), NAN), ("x", (1, 39, first), NAN), ("dout", (1, 0, last), INF), ("x", (0, 12, 1023), NAN),
             ("dout", (1, 20, 1024), NAN), ("dout", (0, 3, 150), NAN)]
    nf.conv_locality(x, w, b, dout, sites, direction, hbl=True)
    nf.conv_locality(x, w, b, dout, [("dout", (0, 30, 150), NAN), ("x", (1, 1, 200), NAN)], direction, hbl=False, use_rule=True)


def test_conv1d_locality_full_size():
    import golden_inputs as gi
    g = gi.conv_inputs(35, 2, 96, 4096, 4)
    x = g["x"].repeat(1, 1, 64).bfloat16().cuda()                      # (2, 96, 262144), stage 0
    dout = g["dout"].repeat(1, 1, 64).bfloat16().cuda()
    for direction in (0, 1):
        sites = [("x", (1, 95, 131072), NAN), ("dout", (0, 0, 262143), NAN), ("dout", (1, 50, 0), INF)]
        nf.conv_locality(x, g["weight"].cuda(), g["bias"].cuda(), dout, sites, direction, hbl=True, use_rule=True)


def test_conv1d_fp16_headroom():
    import golden_inputs as gi
    g = gi.conv_inputs(36, 2, 96, 4100, 4)
    x, w, b = g["x"].half().cuda(), g["weight"].cuda(), g["bias"].cuda()
    top = float(nf.conv_reference(x, w, b, g["dout"], 0)["dx"].abs().max())
    dout = (g["dout"] * nf.headroom_scale(top)).half().cuda()
    for direction in (0, 1):
        got, _ = nf.conv_run(x, w, b, dout, direction, hbl=True)
        ref = nf.conv_reference(x, w, b, dout, direction)
        nf.check_headroom({k: got[k] for k in ("dx", "dweight", "dbias")}, {k: ref[k] for k in ("dx", "dweight", "dbias")},
                          ("dx",), GRAD_TOL[torch.float16], f"[dir={direction}] ")


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("hbl", [False, True], ids=["contig", "hbl"])
def test_conv1d_poisoned(poison, dtype, hbl):
    import golden_inputs as gi
    g = gi.conv_inputs(32, 2, 96, 4100, 4)
    for direction in (0, 1):
        nf.conv_poison(g["x"].to(dtype).cuda(), g["weight"].cuda(), g["bias"].cuda(), g["dout"].to(dtype).cuda(), direction, hbl)


def test_seq_permute_poisoned(poison):
    nf.permute_poison(torch.randn(2, 192, 4096, device="cuda").bfloat16(), 64)
    nf.permute_poison(torch.randn(192, 2, 512, device="cuda").permute(1, 0, 2), 8)


# ------------------------------------------------------------------------------------------------------------------- GEMM
EPIS = ["none", "bias_n", "bias_n_gelu", "bias_m"]


def _epi(name):
    from segmamba_b200 import gemm as G
    return {"none": G.EPI_NONE, "bias_n": G.EPI_BIAS_N, "bias_n_gelu": G.EPI_BIAS_N_GELU, "bias_m": G.EPI_BIAS_M}[name]


def _gemm_case(M, N, K, am, bm, epi, dtype=torch.bfloat16):
    a, b = nf.gemm_operand(M, K, am, dtype, 1), nf.gemm_operand(N, K, bm, dtype, 2)
    bias = None
    if epi != "none":
        g = torch.Generator(device="cpu").manual_seed(3)
        bias = torch.randn(M if epi == "bias_m" else N, generator=g).cuda()
    return a, b, bias


@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("am,bm", [("k", "k"), ("k", "mn"), ("mn", "k"), ("mn", "mn")])
def test_gemm_locality(am, bm, epi):
    """rows 127 / 128 (M tile), columns 63 / 64 / 127 / 128 (N tiles), first and last rows / columns / K"""
    M, N, K = 264, 200, 136
    a, b, bias = _gemm_case(M, N, K, am, bm, epi)
    sites = [("a", (0, 0), NAN), ("a", (127, 5), NAN), ("a", (128, K - 1), INF), ("a", (M - 1, 64), NAN),
             ("b", (0, K - 1), NAN), ("b", (63, 7), NAN), ("b", (64, 0), INF), ("b", (127, 70), NAN), ("b", (128, 3), NAN),
             ("b", (N - 1, 100), NAN)]
    if bias is not None:
        sites += [("bias", (0,), NAN), ("bias", (bias.shape[0] - 1,), NAN), ("bias", (128,), INF)]
    nf.gemm_locality(a, b, bias, _epi(epi), torch.float32 if epi != "none" else None, 1, sites)


@pytest.mark.parametrize("split", [1, 7])
def test_gemm_locality_model_shape(split):
    """weight-gradient shape (K = tokens split over CTAs, both operands MN-major, fp32 atomics) and the in_proj shape, by rule"""
    M, N, K = (192, 48, 65536) if split > 1 else (65536, 192, 48)
    am, bm = ("mn", "mn") if split > 1 else ("k", "k")
    a, b, _ = _gemm_case(M, N, K, am, bm, "none")
    sites = [("a", (M - 1, K - 1), NAN), ("a", (127, 0), NAN), ("b", (N - 1, K // 2), INF), ("b", (0, 1), NAN)]
    nf.gemm_locality(a, b, None, _epi("none"), torch.float32 if split > 1 else None, split, sites, use_rule=True)


@pytest.mark.parametrize("shape,split,am,bm", [((264, 200, 136), 1, "k", "k"), ((4096, 192, 96), 1, "k", "mn"),
                                              ((192, 48, 65536), 7, "mn", "mn"), ((96, 48, 70000), 148, "mn", "mn")],
                         ids=["ragged", "dgrad", "wgrad_split7", "wgrad_split148"])
@pytest.mark.parametrize("epi", ["none", "bias_n_gelu", "bias_m"])
def test_gemm_poisoned(poison, shape, split, am, bm, epi):
    if split > 1 and epi != "none":
        pytest.skip("split-K accumulates without an epilogue")
    M, N, K = shape
    a, b, bias = _gemm_case(M, N, K, am, bm, epi)
    nf.gemm_poison(a, b, bias, _epi(epi), torch.float32 if (split > 1 or epi != "none") else None, split)


@pytest.mark.parametrize("shape", [(65536, 192, 48), (8192, 768, 192)], ids=lambda s: "M%d_K%d_C%d" % s)
def test_gemm_fp16_headroom_dgrad(shape):
    """dx = dy . W at the mixer's dgrad shapes (W as an MN-major operand), fp16 output at a quarter of fp16's range"""
    M, K, C = shape
    dy, wt = nf.gemm_operand(M, K, "k", torch.float16, 4), nf.gemm_operand(C, K, "mn", torch.float16, 5)
    top = float(nf.gemm_reference(dy, wt, None, _epi("none"))["D"].abs().max())
    dy = (dy.float() * nf.headroom_scale(top)).half()
    nf.check_headroom(nf.gemm_run(dy, wt, None, _epi("none"), None, 1), nf.gemm_reference(dy, wt, None, _epi("none")),
                      ("D",), 1e-2, "")


# ----------------------------------------------------------------------------------------------------------------- conv3d
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "f16"])
@pytest.mark.parametrize("b,ci,co,d,h,w", [(2, 48, 48, 4, 9, 20), (1, 16, 96, 3, 17, 33)])
def test_conv3d_locality(dtype, b, ci, co, d, h, w):
    """fp64 zero-padded sum over the 27 taps; sites at the volume's corners, the 16 x 8 brick edges (w 15 / 16, h 7 / 8),
    the first voxel of sample 1 and the last channel"""
    x5, w5, dy5 = nf.conv3d_inputs(b, ci, co, d, h, w, dtype, seed=11)
    s1 = b - 1
    sites = [("x", (0, 0, 0, 0, 0), NAN), ("x", (s1, d - 1, h - 1, w - 1, ci - 1), NAN), ("x", (0, 1, 7, 15, 5), INF),
             ("x", (s1, 2, 8, 16, ci // 2), NAN), ("dy", (0, 0, 0, 0, co - 1), NAN), ("dy", (s1, d - 1, 7, 16, 3), NAN),
             ("dy", (0, 1, 7, 15, 0), INF)]
    if b > 1:
        sites.append(("x", (1, 0, 0, 0, 0), NAN))
    nf.conv3d_locality(x5, w5, dy5, sites)


@pytest.mark.xfail(strict=True, reason=(
    "known bug, off the routed shapes: where the volume is not a whole number of 64-voxel wgrad bricks, the brick tail pairs "
    "zero-filled x with in-volume dY, so a non-finite dY on the last row reaches weight taps that read no input"))
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "f16"])
def test_conv3d_wgrad_ragged_edge_locality(dtype):
    x5, w5, dy5 = nf.conv3d_inputs(2, 48, 48, 4, 9, 20, dtype, seed=11)
    nf.conv3d_locality(x5, w5, dy5, [("dy", (0, 1, 8, 15, 0), INF)])


def test_conv3d_locality_model_shape():
    x5, w5, dy5 = nf.conv3d_inputs(2, 48, 48, 64, 64, 64, torch.bfloat16, seed=12)
    sites = [("x", (1, 63, 63, 63, 47), NAN), ("x", (0, 32, 7, 15, 0), NAN), ("dy", (1, 0, 0, 0, 47), NAN),
             ("dy", (0, 40, 8, 16, 20), INF)]
    nf.conv3d_locality(x5, w5, dy5, sites, use_rule=True)


@pytest.mark.parametrize("b,ci,co,edge", [(2, 48, 48, 64), (2, 192, 96, 64), (1, 96, 192, 32), (2, 48, 48, 13)])
def test_conv3d_poisoned(poison, b, ci, co, edge):
    nf.conv3d_poison(*nf.conv3d_inputs(b, ci, co, edge, edge, edge, torch.bfloat16, seed=13))


def test_conv3d_fp16_headroom_dgrad():
    from segmamba_b200 import conv3d as C3
    x5, w5, dy5 = nf.conv3d_inputs(2, 48, 48, 16, 16, 64, torch.float16, seed=14)
    top = float(nf.conv3d_reference(x5, w5, dy5)["dx"].abs().max())
    dy5 = (dy5.float() * nf.headroom_scale(top)).half()
    ref = nf.conv3d_reference(x5, w5, dy5)
    nf.check_headroom({"dx": C3.conv3d_dgrad(dy5, w5)}, {"dx": ref["dx"]}, ("dx",), 1e-2, "")
