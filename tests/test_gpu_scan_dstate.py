"""The selective scan at 32 and 64 states on the H100: every forward and backward path against the fp64 oracle, the same inputs
through the reference's own CUDA extension (oracle/_ref), the Mamba v3 mixer and MambaLayer at d_state 32 / 64 against
oracle/oracle.py, non-finite locality at 64 states, and the state counts that stay unsupported."""
import importlib.util
import os

import numpy as np
import pytest
import torch

import golden_inputs as gi
import nonfinite_checks as nf
import test_gpu_scan as tg
from dstate_cases import DSTATE_CASES
from util import GRAD_TOL, TOL, assert_close, rand_scan_inputs

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
DT_IDS = ["f32", "f16", "bf16"]


@pytest.mark.parametrize("case", DSTATE_CASES, ids=lambda c: c[0])
def test_dstate_vs_golden_and_oracle(case):
    """the reference's selective_scan_ref (golden) and the oracle, fp32, with and without the saved states."""
    name, seed, batch, dim, L, N, G, tl, has_D, has_z, has_b, sp = case
    d = {k: v.cuda() for k, v in gi.scan_inputs(seed, batch, dim, L, N, G, tl).items()}
    ref = tg._oracle_fwd_bwd(d, has_D, has_z, has_b, sp)
    gold = gi.load("scan_" + name)
    for use_hstates in (True, False):
        res = tg._run_fwd_bwd(d, has_D, has_z, has_b, sp, use_hstates=use_hstates)
        tg._compare(res, ref, torch.float32, has_z)
        assert_close(res[2] if has_z else res[0], gold["out"], 1e-3, "out vs reference golden")
        assert_close(res[1][:, :, -1, 1::2], gold["last_state"], 1e-3, "last_state vs reference golden")
        for i, k in enumerate(["du", "ddelta", "dA", "dB", "dC", "dD", "ddelta_bias", "dz"]):
            if k in gold.files and res[5][i] is not None:
                got = res[5][i].squeeze(1) if res[5][i].dim() == 4 and gold[k].ndim == 3 else res[5][i]
                assert_close(got, gold[k], 2e-3, k + " vs reference golden")


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("shape", [(2, 96, 5000, 32, 1), (1, 40, 777, 32, 2), (2, 96, 5000, 64, 1), (1, 40, 777, 64, 2),
                                   (1, 33, 31, 64, 1)], ids=lambda s: "b%d_d%d_L%d_n%d_g%d" % s)
@pytest.mark.parametrize("direction", [0, 1], ids=["fwd", "rev"])
def test_dstate_random_vs_oracle(dtype, shape, direction):
    """forward, and the backward three ways: scan-free main pass on the dense checkpoints and the state-stash sweep (with the saved
    states), the recompute + Kogge-Stone main pass (without)."""
    batch, dim, L, N, G = shape
    d = rand_scan_inputs(100 + L + N, batch, dim, L, N, G, dtype)
    ref = tg._oracle_fwd_bwd(d, flip=bool(direction))
    for use_hstates in (True, False):
        tg._compare(tg._run_fwd_bwd(d, direction=direction, use_hstates=use_hstates), ref, dtype, True)


@pytest.mark.parametrize("N", [32, 64])
def test_dstate_first_generation_kernels(monkeypatch, N):
    """the first-generation forward / R1 / R3 kernels (the A/B switches) at the new sizes."""
    for k in ("SMB_FWD_V2", "SMB_RAGG_V2", "SMB_R3_V2"):
        monkeypatch.setenv(k, "0")
    d = rand_scan_inputs(31, 2, 48, 1500, N, 2, torch.bfloat16)
    ref = tg._oracle_fwd_bwd(d)
    for use_hstates in (True, False):
        tg._compare(tg._run_fwd_bwd(d, use_hstates=use_hstates), ref, torch.bfloat16, True)
    monkeypatch.setenv("SMB_FWD_V2", "1")                  # the cp.async forward
    tg._compare(tg._run_fwd_bwd(d, use_hstates=True), ref, torch.bfloat16, True)


@pytest.mark.parametrize("N", [32, 64])
def test_dstate_full_size_stage0(N):
    """stage-0 size (D=96, L=262144): forward parity on a channel subset, and the chunk states."""
    from segmamba_b200 import selective_scan_cuda as ssc
    batch, dim, L = 1, 96, 262144
    d = rand_scan_inputs(5, batch, dim, L, N, 1, torch.bfloat16)
    B, C = d["B"].unsqueeze(1), d["C"].unsqueeze(1)
    out, x, out_z, _ = ssc.fwd_ex(d["u"], d["delta"], d["A"], B, C, d["D"], d["z"], d["delta_bias"], True)
    sel = [0, 31, 32, 95]
    from oracle import oracle as orc
    f = lambda t: t.float().cpu()
    y, oz, last, xc = orc.selective_scan_fwd_raw(f(d["u"][:, sel]), f(d["delta"][:, sel]), f(d["A"][sel]), f(d["B"]), f(d["C"]),
                                                 f(d["D"][sel]), f(d["z"][:, sel]), f(d["delta_bias"][sel]), True)
    assert_close(out_z[:, sel], oz, 1e-2, "full-size out_z")
    assert_close(x[:, sel][..., 1::2], xc[..., 1::2], 1e-3, "full-size chunk states")


def _ref_ext():
    path = os.path.join(ROOT, "oracle", "_ref", "selective_scan_cuda.so")
    if not os.path.exists(path):
        pytest.skip("reference extension not built (oracle/build_ref.py)")
    spec = importlib.util.spec_from_file_location("selective_scan_cuda", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("N", [32, 64])
def test_dstate_vs_reference_cuda_extension(dtype, N):
    """the drop-in fwd / bwd against the reference's own kernels on the same inputs (ragged L over two 2048 chunks, 2 groups)."""
    from segmamba_b200 import selective_scan_cuda as ssc
    ref = _ref_ext()
    d = rand_scan_inputs(77 + N, 2, 64, 4100, N, 2, dtype)
    args = (d["u"], d["delta"], d["A"], d["B"], d["C"], d["D"], d["z"], d["delta_bias"], True)
    ro, mo = ref.fwd(*args), ssc.fwd(*args)
    tol, gtol = TOL[dtype], GRAD_TOL[dtype]
    assert_close(mo[2], ro[2], tol, "out_z")
    assert_close(mo[1][..., 1::2], ro[1][..., 1::2], tol, "x (chunk states)")
    rg = ref.bwd(*args[:8], d["dout"], ro[1], ro[0], None, True, False)
    mg = ssc.bwd(*args[:8], d["dout"], mo[1], mo[0], None, True, False)
    for i, k in enumerate(["du", "ddelta", "dA", "dB", "dC", "dD", "ddelta_bias", "dz"]):
        assert_close(mg[i], rg[i], gtol, k)


def _params(m):
    return {k: v.detach().float().cpu() for k, v in m.state_dict().items()}


@pytest.mark.parametrize("N", [32, 64])
def test_mamba_v3_dstate_vs_oracle(N):
    from oracle import oracle as orc
    from segmamba_b200.mamba_simple import Mamba
    torch.manual_seed(N)
    batch, d_model, L, ns = 2, 16, 512, 8
    m = Mamba(d_model=d_model, d_state=N, d_conv=4, expand=2, bimamba_type="v3", nslices=ns).cuda()
    r = np.random.RandomState(N)
    x = torch.from_numpy(r.standard_normal((batch, L, d_model)).astype(np.float32))
    dout = torch.from_numpy(r.standard_normal((batch, L, d_model)).astype(np.float32))
    xg = x.cuda().requires_grad_()
    out = m(xg)
    names = [n for n, _ in m.named_parameters()]
    grads = torch.autograd.grad(out, [xg] + [p for _, p in m.named_parameters()], dout.cuda())
    p = {k: v.requires_grad_() for k, v in _params(m).items()}
    xo = x.clone().requires_grad_()
    ro = orc.mamba_v3_forward(p, xo, ns)
    rgrads = torch.autograd.grad(ro, [xo] + [p[n] for n in names], dout)
    assert_close(out, ro, 1e-3, "out")
    assert_close(grads[0], rgrads[0], 2e-3, "dx")
    for n, g, rg in zip(names, grads[1:], rgrads[1:]):
        assert_close(g, rg, 3e-3, "grad." + n)


@pytest.mark.parametrize("N", [32, 64])
def test_mamba_layer_dstate_vs_oracle(N):
    """MambaLayer (LayerNorm + v3 mixer + residual) on a channels-first volume, forward and backward."""
    from oracle import oracle as orc
    from segmamba_b200.segmamba import MambaLayer
    torch.manual_seed(100 + N)
    B, C, S, ns = 1, 32, 8, 8
    layer = MambaLayer(dim=C, d_state=N, num_slices=ns).cuda()
    r = np.random.RandomState(N + 1)
    x = torch.from_numpy(r.standard_normal((B, C, S, S, S)).astype(np.float32))
    dout = torch.from_numpy(r.standard_normal((B, C, S, S, S)).astype(np.float32))
    xg = x.cuda().requires_grad_()
    out = layer(xg)
    (gx,) = torch.autograd.grad(out, [xg], dout.cuda())
    p = {k: v.requires_grad_() for k, v in _params(layer).items()}
    xo = x.clone().requires_grad_()
    xf = xo.reshape(B, C, -1).transpose(-1, -2)
    xn = torch.nn.functional.layer_norm(xf, (C,), p["norm.weight"], p["norm.bias"], layer.norm.eps)
    ro = orc.mamba_v3_forward(p, xn, ns, prefix="mamba.").transpose(-1, -2).reshape(x.shape) + xo
    (rgx,) = torch.autograd.grad(ro, [xo], dout)
    assert_close(out, ro, 1e-3, "out")
    assert_close(gx, rgx, 2e-3, "dx")


@pytest.mark.parametrize("direction", [0, 1], ids=["fwd", "rev"])
@pytest.mark.parametrize("low_memory", [True, False], ids=["low_memory", "stash"])
def test_dstate64_nonfinite_locality(direction, low_memory):
    """a NaN / Inf in one input makes non-finite exactly what the fp64 oracle makes non-finite, and no workspace or output element
    is read before it is written (poisoned allocations)."""
    d = nf.scan_inputs(3, 2, 40, 600, 64, 2, torch.bfloat16, "cuda")
    L = 600
    nan, inf = float("nan"), float("inf")
    sites = [("u", (1, 7, 300), nan), ("delta", (0, 33, 5), nan), ("B", (1, 0, 63, L - 1), nan), ("C", (0, 0, 40, 256), nan),
             ("z", (1, 0, 511), inf), ("dout", (0, 39, 100), nan)]
    nf.scan_locality(d, sites, direction, low_memory, hbl=False, tag=f"N64 dir{direction} low{int(low_memory)}")
    nf.scan_poison(d, direction, low_memory, hbl=False)


@pytest.mark.parametrize("N", [5, 24, 128])
def test_dstate_unsupported_raise(N):
    from segmamba_b200 import selective_scan_cuda as ssc
    d = rand_scan_inputs(1, 1, 8, 64, N)
    with pytest.raises(RuntimeError, match="8, 16, 32 or 64"):
        ssc.fwd(d["u"], d["delta"], d["A"], d["B"].unsqueeze(1), d["C"].unsqueeze(1), None, None, None, False)
