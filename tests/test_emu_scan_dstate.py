"""The selective-scan kernels at 32 and 64 states, run without a GPU through tools/simt_emu (see tests/test_emu_kernels.py):
the forward and every backward path -- scan-free main pass on the dense checkpoints, recompute + Kogge-Stone main pass, the
state-stash sweep -- with both kernel generations where two exist, fp32 and bf16, both walk directions, against the oracle
with the tolerances of the parity tests.  Plus the C oracle against the reference's own golden vectors at these sizes."""
import numpy as np
import pytest
import torch

import emu
import golden_inputs as gi
import test_gpu_scan as tg
from dstate_cases import DSTATE_CASES
from util import assert_close, rand_scan_inputs


@pytest.fixture
def emulated():
    with emu.emulated():
        emu.emu_lib().smb_emu_set_reverse(0)
        yield


def _close(a, b, rtol, atol, what):
    a = torch.as_tensor(np.asarray(a)).double()
    b = torch.as_tensor(np.asarray(b)).double()
    assert a.shape == b.shape, f"{what}: shape {tuple(a.shape)} vs {tuple(b.shape)}"
    err = (a - b).abs()
    assert bool((err <= atol + rtol * b.abs()).all()), f"{what}: max err {err.max().item():.3e}"


@pytest.mark.parametrize("case", DSTATE_CASES, ids=lambda c: c[0])
def test_oracle_vs_reference_golden_dstate(case):
    """oracle/segmamba_oracle.c (fp64) against the reference's selective_scan_ref (fp32) at 32 / 64 states."""
    from oracle import oracle as orc
    name, seed, batch, dim, L, N, G, tl, has_D, has_z, has_b, sp = case
    d = gi.scan_inputs(seed, batch, dim, L, N, G, tl)
    gold = gi.load("scan_" + name)
    assert np.allclose(gold["input_checksum"], [float(d["u"].double().sum()), float(d["B"].double().sum())])
    D, z, bias = (d["D"] if has_D else None), (d["z"] if has_z else None), (d["delta_bias"] if has_b else None)
    y, oz, last, xc = orc.selective_scan_fwd_raw(d["u"], d["delta"], d["A"], d["B"], d["C"], D, z, bias, sp)
    out = oz if has_z else y
    _close(out, gold["out"], 2e-5, 2e-5 * float(np.abs(gold["out"]).max()), "out")
    _close(last, gold["last_state"], 2e-5, 2e-5 * float(np.abs(gold["last_state"]).max()), "last_state")
    g = orc.selective_scan_bwd_raw(d["u"], d["delta"], d["A"], d["B"], d["C"], D, z, bias, sp, d["dout"])
    for k in ("du", "ddelta", "dA", "dB", "dC", "dD", "dz", "ddelta_bias"):
        if k in gold.files:
            got = g[k].squeeze(1) if g[k].dim() == 4 and gold[k].ndim == 3 else g[k]
            _close(got, gold[k], 1e-4, 1e-4 * float(np.abs(gold[k]).max()), k)


@pytest.mark.parametrize("case", DSTATE_CASES[:4], ids=lambda c: c[0])
def test_emu_dstate_vs_golden_and_oracle(emulated, case):
    name, seed, batch, dim, L, N, G, tl, has_D, has_z, has_b, sp = case
    d = gi.scan_inputs(seed, batch, dim, L, N, G, tl)
    for use_hstates in (True, False):
        res = tg._run_fwd_bwd(d, has_D, has_z, has_b, sp, use_hstates=use_hstates)
        tg._compare(res, tg._oracle_fwd_bwd(d, has_D, has_z, has_b, sp), torch.float32, has_z)
    gold = gi.load("scan_" + name)
    assert_close(res[2] if has_z else res[0], gold["out"], 1e-3, "out vs reference golden")
    assert_close(res[1][:, :, -1, 1::2], gold["last_state"], 1e-3, "last_state vs reference golden")


# (env overrides) -> which kernel generation runs: default (TMA forward for 16-bit, pipelined R1, R3 v2), the cp.async forward,
# and the first-generation R1 / R3
VARIANTS = {"default": {}, "first_gen": {"SMB_FWD_V2": "0", "SMB_RAGG_V2": "0", "SMB_R3_V2": "0"}, "cp_async": {"SMB_FWD_V2": "1"}}


@pytest.mark.parametrize("variant,dtype", [("default", torch.float32), ("default", torch.bfloat16), ("first_gen", torch.float32),
                                           ("first_gen", torch.bfloat16), ("cp_async", torch.bfloat16)],
                         ids=["default-f32", "default-bf16", "first_gen-f32", "first_gen-bf16", "cp_async-bf16"])
@pytest.mark.parametrize("shape", [(1, 40, 300, 32, 1), (1, 36, 264, 64, 2)], ids=lambda s: "b%d_d%d_L%d_n%d_g%d" % s)
@pytest.mark.parametrize("direction", [0, 1], ids=["fwd", "rev"])
def test_emu_dstate_random_vs_oracle(emulated, monkeypatch, variant, dtype, shape, direction):
    """(the pipelined forward is for 16-bit activations only)"""
    for k, v in VARIANTS[variant].items():
        monkeypatch.setenv(k, v)
    batch, dim, L, N, G = shape
    d = rand_scan_inputs(100 + L, batch, dim, L, N, G, dtype, device="cpu")
    ref = tg._oracle_fwd_bwd(d, flip=bool(direction))
    for use_hstates in (True, False):
        res = tg._run_fwd_bwd(d, direction=direction, use_hstates=use_hstates)
        tg._compare(res, ref, dtype, True)


def test_emu_dstate_thread_orders(emulated):
    """64 states with the threads of every block resumed in descending / pseudo-random order (a missing barrier shows up)."""
    d = rand_scan_inputs(5, 1, 40, 300, 64, 1, torch.bfloat16, device="cpu")
    ref = tg._oracle_fwd_bwd(d)
    for order in (1, 3):
        emu.emu_lib().smb_emu_set_reverse(order)
        tg._compare(tg._run_fwd_bwd(d, use_hstates=True), ref, torch.bfloat16, True)
    emu.emu_lib().smb_emu_set_reverse(0)


@pytest.mark.parametrize("N", [5, 24, 128])
def test_emu_unsupported_dstate_raises(emulated, N):
    from segmamba_b200 import selective_scan_cuda as ssc
    d = rand_scan_inputs(1, 1, 8, 64, N, device="cpu")
    with pytest.raises(RuntimeError, match="8, 16, 32 or 64"):
        ssc.fwd(d["u"], d["delta"], d["A"], d["B"].unsqueeze(1), d["C"].unsqueeze(1), None, None, None, False)
