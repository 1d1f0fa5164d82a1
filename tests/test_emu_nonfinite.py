"""Non-finite locality and poisoned memory (tests/nonfinite_checks.py) for the kernels the CPU SIMT emulator runs: selective
scan, causal conv1d, sequence permute, instance norm and layer norm, at small sizes against the fp64 oracle / torch.
The `-m gpu` twin is tests/test_gpu_nonfinite.py."""
import pytest
import torch

import emu
import nonfinite_checks as nf

NAN, INF = nf.NAN, nf.INF


@pytest.fixture(autouse=True)
def _emulated():
    with emu.emulated():
        emu.emu_lib().smb_emu_set_reverse(0)
        yield


@pytest.fixture
def poison():
    """poisoned torch.empty / torch.empty_like (checked to poison before it is used)"""
    nf.check_poison_works("cpu")
    return nf.poisoned


def test_emu_poison_fixture(poison):
    with poison():
        assert bool(torch.empty(7, 3).isnan().all())
    assert torch.empty is nf.TORCH_EMPTY and torch.empty_like is nf.TORCH_EMPTY_LIKE        # restored


# ------------------------------------------------------------------------------------------------------- instance norm
def test_emu_instnorm_relu_propagates_nan():
    nf.relu_nan_semantics("cpu")


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
@pytest.mark.parametrize("mode", ["plain", "add", "addnorm"])
@pytest.mark.parametrize("act", [None, "relu", "leaky_relu"])
def test_emu_instnorm_locality(dtype, mode, act):
    C = 44 if dtype == torch.float32 else 48                    # a partial 8-channel group / a partial 64-channel box
    shape = (2, C, 5, 4, 3)
    x, add, dy = nf.in_inputs(shape, dtype, mode, "cpu", seed=1)
    sites = [("x", (0, 0, 0, 0, 0), NAN), ("x", (1, C - 1, 4, 3, 2), INF), ("x", (1, 0, 0, 0, 0), NAN),
             ("dy", (0, C - 5, 2, 1, 1), NAN)]
    if mode != "plain":
        sites.append(("add", (1, 7, 0, 0, 1), NAN))
    nf.in_locality(x, add, dy, act, mode, sites)


def test_emu_instnorm_locality_rule():
    shape = (2, 48, 6, 6, 6)
    for mode in ("plain", "add", "addnorm"):
        x, add, dy = nf.in_inputs(shape, torch.float32, mode, "cpu", seed=2)
        sites = [("x", (1, 47, 5, 5, 5), NAN)] + ([("add", (0, 9, 3, 0, 2), NAN)] if mode == "add" else [])
        nf.in_locality(x, add, dy, "relu", mode, sites, use_rule=True)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
def test_emu_instnorm_poisoned_workspace(poison, dtype):
    for mode in ("plain", "add", "addnorm"):
        x, add, dy = nf.in_inputs((2, 48, 7, 5, 3), dtype, mode, "cpu", seed=3)
        nf.in_poison(x, add, dy, "leaky_relu", mode)


# ---------------------------------------------------------------------------------------------------------- layer norm
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
@pytest.mark.parametrize("rows,C", [(300, 48), (70, 384)], ids=lambda v: str(v))
def test_emu_layernorm_locality(dtype, rows, C):
    x, w, b, dy = nf.ln_inputs(rows, C, dtype, "cpu", seed=4)
    sites = [("x", (0, 0), NAN), ("x", (rows - 1, C - 1), INF), ("dy", (rows // 2, C - 1), NAN), ("dy", (0, 7), NAN)]
    nf.ln_locality(x, w, b, dy, sites)
    nf.ln_locality(x, w, b, dy, [("x", (rows - 2, 3), NAN), ("dy", (1, C - 2), NAN)], use_rule=True)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
def test_emu_layernorm_poisoned(poison, dtype):
    nf.ln_poison(*nf.ln_inputs(513, 96, dtype, "cpu", seed=5))


# ------------------------------------------------------------------------------------------------------ selective scan
@pytest.mark.parametrize("low_memory", [True, False], ids=["low_mem", "stash"])
@pytest.mark.parametrize("direction", [0, 1], ids=["fwd", "rev"])
def test_emu_scan_locality_hbl(direction, low_memory):
    """mixer layout: the row after (b, d) in memory is (b + 1, d), so a tail read past L of row (0, d) meets sample 1."""
    d = nf.scan_inputs(21, 2, 40, 300, 16, 1, torch.float32, "cpu")
    sites = [("u", (0, 39, 299), NAN), ("u", (1, 39, 0), NAN), ("B", (1, 0, 3, 32), NAN), ("C", (0, 0, 15, 255), NAN),
             ("z", (1, 8, 256), INF), ("dout", (0, 17, 0), NAN), ("dout", (1, 2, 299), NAN)]
    nf.scan_locality(d, sites, direction, low_memory, hbl=True)


@pytest.mark.parametrize("low_memory", [True, False], ids=["low_mem", "stash"])
@pytest.mark.parametrize("direction", [0, 1], ids=["fwd", "rev"])
def test_emu_scan_delta_locality_inside_run(direction, low_memory):
    """delta at a position that is not the last of its 8-position run in walk order: the later positions of the run take
    the adjoint entering from the right, whose decay must not include the run's own (non-finite) dt"""
    d = nf.scan_inputs(24, 2, 40, 300, 16, 1, torch.float32, "cpu")
    nf.scan_locality(d, [("delta", (0, 5, 101), NAN)], direction, low_memory, hbl=True)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "f16"])
def test_emu_scan_locality_groups(dtype):
    d = nf.scan_inputs(22, 1, 48, 257, 8, 2, dtype, "cpu")
    sites = [("B", (0, 1, 7, 256), NAN), ("u", (0, 47, 128), NAN), ("dout", (0, 24, 256), NAN)]
    for direction in (0, 1):
        nf.scan_locality(d, sites, direction, True, hbl=False)


@pytest.mark.parametrize("hbl", [False, True], ids=["contig", "hbl"])
def test_emu_scan_poisoned(poison, hbl):
    d = nf.scan_inputs(23, 2, 40, 600, 16, 1, torch.bfloat16, "cpu")
    for direction in (0, 1):
        for low in (True, False):
            nf.scan_poison(d, direction, low, hbl)


# -------------------------------------------------------------------------------------------------- conv1d and permute
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
@pytest.mark.parametrize("direction", [0, 1], ids=["fwd", "rev"])
def test_emu_conv1d_locality_hbl(dtype, direction):
    import golden_inputs as gi
    g = gi.conv_inputs(31, 2, 40, 300, 4)
    x, dout = g["x"].to(dtype), g["dout"].to(dtype)
    first, last = (0, 299) if direction == 0 else (299, 0)      # first / last position of the walk
    sites = [("x", (0, 39, last), NAN), ("x", (1, 39, first), NAN), ("dout", (1, 0, last), INF), ("x", (0, 12, 127), NAN),
             ("dout", (1, 20, 128), NAN), ("dout", (0, 3, 150), NAN)]
    nf.conv_locality(x, g["weight"], g["bias"], dout, sites, direction, hbl=True)
    nf.conv_locality(x, g["weight"], g["bias"], dout, [("dout", (0, 30, 150), NAN), ("x", (1, 1, 200), NAN)], direction,
                     hbl=False, use_rule=True)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])     # 8 / 16 positions per thread
@pytest.mark.parametrize("direction", [0, 1], ids=["fwd", "rev"])
def test_emu_conv1d_dweight_padding_locality(dtype, direction):
    """a non-finite dout at the first position of the walk reaches only the weight taps that read input, not the ones over
    the zero padding before it"""
    import golden_inputs as gi
    g = gi.conv_inputs(33, 2, 40, 300, 4)
    first = 0 if direction == 0 else 299
    nf.conv_locality(g["x"].to(dtype), g["weight"], g["bias"], g["dout"].to(dtype),
                     [("dout", (0, 3, first), NAN), ("dout", (1, 39, first), INF)], direction, hbl=True)


@pytest.mark.parametrize("hbl", [False, True], ids=["contig", "hbl"])
def test_emu_conv1d_poisoned(poison, hbl):
    import golden_inputs as gi
    g = gi.conv_inputs(32, 2, 40, 700, 4)
    for direction in (0, 1):
        nf.conv_poison(g["x"].bfloat16(), g["weight"], g["bias"], g["dout"].bfloat16(), direction, hbl)


def test_emu_seq_permute_poisoned(poison):
    nf.permute_poison(torch.randn(2, 12, 512).bfloat16(), 16)
    nf.permute_poison(torch.randn(12, 2, 96).permute(1, 0, 2), 8)
