"""The case-prediction kernels (csrc/predict.cu) on the CPU SIMT emulator against the oracle, at ragged shapes."""
import pytest

from emu import emulated
from predict_checks import FAMILIES, check_cc, check_restore, family, logits_like


@pytest.fixture(scope="module")
def emu():
    with emulated():
        yield "cpu"


@pytest.mark.parametrize("shape", [(13, 17, 19), (1, 9, 7), (5, 1, 1), (1, 1, 1)])
@pytest.mark.parametrize("name", FAMILIES)
def test_emu_components(emu, shape, name):
    assert check_cc(family(name, shape), emu) == []


@pytest.mark.parametrize("shape,crop,lo,full", [
    ((9, 10, 11), (9, 10, 11), (1, 2, 3), (12, 14, 17)),                 # identity resample
    ((9, 10, 11), (12, 7, 16), (2, 0, 1), (15, 9, 18)),                  # up, down and up
    ((1, 9, 7), (3, 9, 5), (0, 0, 0), (3, 9, 5)),                        # box covers the whole volume
])
def test_emu_restore(emu, shape, crop, lo, full):
    r = check_restore(logits_like(shape, seed=4), crop, lo, full, emu)
    assert all(v == (0, 0) for v in r.values()), r
