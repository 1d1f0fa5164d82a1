"""The augmentation kernels (csrc/augment.cu) on the CPU SIMT emulator against the oracle, at a small ragged patch."""
import pytest

from aug_checks import check_blur_stats_pointwise, check_chain, check_prefilter, check_resample
from emu import emulated

SHAPE = (13, 17, 19)


@pytest.fixture(scope="module")
def emu():
    with emulated():
        yield "cpu"


def test_emu_prefilter(emu):
    e = check_prefilter(SHAPE, emu)
    assert e["mirror"] < 1e-4 and e["edge"] < 1e-4, e


def test_emu_resample(emu):
    e = check_resample(SHAPE, emu)
    assert e["order3"] < 1e-4 and e["up"] < 1e-4 and e["down"] == 0 and e["seg_mismatch"] == 0, e
    assert e["lowres"] < 1e-4, e


def test_emu_blur_stats_pointwise(emu):
    e = check_blur_stats_pointwise(SHAPE, emu)
    assert e["blur"] < 1e-5 and e["stats"] < 1e-6 and e["noise"] < 1e-6 and e["contrast"] < 1e-5 and e["gamma"] < 1e-5, e


def test_emu_whole_chain_forced(emu):
    r = check_chain(SHAPE, emu)
    assert r["crop_exact"] and r["chain"] < 1e-3 and r["seg_mismatch"] == 0, {k: v for k, v in r.items() if k not in ("image", "label")}
