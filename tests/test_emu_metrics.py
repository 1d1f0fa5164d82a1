"""The metric kernels (csrc/metrics.cu) on the CPU SIMT emulator against the oracle, at ragged shapes."""
import pytest

from emu import emulated
from metrics_checks import check_labels_and_logits


@pytest.fixture(scope="module")
def emu():
    with emulated():
        yield "cpu"


@pytest.mark.parametrize("shape", [(13, 17, 19), (1, 9, 7), (5, 1, 1)])
def test_emu_metrics(emu, shape):
    r = check_labels_and_logits(shape, emu)
    for s in ((1.0, 1.0, 1.0), (2.5, 0.9, 0.9)):
        assert r[s]["dice_exact"], r
        assert r[s]["hd_err"] <= 1e-12 and r[s]["hd100_err"] <= 1e-12, r
    assert r[(1.0, 1.0, 1.0)]["hd_exact"] and r[(1.0, 1.0, 1.0)]["hd100_exact"], r
    assert all(r["logits"].values()), r["logits"]
