"""Per-class evaluation (csrc/metrics.cu class kernels, through metrics.class_metrics) on the CPU SIMT emulator against the
oracle and the reference fixture, at ragged shapes."""
import numpy as np
import pytest
import torch

from class_metrics_checks import compare, golden_cases, organ_labels, perturb_organs
from emu import emulated
from oracle import class_metrics_oracle as orc
from segmamba_b200 import metrics as M


@pytest.fixture(scope="module")
def emu():
    with emulated():
        yield "cpu"


@pytest.mark.parametrize("shape", [(13, 17, 19), (1, 9, 7), (5, 1, 1), (1, 1, 1)])
@pytest.mark.parametrize("spacing", [(1.0, 1.0, 1.0), (2.5, 0.9, 0.9)])
def test_emu_class_metrics(emu, shape, spacing):
    gt = organ_labels(shape, seed=11)
    pred = perturb_organs(gt, seed=12)
    classes = tuple(range(1, 10))
    ref = orc.class_table(pred, gt, classes, spacing)
    t = M.class_metrics(torch.from_numpy(pred), torch.from_numpy(gt), classes=classes, spacing=spacing)
    assert not compare(t, ref, spacing == (1.0, 1.0, 1.0))


def test_emu_golden(emu):
    for name, (pred, gt, spacing, classes, vals) in golden_cases().items():
        for nan in (True, False):
            t = M.class_metrics(torch.from_numpy(pred), torch.from_numpy(gt), classes=classes, spacing=spacing,
                                nan_for_nonexisting=nan)
            assert not compare(t, vals[nan], spacing == (1.0, 1.0, 1.0)), name
