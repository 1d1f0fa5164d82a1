"""Per-class evaluation (metrics.class_metrics) on the H100: against the oracle and the reference fixture, at raw-CT size
against numpy counts and box-cropped oracle distances, against the existing single-region path, across input dtypes and
layouts, batch and run-to-run invariance, and the readback count."""
import numpy as np
import pytest
import torch

from class_metrics_checks import (bincount_confusion, compare, ct_organs, golden_cases, organ_labels, perturb_organs,
                                  rel_err)
from metrics_checks import logits_for
from oracle import class_metrics_oracle as orc
from segmamba_b200 import metrics as M

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CLASSES = tuple(range(1, 10))
UNIT, ANISO = (1.0, 1.0, 1.0), (2.5, 0.9, 0.9)


def _run(pred, gt, **kw):
    return M.class_metrics(torch.from_numpy(pred).to(DEV), torch.from_numpy(gt).to(DEV), **kw)


@pytest.fixture(scope="module")
def organs():
    gt = organ_labels((40, 56, 60), seed=21)
    return perturb_organs(gt, seed=22), gt


@pytest.mark.parametrize("spacing", [UNIT, ANISO])
def test_nine_classes_against_oracle(organs, spacing):
    pred, gt = organs
    t = _run(pred, gt, classes=CLASSES, spacing=spacing)
    assert not compare(t, orc.class_table(pred, gt, CLASSES, spacing), spacing == UNIT)


def test_golden_cases():
    for name, (pred, gt, spacing, classes, vals) in golden_cases().items():
        for nan in (True, False):
            t = _run(pred, gt, classes=classes, spacing=spacing, nan_for_nonexisting=nan)
            assert not compare(t, vals[nan], spacing == UNIT), name


def test_raw_ct_size():
    pred, gt = ct_organs((400, 512, 512), seed=3)
    spacing = (1.0, 0.8, 0.8)
    t = _run(pred, gt, classes=CLASSES, spacing=spacing)
    cnt = bincount_confusion(pred, gt, CLASSES)
    p, g, tp = cnt[..., 0], cnt[..., 1], cnt[..., 2]
    n = gt[0].size
    assert np.array_equal(t["Total Positives Test"], p) and np.array_equal(t["Total Positives Reference"], g)
    assert np.array_equal(t["total Negatives Reference"], n - g) and np.array_equal(t["Total Negatives Test"], n - p)
    assert np.array_equal(t["Dice"], 2.0 * tp / (p + g))
    for k, c in enumerate(CLASSES):
        cp, cg = orc.box_crop(pred[0], gt[0], c)
        row = orc.all_metrics(cp, cg, spacing)
        for m in ("Hausdorff Distance", "Hausdorff Distance 95", "Avg. Surface Distance", "Avg. Symmetric Surface Distance"):
            assert rel_err(t[m][0, k], row[m]) <= 1e-12, (c, m, t[m][0, k], row[m])


@pytest.mark.parametrize("spacing", [UNIT, ANISO])
def test_agrees_with_region_path(organs, spacing):
    pred, gt = organs
    tp, tg = torch.from_numpy(pred).to(DEV), torch.from_numpy(gt).to(DEV)
    t = M.class_metrics(tp, tg, classes=CLASSES, spacing=spacing)
    checked = 0
    for k, c in enumerate(CLASSES):
        p, g = pred == c, gt == c
        if not p.any() or not g.any() or p.all() or g.all():
            continue
        reg = ((c,),)
        assert M.dice(tp, tg, regions=reg).cpu().numpy()[0, 0] == t["Dice"][0, k]
        hd = M.hd95(tp, tg, spacing=spacing, regions=reg, q=100.0).cpu().numpy()[0, 0]
        h95 = M.hd95(tp, tg, spacing=spacing, regions=reg).cpu().numpy()[0, 0]
        if spacing == UNIT:
            assert hd == t["Hausdorff Distance"][0, k] and h95 == t["Hausdorff Distance 95"][0, k], c
        else:
            assert rel_err(t["Hausdorff Distance"][0, k], hd) <= 1e-12 and rel_err(t["Hausdorff Distance 95"][0, k], h95) <= 1e-12
        checked += 1
    assert checked == 9


def _same(a, b):
    return all(np.array_equal(a[m], b[m], equal_nan=True) for m in M.ALL_METRICS)


def test_dtypes_and_layouts(organs):
    pred, gt = organs
    ref = _run(pred, gt, classes=CLASSES)
    tg = torch.from_numpy(gt).to(DEV)
    for dt in (torch.int8, torch.uint8, torch.int16, torch.int32, torch.int64):
        assert _same(M.class_metrics(torch.from_numpy(pred).to(DEV, dt), tg.to(dt), classes=CLASSES), ref), dt
    for dt in (torch.float32, torch.bfloat16, torch.float16):
        for cl in (False, True):
            lg = logits_for(pred, C=10, dtype=dt, channels_last=cl).to(DEV)
            assert _same(M.class_metrics(lg, tg, classes=CLASSES), ref), (dt, cl)


def test_wide_labels_int16():
    gt = organ_labels((20, 24, 26), seed=30)
    wide = np.array([0, 130, 200, 255, 300, 1000, 130, 200, 255, 300], dtype=np.int16)
    pred, tgt = wide[perturb_organs(gt, seed=31)], wide[gt]
    classes = (130, 200, 255)
    t = _run(pred, tgt, classes=classes)
    assert not compare(t, orc.class_table(pred, tgt, classes), True)


def test_batch_and_reruns(organs):
    pred, gt = organs
    gt2 = organ_labels((40, 56, 60), seed=23)
    pred2 = perturb_organs(gt2, seed=24)
    both = _run(np.concatenate([pred, pred2]), np.concatenate([gt, gt2]), classes=CLASSES, spacing=ANISO)
    one, two = _run(pred, gt, classes=CLASSES, spacing=ANISO), _run(pred2, gt2, classes=CLASSES, spacing=ANISO)
    for m in M.ALL_METRICS:
        assert np.array_equal(both[m], np.concatenate([one[m], two[m]]), equal_nan=True), m
    assert _same(_run(pred, gt, classes=CLASSES, spacing=ANISO), one)


def test_two_readbacks_and_no_other_sync(organs, monkeypatch):
    pred, gt = organs
    tp, tg = torch.from_numpy(pred).to(DEV), torch.from_numpy(gt).to(DEV)
    M.class_metrics(tp, tg, classes=CLASSES)                               # warm-up
    real = M._readback

    def readback(*t):
        torch.cuda.set_sync_debug_mode(0)
        try:
            return real(*t)
        finally:
            torch.cuda.set_sync_debug_mode("error")

    monkeypatch.setattr(M, "_readback", readback)
    torch.cuda.synchronize()
    n0 = M._readbacks
    torch.cuda.set_sync_debug_mode("error")
    try:
        M.class_metrics(tp, tg, classes=CLASSES)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert M._readbacks - n0 == M.READBACKS_PER_CALL == 2
