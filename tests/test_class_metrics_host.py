"""Host-side checks of per-class evaluation: the oracle against the fixture made by the reference's own metric.py, the EDT
planning from a count record, the exactness of the box crop, and argument validation."""
import ctypes

import numpy as np
import pytest
import torch

from class_metrics_checks import GOLDEN, golden_cases, organ_labels, perturb_organs
from oracle import class_metrics_oracle as orc
from segmamba_b200 import _lib
from segmamba_b200 import metrics as M


@pytest.mark.parametrize("nan", [True, False])
def test_oracle_matches_reference_fixture(nan):
    for name, (pred, gt, spacing, classes, vals) in golden_cases().items():
        t = orc.class_table(pred, gt, classes, spacing, nan)
        for m in orc.ALL_METRICS:
            assert np.array_equal(t[m], vals[nan][m], equal_nan=True), (name, m)


def test_metric_names_match_reference_order():
    z = np.load(GOLDEN)
    assert tuple(str(v) for v in z["metric_names"]) == M.ALL_METRICS == orc.ALL_METRICS


def test_host_confusion_rules_match_fixture():
    """metrics._confusion on exact counts gives the reference's values bit for bit, both empty / full rules included"""
    for name, (pred, gt, spacing, classes, vals) in golden_cases().items():
        for nan in (True, False):
            for b in range(pred.shape[0]):
                for k, c in enumerate(classes):
                    p, g = pred[b] == c, gt[b] == c
                    tp, n = int((p & g).sum()), p.size
                    row = M._confusion(tp, int(p.sum()) - tp, n - int(p.sum()) - int(g.sum()) + tp, int(g.sum()) - tp,
                                       not p.any(), bool(p.all()), not g.any(), bool(g.all()), nan)
                    for m, v in row.items():
                        assert np.array_equal(np.float64(v), vals[nan][m][b, k], equal_nan=True), (name, m, b, k)


def _record(pred, gt, classes):
    """the count record smb_metric_class_count writes, computed in numpy"""
    from oracle.metrics_oracle import border
    B, K = pred.shape[0], len(classes)
    shape = pred.shape[1:]
    rec = np.zeros((B, K, _lib.METRIC_CLASS_NREC), np.int64)
    for b in range(B):
        for k, c in enumerate(classes):
            p, g = pred[b] == c, gt[b] == c
            bp, bg = border(p), border(g)
            rec[b, k, :5] = p.sum(), g.sum(), (p & g).sum(), bp.sum(), bg.sum()
            idx = np.argwhere(bp | bg)
            if len(idx):
                rec[b, k, 5:8] = np.array(shape) - idx.min(0)
                rec[b, k, 8:11] = idx.max(0) + 1
    return rec


def test_plan_boxes_jobs_and_pools():
    gt = organ_labels((14, 16, 18), seed=4, batch=2)
    pred = perturb_organs(gt, seed=5)
    pred[0][pred[0] == 3] = 0                        # class 3 empty in sample 0's prediction
    gt[1][...] = np.where(gt[1] == 0, 2, gt[1])       # class 2 covers most of sample 1's target, not all of it
    full = np.full_like(gt[:1], 4)
    pred, gt = np.concatenate([pred, full]), np.concatenate([gt, gt[:1]])
    classes = tuple(range(1, 10))
    rec = _record(pred, gt, classes)
    plan = M.plan_edt(rec, gt.shape[1:])
    te, tf, re, rf = M.existence(rec, gt[0].size)
    want = [(b, k) for b in range(3) for k in range(9) if not (te[b, k] or tf[b, k] or re[b, k] or rf[b, k])]
    assert [tuple(r[:2]) for r in plan.pairs.tolist()] == want
    assert (0, 2) not in want and all(b != 2 for b, _ in want)            # empty and full classes are skipped
    from oracle.metrics_oracle import border
    for (b, k, z0, y0, x0, bd, bh, bw, n0, n1) in plan.pairs.tolist():
        bp, bg = border(pred[b] == classes[k]), border(gt[b] == classes[k])
        idx = np.argwhere(bp | bg)
        assert (z0, y0, x0) == tuple(idx.min(0)) and (bd, bh, bw) == tuple(idx.max(0) - idx.min(0) + 1)
        assert (n0, n1) == (bp.sum(), bg.sum())
    vol = plan.pairs[:, 5] * plan.pairs[:, 6] * plan.pairs[:, 7]
    assert plan.feat_len == 2 * vol.sum() and plan.pool_len == (plan.pairs[:, 8] + plan.pairs[:, 9]).sum()
    assert plan.line_len == 2 * (plan.pairs[:, 5] * plan.pairs[:, 7]).sum()
    assert np.array_equal(np.diff(plan.feat_off), 2 * vol[:-1]) and plan.feat_off[0] == 0
    assert np.array_equal(np.diff(plan.pool_off), (plan.pairs[:, 8] + plan.pairs[:, 9])[:-1])
    assert plan.max_box == tuple(int(plan.pairs[:, 5 + a].max()) for a in range(3))


def test_plan_of_nothing():
    rec = np.zeros((1, 3, _lib.METRIC_CLASS_NREC), np.int64)
    plan = M.plan_edt(rec, (4, 5, 6))
    assert len(plan.pairs) == 0 and plan.feat_len == plan.pool_len == plan.line_len == 0


@pytest.mark.parametrize("spacing", [None, (2.5, 0.9, 0.9)])
def test_box_crop_is_exact(spacing):
    gt = organ_labels((16, 18, 20), seed=9)[0]
    pred = perturb_organs(gt[None], seed=10)[0]
    for c in range(1, 10):
        p, g = pred == c, gt == c
        if not (p.any() and g.any()) or p.all() or g.all():
            continue
        cp, cg = orc.box_crop(pred, gt, c)
        assert cp.sum() == p.sum() and cg.sum() == g.sum()
        for fn in (orc.hd, orc.hd95, orc.asd, orc.assd):
            assert fn(cp, cg, spacing) == fn(p, g, spacing), (c, fn.__name__)


def test_class_lut():
    lut = M.class_lut((3, 200, 0))
    assert lut[3] == 1 and lut[200] == 2 and lut[0] == 3 and sum(1 for v in lut if v) == 3
    with pytest.raises(ValueError, match="1..255 classes"):
        M.class_lut(range(256))
    with pytest.raises(ValueError, match="1..255 classes"):
        M.class_lut(())
    with pytest.raises(ValueError, match="listed twice"):
        M.class_lut((1, 2, 1))
    with pytest.raises(ValueError, match="0..255"):
        M.class_lut((1, 256))
    with pytest.raises(ValueError, match="0..255"):
        M.class_lut((-1,))
    with pytest.raises(TypeError):
        M.class_lut((1.5,))


def test_argument_validation():
    x = torch.zeros((1, 4, 5, 6), dtype=torch.int64)
    with pytest.raises(ValueError, match="connectivity"):
        M.class_metrics(x, x, connectivity=2)
    with pytest.raises(ValueError, match="unknown metric"):
        M.class_metrics(x, x, metrics=("Dice", "Volume"))
    with pytest.raises(ValueError, match="spacing"):
        M.class_metrics(x, x, spacing=(1.0, 0.0, 1.0))
    with pytest.raises(ValueError, match="listed twice"):
        M.class_metrics(x, x, classes=(1, 1))
    with pytest.raises(RuntimeError, match="CUDA"):                  # no CPU path
        M.class_metrics(x, x)


def test_ctypes_layouts_match_header():
    import os
    import re
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(_lib.__file__))), "include", "segmamba_b200.h")).read()
    for cname, py in (("smb_metric_class_count_args", _lib.MetricClassCountArgs), ("smb_metric_edt_job", _lib.MetricEdtJob),
                      ("smb_metric_class_edt_args", _lib.MetricClassEdtArgs), ("smb_metric_pool", _lib.MetricPool),
                      ("smb_metric_class_reduce_args", _lib.MetricClassReduceArgs)):
        body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (cname, cname), src, re.S).group(1)
        body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
        fields = []
        for stmt in filter(None, (t.strip() for t in body.split(";"))):
            decl = re.sub(r"^(const\s+)?(void|double|int32_t|int64_t|smb_\w+)\s*", "", stmt)
            fields += [p.replace("*", "").strip() for p in decl.split(",")]
        assert [f[0] for f in py._fields_] == fields, cname
    assert ctypes.sizeof(_lib.MetricEdtJob) == 80 and ctypes.sizeof(_lib.MetricPool) == 40
