"""Test-only restatement of the reference's per-class evaluation (light_training/evaluation/metric.py, ALL_METRICS) in numpy /
scipy: the confusion-matrix family with each function's empty / full rule, and medpy.metric.binary's hd, hd95, asd and assd at
connectivity 1 on top of metrics_oracle.surface_distances (medpy is not installed, so its semantics are written out)."""
from __future__ import annotations

import numpy as np

from oracle.metrics_oracle import surface_distances

ALL_METRICS = ("False Positive Rate", "Dice", "Jaccard", "Hausdorff Distance", "Hausdorff Distance 95", "Precision", "Recall",
               "Avg. Symmetric Surface Distance", "Avg. Surface Distance", "Accuracy", "False Omission Rate",
               "Negative Predictive Value", "False Negative Rate", "True Negative Rate", "False Discovery Rate",
               "Total Positives Test", "Total Negatives Test", "Total Positives Reference", "total Negatives Reference")


def _check(result, reference, connectivity):
    if connectivity != 1:
        raise ValueError("only connectivity 1 is restated")
    if not np.any(result) or not np.any(reference):
        raise RuntimeError("a mask has no foreground")          # medpy raises here too


def hd(result, reference, voxelspacing=None, connectivity=1) -> float:
    _check(result, reference, connectivity)
    return float(max(surface_distances(result, reference, voxelspacing).max(),
                     surface_distances(reference, result, voxelspacing).max()))


def hd95(result, reference, voxelspacing=None, connectivity=1) -> float:
    _check(result, reference, connectivity)
    return float(np.percentile(np.hstack((surface_distances(result, reference, voxelspacing),
                                          surface_distances(reference, result, voxelspacing))), 95))


def asd(result, reference, voxelspacing=None, connectivity=1) -> float:
    """mean distance from result's border to reference's border"""
    _check(result, reference, connectivity)
    return surface_distances(result, reference, voxelspacing).mean()


def assd(result, reference, voxelspacing=None, connectivity=1) -> float:
    return np.mean((asd(result, reference, voxelspacing, connectivity), asd(reference, result, voxelspacing, connectivity)))


def all_metrics(test: np.ndarray, reference: np.ndarray, voxel_spacing=None, nan_for_nonexisting=True) -> dict:
    """{name: value} of every ALL_METRICS entry for one pair of binary masks"""
    test, reference = test != 0, reference != 0
    tp = int((test & reference).sum())
    fp = int((test & ~reference).sum())
    tn = int((~test & ~reference).sum())
    fn = int((~test & reference).sum())
    te, tf, re, rf = not test.any(), bool(test.all()), not reference.any(), bool(reference.all())
    miss = float("NaN") if nan_for_nonexisting else 0.
    spec = miss if rf else float(tn / (tn + fp))
    prec = miss if te else float(tp / (tp + fp))
    rec = miss if re else float(tp / (tp + fn))
    fomr = miss if tf else float(fn / (fn + tn))
    out = {"Dice": miss if te and re else float(2. * tp / (2 * tp + fp + fn)),
           "Jaccard": miss if te and re else float(tp / (tp + fp + fn)),
           "Precision": prec, "Recall": rec, "True Negative Rate": spec, "False Positive Rate": 1 - spec,
           "Accuracy": float((tp + tn) / (tp + fp + tn + fn)), "False Omission Rate": fomr, "Negative Predictive Value": 1 - fomr,
           "False Negative Rate": 1 - rec, "False Discovery Rate": 1 - prec, "Total Positives Test": tp + fp,
           "Total Negatives Test": tn + fn, "Total Positives Reference": tp + fn, "total Negatives Reference": tn + fp}
    degenerate = te or tf or re or rf
    dmiss = float("NaN") if nan_for_nonexisting else 0
    for name, fn_ in (("Hausdorff Distance", hd), ("Hausdorff Distance 95", hd95), ("Avg. Surface Distance", asd),
                      ("Avg. Symmetric Surface Distance", assd)):
        out[name] = dmiss if degenerate else fn_(test, reference, voxel_spacing)
    return out


def class_table(pred: np.ndarray, target: np.ndarray, classes, spacing=None, nan_for_nonexisting=True) -> dict:
    """(B, D, H, W) label maps -> {name: (B, K) float64}, class k = label classes[k]"""
    B, K = pred.shape[0], len(classes)
    out = {m: np.empty((B, K)) for m in ALL_METRICS}
    for b in range(B):
        for k, c in enumerate(classes):
            row = all_metrics(pred[b] == c, target[b] == c, spacing, nan_for_nonexisting)
            for m in ALL_METRICS:
                out[m][b, k] = row[m]
    return out


def box_crop(pred: np.ndarray, target: np.ndarray, c):
    """the two masks of class c cropped to the bounding box of their border voxels.  Every voxel of a mask lies between
    border voxels of it along each axis, so the box holds both masks whole and an interior voxel never lies on the box's face:
    the crop has the same border voxels at the same relative offsets, and the same distances."""
    from oracle.metrics_oracle import border
    p, g = pred == c, target == c
    idx = np.argwhere(border(p) | border(g))
    sl = tuple(slice(int(l), int(h) + 1) for l, h in zip(idx.min(0), idx.max(0)))
    return p[sl], g[sl]
