"""Test-only restatement of the evaluation the reference runs on the CPU (float64, numpy / scipy): medpy.metric.binary.dc and
hd95 / hd with connectivity 1 (medpy is not installed, so their semantics are written out here), the BraTS region
conversion, and the two case rules of 5_compute_metrics.cal_metric and 3_train.cal_metric / validation_step."""
from __future__ import annotations

import numpy as np
from scipy import ndimage

BRATS_REGIONS = ((1, 3), (1, 2, 3), (3,))


def regions_of(labels: np.ndarray, regions=BRATS_REGIONS) -> np.ndarray:
    """(..., D, H, W) labels -> (..., R, D, H, W) bool, region r = label in regions[r]."""
    return np.stack([np.isin(labels, r) for r in regions], axis=-4)


def dc(p: np.ndarray, g: np.ndarray) -> float:
    """medpy.metric.binary.dc: 2 |P and G| / (|P| + |G|), 0 when both are empty."""
    p, g = p.astype(bool), g.astype(bool)
    i, a, b = np.count_nonzero(p & g), np.count_nonzero(p), np.count_nonzero(g)
    return 2.0 * i / float(a + b) if a + b else 0.0


def border(m: np.ndarray) -> np.ndarray:
    m = m.astype(bool)
    return m ^ ndimage.binary_erosion(m, structure=ndimage.generate_binary_structure(m.ndim, 1), iterations=1)


def surface_distances(p: np.ndarray, g: np.ndarray, spacing=None) -> np.ndarray:
    """distance from every border voxel of p to the nearest border voxel of g (medpy's __surface_distances)."""
    sp = None if spacing is None else np.asarray(spacing, dtype=np.float64)
    dt = ndimage.distance_transform_edt(~border(g), sampling=sp)
    return dt[border(p)]


def hd_percentile(p: np.ndarray, g: np.ndarray, spacing=None, q: float = 95.0) -> float:
    """medpy.metric.binary.hd95 (q = 95) / hd (q = 100); NaN where either mask is empty (medpy raises)."""
    if not p.any() or not g.any():
        return float("nan")
    return float(np.percentile(np.hstack((surface_distances(p, g, spacing), surface_distances(g, p, spacing))), q))


def case_metric(p: np.ndarray, g: np.ndarray, spacing=None) -> np.ndarray:
    """5_compute_metrics.cal_metric: [dc, hd95] when both are non-empty, else [0, 50]."""
    if p.sum() > 0 and g.sum() > 0:
        return np.array([dc(p, g), hd_percentile(p, g, spacing)])
    return np.array([0.0, 50])


def each_cases_metric(pred_regions: np.ndarray, gt_regions: np.ndarray, spacing=None) -> np.ndarray:
    """(R, D, H, W) region masks -> (R, 2), as 5_compute_metrics.each_cases_metric."""
    return np.stack([case_metric(pred_regions[r], gt_regions[r], spacing) for r in range(pred_regions.shape[0])])


def validation_dices(pred_labels: np.ndarray, gt_labels: np.ndarray, regions=BRATS_REGIONS) -> list:
    """3_train.validation_step on (B, D, H, W) label maps: per region, Dice pooled over the batch; 1 when both are empty,
    0 when only one is."""
    p, g = regions_of(pred_labels, regions), regions_of(gt_labels, regions)
    out = []
    for r in range(len(regions)):
        pc, gc = p[:, r], g[:, r]
        if pc.sum() > 0 and gc.sum() > 0:
            tp = int((pc & gc).sum())
            out.append(np.float64(float(2.0 * tp / (pc.sum() + gc.sum()))))
        elif pc.sum() == 0 and gc.sum() == 0:
            out.append(np.float64(1.0))
        else:
            out.append(np.float64(0.0))
    return out
