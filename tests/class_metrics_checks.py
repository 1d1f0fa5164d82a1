"""Shared inputs and checks of metrics.class_metrics against oracle/class_metrics_oracle.py and the golden fixture, for the
CPU, the emulator and the GPU."""
import os

import numpy as np

from oracle import class_metrics_oracle as orc

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "class_metrics_cases.npz")
CONFUSION = tuple(m for m in orc.ALL_METRICS if m not in ("Hausdorff Distance", "Hausdorff Distance 95", "Avg. Surface Distance",
                                                         "Avg. Symmetric Surface Distance"))


def organ_labels(shape, seed=0, organs=9, batch=1):
    """(B, *shape) int64 labels 0..organs: ellipsoid organs of random centre and radii, later organs drawn over earlier ones"""
    rng = np.random.default_rng(seed)
    g = np.stack(np.meshgrid(*[np.arange(n) for n in shape], indexing="ij"), axis=0).astype(np.float64)
    out = np.zeros((batch,) + tuple(shape), dtype=np.int64)
    for b in range(batch):
        for k in range(1, organs + 1):
            c = np.array([rng.uniform(0.2, 0.8) * n for n in shape])
            r = np.array([max(n * rng.uniform(0.08, 0.25), 1.0) for n in shape])
            d = np.sqrt((((g - c[:, None, None, None]) / r[:, None, None, None]) ** 2).sum(0))
            out[b][d < 1.0] = k
    return out


def perturb_organs(labels, seed=1, organs=9):
    """a plausible prediction: a one-voxel shift along the last axis, with 1 % of the voxels relabelled at random"""
    rng = np.random.default_rng(seed)
    p = np.roll(labels, shift=1, axis=-1).copy()
    flip = rng.random(p.shape) < 0.01
    p[flip] = rng.integers(0, organs + 1, int(flip.sum())).astype(p.dtype)
    return p


def golden_cases():
    z = np.load(GOLDEN)
    names = sorted({k.split("/")[0] for k in z.files if "/" in k})
    metric_names = [str(v) for v in z["metric_names"]]
    out = {}
    for n in names:
        vals = {nan: {m: z[f"{n}/values_nan{int(nan)}"][i] for i, m in enumerate(metric_names)} for nan in (True, False)}
        out[n] = (z[f"{n}/pred"], z[f"{n}/gt"], tuple(z[f"{n}/spacing"].tolist()), tuple(int(c) for c in z[f"{n}/classes"]), vals)
    return out


def rel_err(a, b):
    """worst relative error, inf where the NaN patterns differ"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    if not np.array_equal(np.isnan(a), np.isnan(b)):
        return float("inf")
    m = ~np.isnan(b)
    if not m.any():
        return 0.0
    return float(np.max(np.abs(a[m] - b[m]) / np.maximum(np.abs(b[m]), 1e-300)))


def compare(table, ref, unit_spacing):
    """failures of a class_metrics table against reference values: confusion metrics bitwise, hd / hd95 bitwise at unit
    spacing and within 1e-12 otherwise, asd / assd within 1e-12"""
    bad = []
    for m in CONFUSION:
        if not np.array_equal(table[m], ref[m], equal_nan=True):
            bad.append((m, table[m], ref[m]))
    for m in ("Hausdorff Distance", "Hausdorff Distance 95"):
        ok = np.array_equal(table[m], ref[m], equal_nan=True) if unit_spacing else rel_err(table[m], ref[m]) <= 1e-12
        if not ok:
            bad.append((m, table[m], ref[m]))
    for m in ("Avg. Surface Distance", "Avg. Symmetric Surface Distance"):
        if rel_err(table[m], ref[m]) > 1e-12:
            bad.append((m, table[m], ref[m]))
    return bad


def ct_organs(shape, seed=0, organs=9):
    """(1, *shape) uint8 target and prediction of an abdominal-CT-like case: ellipsoid organs of 4-12 % of each axis, drawn
    inside their own boxes (fast at 400 x 512 x 512).  The prediction shifts every organ by one voxel along the last axis,
    odd organs by one more along axis 1, and adds a false-positive cube of organs 2 and 5 away from them."""
    rng = np.random.default_rng(seed)
    gt = np.zeros(shape, np.uint8)
    for k in range(1, organs + 1):
        c = np.array([rng.uniform(0.25, 0.75) * n for n in shape])
        r = np.array([max(n * rng.uniform(0.04, 0.12), 1.5) for n in shape])
        lo = np.maximum(np.floor(c - r).astype(int), 0)
        hi = np.minimum(np.ceil(c + r).astype(int) + 1, shape)
        g = np.meshgrid(*[np.arange(l, h) for l, h in zip(lo, hi)], indexing="ij")
        d = sum(((g[a] - c[a]) / r[a]) ** 2 for a in range(3))
        sub = gt[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]]
        sub[d < 1.0] = k
    pred = np.roll(gt, 1, axis=-1)
    odd = (pred % 2 == 1) & (pred > 0)
    pred = np.where(odd, 0, pred) + np.roll(np.where(odd, pred, 0), 1, axis=1).astype(np.uint8)
    pred[8:14, 20:26, 30:36] = 2
    pred[-20:-12, -40:-30, 10:18] = 5
    return pred[None].astype(np.uint8), gt[None]


def bincount_confusion(pred, gt, classes):
    """(B, K, 3) int64 |P|, |G|, |P and G| from numpy bincount"""
    B = pred.shape[0]
    out = np.zeros((B, len(classes), 3), np.int64)
    for b in range(B):
        p, g = pred[b].ravel().astype(np.int64), gt[b].ravel().astype(np.int64)
        cp, cg = np.bincount(p, minlength=256), np.bincount(g, minlength=256)
        cpg = np.bincount(p[p == g], minlength=256)
        for k, c in enumerate(classes):
            out[b, k] = cp[c], cg[c], cpg[c]
    return out
