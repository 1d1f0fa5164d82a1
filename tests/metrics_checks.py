"""Shared checks of the metric kernels (segmamba_b200/metrics.py) against oracle/metrics_oracle.py, for the emulator and the GPU."""
import numpy as np
import torch

from oracle import metrics_oracle as orc
from segmamba_b200 import metrics as M


def nested_labels(shape, seed=0, batch=1):
    """(B, *shape) int64 labels with nested blobs: 2 (edema) around 1 (necrosis) around 3 (enhancing), plus speckle."""
    rng = np.random.default_rng(seed)
    out = np.zeros((batch,) + tuple(shape), dtype=np.int64)
    g = np.stack(np.meshgrid(*[np.arange(n) for n in shape], indexing="ij"), axis=0).astype(np.float64)
    for b in range(batch):
        c = np.array([rng.uniform(0.3, 0.7) * n for n in shape])
        r = np.array([max(n * rng.uniform(0.15, 0.3), 0.8) for n in shape])
        d = np.sqrt((((g - c[:, None, None, None]) / r[:, None, None, None]) ** 2).sum(0))
        d = d + 0.15 * rng.standard_normal(d.shape)
        lab = np.where(d < 1.0, 2, 0)
        lab = np.where(d < 0.7, 1, lab)
        lab = np.where(d < 0.4, 3, lab)
        lab = np.where(rng.random(d.shape) < 0.002, rng.integers(1, 4, d.shape), lab)
        out[b] = lab
    return out


def perturb(labels, seed=1):
    """a plausible prediction: labels shifted by a voxel along each axis in some places, with random flips."""
    rng = np.random.default_rng(seed)
    p = np.roll(labels, shift=1, axis=-1).copy()
    flip = rng.random(p.shape) < 0.01
    p[flip] = rng.integers(0, 4, int(flip.sum()))
    return p


def oracle_case(pred, gt, spacing, q=95.0):
    """per (b, r): dice, hd_q from region masks (float64)."""
    P, G = orc.regions_of(pred), orc.regions_of(gt)
    B, R = P.shape[:2]
    d = np.array([[orc.dc(P[b, r], G[b, r]) for r in range(R)] for b in range(B)])
    h = np.array([[orc.hd_percentile(P[b, r], G[b, r], spacing, q) for r in range(R)] for b in range(B)])
    return d, h


def run_case(pred, gt, spacing, device, q=95.0):
    tp, tg = torch.from_numpy(pred).to(device), torch.from_numpy(gt).to(device)
    d = M.dice(tp, tg).cpu().numpy()
    h = M.hd95(tp, tg, spacing=spacing, q=q).cpu().numpy()
    return d, h


def logits_for(labels, C=4, dtype=torch.float32, channels_last=False, ties=True, seed=3):
    """logits whose argmax is `labels`, with exact ties between the winner and a later class where `ties`."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((labels.shape[0], C) + labels.shape[1:]).astype(np.float32)
    np.put_along_axis(x, labels[:, None], 4.0 + np.abs(x).max(), axis=1)
    if ties:
        later = np.minimum(labels + 1, C - 1)
        tie = (rng.random(labels.shape) < 0.3) & (later != labels)
        v = np.take_along_axis(x, labels[:, None], axis=1)
        cur = np.take_along_axis(x, later[:, None], axis=1)
        np.put_along_axis(x, later[:, None], np.where(tie[:, None], v, cur), axis=1)
    t = torch.from_numpy(x).to(dtype)
    if channels_last:
        t = t.contiguous(memory_format=torch.channels_last_3d)
    return t


def check_labels_and_logits(shape, device, spacings=((1.0, 1.0, 1.0), (2.5, 0.9, 0.9))):
    """worst relative errors of dice / hd95 / hd against the oracle, and whether logits give the label path's bits."""
    gt = nested_labels(shape, seed=0)
    pred = perturb(gt)
    res = {}
    for s in spacings:
        d_ref, h_ref = oracle_case(pred, gt, s)
        d, h = run_case(pred, gt, s, device)
        _, h100_ref = oracle_case(pred, gt, s, q=100.0)
        _, h100 = run_case(pred, gt, s, device, q=100.0)
        res[s] = {"dice_exact": np.array_equal(d, d_ref), "hd_err": _rel(h, h_ref), "hd100_err": _rel(h100, h100_ref),
                  "hd_exact": np.array_equal(h, h_ref, equal_nan=True), "hd100_exact": np.array_equal(h100, h100_ref, equal_nan=True)}
    ref_bits = M.region_bits(torch.from_numpy(pred).to(device)).cpu()
    logit_ok = {}
    for dt in (torch.float32, torch.bfloat16):
        for cl in (False, True):
            lg = logits_for(pred, dtype=dt, channels_last=cl).to(device)
            am = torch.argmax(lg.float(), dim=1)
            logit_ok[(str(dt), cl)] = bool(torch.equal(M.region_bits(lg).cpu(), ref_bits)
                                         and torch.equal(M.region_bits(am).cpu(), ref_bits))
    res["logits"] = logit_ok
    return res


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    if not np.array_equal(np.isnan(a), np.isnan(b)):
        return float("inf")
    m = ~np.isnan(b)
    if not m.any():
        return 0.0
    return float(np.max(np.abs(a[m] - b[m]) / np.maximum(np.abs(b[m]), 1e-300)))
