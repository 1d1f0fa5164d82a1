"""Dice and HD95 of segmentations on the GPU (csrc/metrics.cu): medpy.metric.binary.dc and hd95 / hd (connectivity 1), as the
reference's 5_compute_metrics.py and the validation_step of 3_train.py compute them on the CPU.

A prediction or target is one of
  * an integer label map (B, D, H, W);
  * logits (B, C, D, H, W) in fp32 / bf16 / fp16, contiguous or channels_last_3d: the argmax over C (first maximum) is fused
    into the region pass;
  * boolean region masks (B, R, D, H, W), one mask per region (the form 5_compute_metrics.py reads back).
A region is a set of label values (BRATS_REGIONS: TC, WT, ET).  HD95 is the 95th percentile (numpy 'linear') of the pooled
distances from each border voxel of P to the nearest border voxel of G and back, with `spacing` per array axis; a border voxel
is a foreground voxel with a 6-neighbour in the background or outside the volume.  Everything stays on the device and nothing
synchronises with the host except case_metrics / validation_dices, which read their small result once.  Results are bitwise
deterministic.

class_metrics evaluates disjoint classes (a class is one label value, up to 255 of them) with the full metric table of the
reference's light_training/evaluation/metric.py (ALL_METRICS): the confusion-matrix family from exact counts, and hd, hd95, asd
and assd from an EDT restricted to each class's box.  It reads back from the device at most READBACKS_PER_CALL (2) times.
"""
from __future__ import annotations

import ctypes
import operator
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib

BRATS_REGIONS = ((1, 3), (1, 2, 3), (3,))

_LABEL_KINDS = {torch.int8: _lib.METRIC_I8, torch.uint8: _lib.METRIC_U8, torch.int32: _lib.METRIC_I32, torch.int64: _lib.METRIC_I64}


def _lut(regions) -> list:
    regions = tuple(tuple(int(v) for v in r) for r in regions)
    if not 1 <= len(regions) <= _lib.METRIC_MAX_REGIONS:
        raise ValueError(f"1..{_lib.METRIC_MAX_REGIONS} regions are supported, got {len(regions)}")
    lut = [0] * 256
    for r, vals in enumerate(regions):
        for v in vals:
            if not 0 <= v < 256:
                raise ValueError(f"region label values must be in 0..255, got {v}")
            lut[v] |= 1 << r
    return lut


def region_bits(x: torch.Tensor, regions=BRATS_REGIONS) -> torch.Tensor:
    """labels (B, D, H, W), logits (B, C, D, H, W) or bool masks (B, R, D, H, W) -> (B, D, H, W) uint8, bit r = region r."""
    _lib.require_cuda(x)
    lut = _lut(regions)
    if x.dtype == torch.bool:
        if x.dim() != 5 or x.shape[1] != len(regions):
            raise ValueError(f"region masks must be (B, {len(regions)}, D, H, W), got {tuple(x.shape)}")
        shift = torch.arange(x.shape[1], dtype=torch.uint8, device=x.device).view(1, -1, 1, 1, 1)
        return (x.to(torch.uint8) << shift).sum(dim=1, dtype=torch.uint8)
    return _lut_bits(x, lut, _LABEL_KINDS)


def _lut_bits(x: torch.Tensor, lut, kinds) -> torch.Tensor:
    """labels (B, D, H, W) of a dtype in `kinds` or logits (B, C, D, H, W) -> (B, D, H, W) uint8 lut[label] (0 outside 0..255)"""
    if x.dtype in kinds:
        if x.dim() != 4:
            raise ValueError(f"a label map must be (B, D, H, W), got {tuple(x.shape)}")
        x = x.contiguous()
        B, vol = x.shape[0], x[0].numel()
        kind, dtype, classes, ss, cs, vs = kinds[x.dtype], 0, 0, vol, 0, 1
    elif x.dtype in (torch.float32, torch.float16, torch.bfloat16):
        if x.dim() != 5:
            raise ValueError(f"logits must be (B, C, D, H, W), got {tuple(x.shape)}")
        B, C, D, H, W = x.shape
        st = x.stride()
        vs = st[4]
        if st[2:] != (H * W * vs, W * vs, vs) or vs <= 0:           # neither NCDHW nor channels_last_3d
            x = x.contiguous()
            st, vs = x.stride(), 1
        vol = D * H * W
        kind, dtype, classes, ss, cs = _lib.METRIC_LOGITS, _lib.dtype_code(x.dtype), C, st[0], st[1]
    else:
        raise TypeError(f"unsupported prediction / target dtype {x.dtype}")
    bits = torch.empty((B,) + tuple(x.shape[-3:]), dtype=torch.uint8, device=x.device)
    a = _lib.MetricBitsArgs(src=x.data_ptr(), bits=bits.data_ptr(), voxels=vol, sample_stride=ss, class_stride=cs,
                            voxel_stride=vs, batch=B, kind=kind, dtype=dtype, classes=classes)
    a.lut[:] = lut
    dev = x.device
    sp = _lib.stream_ptr(dev)
    _lib.call("smb_metric_region_bits", (B,), lambda: _lib.lib().smb_metric_region_bits(ctypes.byref(a), sp), dev)
    return bits


def _prepare(pred, target, regions):
    pb, gb = region_bits(pred, regions), region_bits(target, regions)
    if pb.shape != gb.shape:
        raise ValueError(f"prediction and target cover different volumes: {tuple(pb.shape)} vs {tuple(gb.shape)}")
    return pb, gb


def _counts(pb: torch.Tensor, gb: torch.Tensor, R: int):
    """(B, R, 8) int64 counts (|P|, |G|, |P and G|, |border P|, |border G|, pool fill, 0, 0) and the two border masks."""
    B, D, H, W = pb.shape
    counts = torch.zeros((B, R, _lib.METRIC_NCOUNTS), dtype=torch.int64, device=pb.device)
    pbd, gbd = torch.empty_like(pb), torch.empty_like(gb)
    a = _lib.MetricCountArgs(pb.data_ptr(), gb.data_ptr(), pbd.data_ptr(), gbd.data_ptr(), counts.data_ptr(), B, R, D, H, W)
    dev = pb.device
    sp = _lib.stream_ptr(dev)
    _lib.call("smb_metric_count", (B, R), lambda: _lib.lib().smb_metric_count(ctypes.byref(a), sp), dev)
    return counts, pbd, gbd


def _dice_from(counts: torch.Tensor) -> torch.Tensor:
    c = counts.to(torch.float64)
    den = c[..., 0] + c[..., 1]
    return torch.where(den > 0, (2.0 * c[..., 2]) / torch.where(den > 0, den, torch.ones_like(den)), torch.zeros_like(den))


def _hd_from(counts, pbd, gbd, spacing, q: float) -> torch.Tensor:
    B, R = counts.shape[:2]
    D, H, W = pbd.shape[1:]
    s = tuple(float(v) for v in spacing)
    if len(s) != 3:
        raise ValueError(f"spacing must give three axes, got {spacing}")
    if not 0.0 <= float(q) <= 100.0:
        raise ValueError(f"q must be in [0, 100], got {q}")
    n = D * H * W
    cap = 2 * n
    dev = pbd.device
    feat = torch.empty((B * R * 2, n), dtype=torch.int32, device=dev)
    pool = torch.empty((B * R, cap), dtype=torch.float64, device=dev)
    out = torch.empty((B, R), dtype=torch.float64, device=dev)
    sp = _lib.stream_ptr(dev)
    e = _lib.MetricEdtArgs(pbd.data_ptr(), gbd.data_ptr(), feat.data_ptr(), pool.data_ptr(), counts.data_ptr(), cap,
                           B, R, D, H, W, *s)
    _lib.call("smb_metric_edt", (B, R, D, H, W), lambda: _lib.lib().smb_metric_edt(ctypes.byref(e), sp), dev)
    sel = _lib.MetricSelectArgs(pool.data_ptr(), counts.data_ptr(), out.data_ptr(), cap, B, R, float(q) / 100.0)
    _lib.call("smb_metric_select", (B, R), lambda: _lib.lib().smb_metric_select(ctypes.byref(sel), sp), dev)
    return out


def overlap_counts(pred, target, regions=BRATS_REGIONS) -> torch.Tensor:
    """(B, R, 3) int64: |P|, |G|, |P and G| per sample and region."""
    pb, gb = _prepare(pred, target, regions)
    return _counts(pb, gb, len(regions))[0][..., :3]


def dice(pred, target, regions=BRATS_REGIONS) -> torch.Tensor:
    """(B, R) fp64 medpy.metric.binary.dc: 2 |P and G| / (|P| + |G|), 0 where both are empty."""
    pb, gb = _prepare(pred, target, regions)
    return _dice_from(_counts(pb, gb, len(regions))[0])


def hd95(pred, target, spacing=(1.0, 1.0, 1.0), regions=BRATS_REGIONS, q: float = 95.0) -> torch.Tensor:
    """(B, R) fp64 medpy.metric.binary.hd95 (q = 100: hd) with voxelspacing `spacing` in array-axis order; NaN where P or
    G is empty."""
    pb, gb = _prepare(pred, target, regions)
    counts, pbd, gbd = _counts(pb, gb, len(regions))
    return _hd_from(counts, pbd, gbd, spacing, q)


def case_metrics(pred, target, spacing=(1.0, 1.0, 1.0), regions=BRATS_REGIONS) -> np.ndarray:
    """(R, 2) numpy array of 5_compute_metrics.each_cases_metric for one case (batch 1): [dice, hd95] per region when both
    P and G are non-empty, else [0, 50]."""
    pb, gb = _prepare(pred, target, regions)
    if pb.shape[0] != 1:
        raise ValueError(f"case_metrics takes one case (batch 1), got batch {pb.shape[0]}")
    counts, pbd, gbd = _counts(pb, gb, len(regions))
    both = (counts[0, :, 0] > 0) & (counts[0, :, 1] > 0)
    res = torch.stack([_dice_from(counts)[0], _hd_from(counts, pbd, gbd, spacing, 95.0)[0]], dim=1)
    res = torch.where(both[:, None], res, torch.tensor([0.0, 50.0], dtype=torch.float64, device=res.device))
    return res.cpu().numpy()


def validation_dices(logits, label, regions=BRATS_REGIONS) -> list:
    """The list validation_step of 3_train.py returns: per region, Dice over the whole batch (argmax of the logits against
    the label map), 1 when both are empty, 0 when only one is."""
    pb, gb = _prepare(logits, label, regions)
    c = _counts(pb, gb, len(regions))[0].sum(dim=0)
    p, g = c[:, 0], c[:, 1]
    d = torch.where((p > 0) & (g > 0), _dice_from(c), torch.where((p == 0) & (g == 0), 1.0, 0.0).to(torch.float64))
    return [np.float64(v) for v in d.cpu().numpy()]


# ---- per-class evaluation: the metric table of light_training/evaluation/metric.py --------------------------------------------
ALL_METRICS = ("False Positive Rate", "Dice", "Jaccard", "Hausdorff Distance", "Hausdorff Distance 95", "Precision", "Recall",
               "Avg. Symmetric Surface Distance", "Avg. Surface Distance", "Accuracy", "False Omission Rate",
               "Negative Predictive Value", "False Negative Rate", "True Negative Rate", "False Discovery Rate",
               "Total Positives Test", "Total Negatives Test", "Total Positives Reference", "total Negatives Reference")
DISTANCE_METRICS = ("Hausdorff Distance", "Hausdorff Distance 95", "Avg. Surface Distance", "Avg. Symmetric Surface Distance")
READBACKS_PER_CALL = 2
_readbacks = 0                   # device-to-host synchronisations made by _readback (tests count them)

_CLASS_KINDS = dict(_LABEL_KINDS)
_CLASS_KINDS[torch.int16] = _lib.METRIC_I16
_REC_P, _REC_G, _REC_PG, _REC_BP, _REC_BG = range(5)


def _readback(*tensors) -> list:
    """one synchronisation: every tensor copied to the host, as numpy arrays"""
    global _readbacks
    _readbacks += 1
    out = [t.to("cpu", non_blocking=True) for t in tensors]
    if any(t.is_cuda for t in tensors):
        torch.cuda.synchronize(tensors[0].device)
    return [o.numpy() for o in out]


def _upload(arr, device) -> torch.Tensor:
    """a ctypes array as device bytes, copied from page-locked memory without synchronising"""
    t = torch.frombuffer(bytearray(arr), dtype=torch.uint8)
    if torch.device(device).type != "cuda":
        return t
    return t.pin_memory().to(device, non_blocking=True)


def class_lut(classes) -> list:
    """256-entry label -> class-index + 1 table (0: no class) for up to 255 distinct labels in 0..255"""
    cls = [operator.index(c) for c in classes]
    if not 1 <= len(cls) <= _lib.METRIC_MAX_CLASSES:
        raise ValueError(f"1..{_lib.METRIC_MAX_CLASSES} classes are supported, got {len(cls)}")
    lut = [0] * 256
    for k, c in enumerate(cls):
        if not 0 <= c < 256:
            raise ValueError(f"class labels must be in 0..255, got {c}")
        if lut[c]:
            raise ValueError(f"class label {c} is listed twice")
        lut[c] = k + 1
    return lut


@dataclass
class EdtPlan:
    """the EDT work of one class_metrics call, planned from the count record.  pairs[i] = (b, k, z0, y0, x0, bd, bh, bw, n0,
    n1) for the (sample, class) pairs whose masks are both non-empty and non-full; the box is that of the border voxels of P
    and G.  Pair i has two jobs (P's border -> G's, then G's -> P's), each with bd * bh * bw features from feat_off[i] + dir
    * bd * bh * bw, and bd * bw lines from line_off[i] + dir * bd * bw; its pool holds n0 + n1 distances from pool_off[i]."""
    pairs: np.ndarray
    feat_off: np.ndarray
    line_off: np.ndarray
    pool_off: np.ndarray
    feat_len: int
    line_len: int
    pool_len: int
    max_box: tuple


def existence(record: np.ndarray, voxels: int):
    """(test_empty, test_full, reference_empty, reference_full) boolean arrays of a (B, K, NREC) count record"""
    p, g = record[..., _REC_P], record[..., _REC_G]
    return p == 0, p == voxels, g == 0, g == voxels


def plan_edt(record: np.ndarray, shape) -> EdtPlan:
    D, H, W = (int(v) for v in shape)
    te, tf, re, rf = existence(record, D * H * W)
    todo = ~(te | tf | re | rf)
    rows = []
    for b, k in zip(*np.nonzero(todo)):
        r = record[b, k]
        lo = (D - int(r[5]), H - int(r[6]), W - int(r[7]))
        ext = tuple(int(r[8 + a]) - lo[a] for a in range(3))
        rows.append((int(b), int(k)) + lo + ext + (int(r[_REC_BP]), int(r[_REC_BG])))
    pairs = np.array(rows, dtype=np.int64).reshape(-1, 10)
    vol = pairs[:, 5] * pairs[:, 6] * pairs[:, 7]
    lines = pairs[:, 5] * pairs[:, 7]
    npool = pairs[:, 8] + pairs[:, 9]

    def offsets(sizes):
        return np.concatenate(([0], np.cumsum(sizes)[:-1])).astype(np.int64) if len(sizes) else np.zeros(0, np.int64)

    max_box = tuple(int(pairs[:, 5 + a].max()) if len(pairs) else 0 for a in range(3))
    if max_box[1] > _lib.METRIC_MAX_AXIS or max_box[2] > _lib.METRIC_MAX_AXIS:
        raise ValueError(f"class boxes are limited to {_lib.METRIC_MAX_AXIS} voxels along axes 1 and 2, got {max_box}")
    return EdtPlan(pairs, offsets(2 * vol), offsets(2 * lines), offsets(npool), int(2 * vol.sum()), int(2 * lines.sum()),
                   int(npool.sum()), max_box)


def _distances(plan: EdtPlan, pbd, gbd, spacing, device):
    """(npairs, 4) fp64 on the device: hd, hd95, asd, assd per planned pair"""
    B, D, H, W = pbd.shape
    n = D * H * W
    npairs = len(plan.pairs)
    feat = torch.empty(plan.feat_len, dtype=torch.int32, device=device)
    pool = torch.empty(plan.pool_len, dtype=torch.float64, device=device)
    lines = torch.empty(2 * plan.line_len, dtype=torch.float64, device=device)
    fill = torch.zeros(npairs, dtype=torch.int64, device=device)
    out = torch.empty((npairs, 4), dtype=torch.float64, device=device)
    jobs = (_lib.MetricEdtJob * (2 * npairs))()
    pools = (_lib.MetricPool * npairs)()
    maps = (pbd.data_ptr(), gbd.data_ptr())
    for i, (b, k, z0, y0, x0, bd, bh, bw, n0, n1) in enumerate(plan.pairs.tolist()):
        origin = b * n + (z0 * H + y0) * W + x0
        for d in (0, 1):
            j = jobs[2 * i + d]
            j.src, j.tgt = maps[d] + origin, maps[1 - d] + origin
            j.feat = feat.data_ptr() + 4 * (int(plan.feat_off[i]) + d * bd * bh * bw)
            j.pool = pool.data_ptr() + 8 * int(plan.pool_off[i])
            j.fill = fill.data_ptr() + 8 * i
            j.lines = lines.data_ptr() + 16 * (int(plan.line_off[i]) + d * bd * bw)
            j.bd, j.bh, j.bw = bd, bh, bw
            j.src_mask = j.tgt_mask = 0xFF
            j.src_val = j.tgt_val = k + 1
        pools[i] = _lib.MetricPool(pool.data_ptr() + 8 * int(plan.pool_off[i]), lines.data_ptr() + 16 * int(plan.line_off[i]),
                                   n0, n1, bd * bw, bd * bw)
    jobs_dev, pools_dev = _upload(jobs, device), _upload(pools, device)
    sp = _lib.stream_ptr(device)
    e = _lib.MetricClassEdtArgs(jobs_dev.data_ptr(), W, H * W, 2 * npairs, *plan.max_box, *spacing)
    _lib.call("smb_metric_class_edt", (npairs,) + plan.max_box, lambda: _lib.lib().smb_metric_class_edt(ctypes.byref(e), sp), device)
    r = _lib.MetricClassReduceArgs(pools_dev.data_ptr(), out.data_ptr(), npairs, 0.95)
    _lib.call("smb_metric_class_reduce", (npairs,), lambda: _lib.lib().smb_metric_class_reduce(ctypes.byref(r), sp), device)
    return out, (jobs_dev, pools_dev)


def _confusion(tp: int, fp: int, tn: int, fn: int, te, tf, re, rf, nan_for_nonexisting: bool) -> dict:
    """the confusion-matrix rows of ALL_METRICS for one class, with metric.py's Python arithmetic and empty / full rules"""
    miss = float("NaN") if nan_for_nonexisting else 0.
    dice = miss if te and re else float(2. * tp / (2 * tp + fp + fn))
    jaccard = miss if te and re else float(tp / (tp + fp + fn))
    precision = miss if te else float(tp / (tp + fp))
    recall = miss if re else float(tp / (tp + fn))
    specificity = miss if rf else float(tn / (tn + fp))
    omission = miss if tf else float(fn / (fn + tn))
    return {"False Positive Rate": 1 - specificity, "Dice": dice, "Jaccard": jaccard, "Precision": precision, "Recall": recall,
            "Accuracy": float((tp + tn) / (tp + fp + tn + fn)), "False Omission Rate": omission,
            "Negative Predictive Value": 1 - omission, "False Negative Rate": 1 - recall, "True Negative Rate": specificity,
            "False Discovery Rate": 1 - precision, "Total Positives Test": tp + fp, "Total Negatives Test": tn + fn,
            "Total Positives Reference": tp + fn, "total Negatives Reference": tn + fp}


def class_metrics(pred, target, classes=range(1, 10), spacing=(1.0, 1.0, 1.0), metrics=None, nan_for_nonexisting=True,
                  connectivity=1) -> dict:
    """{metric name: (B, K) fp64 numpy array} of light_training/evaluation/metric.py's ALL_METRICS for each sample and class
    k, with P = (pred == classes[k]) and G = (target == classes[k]).  pred is labels (B, D, H, W) (int8 / uint8 / int16 /
    int32 / int64) or logits (B, C, D, H, W) (fp32 / bf16 / fp16; argmax, first maximum); target is labels.  `spacing` is
    medpy's voxelspacing in array-axis order (None: unit); `metrics` a subset of ALL_METRICS (None: all).  The distance metrics
    are medpy's hd, hd95, asd and assd at connectivity 1, NaN (or 0 without nan_for_nonexisting) where P or G is empty or fills
    the volume."""
    if connectivity != 1:
        raise ValueError(f"only connectivity 1 is supported, got {connectivity}")
    names = ALL_METRICS if metrics is None else tuple(metrics)
    for m in names:
        if m not in ALL_METRICS:
            raise ValueError(f"unknown metric {m!r}; the names are those of ALL_METRICS")
    s = (1.0, 1.0, 1.0) if spacing is None else tuple(float(v) for v in spacing)
    if len(s) != 3 or not all(np.isfinite(v) and v > 0 for v in s):
        raise ValueError(f"spacing must give three positive axes, got {spacing}")
    lut = class_lut(classes)
    K = sum(1 for v in lut if v)
    _lib.require_cuda(pred, target)
    if target.dtype not in _CLASS_KINDS:
        raise TypeError(f"the target must be a label map, got dtype {target.dtype}")
    pb, gb = _lut_bits(pred, lut, _CLASS_KINDS), _lut_bits(target, lut, _CLASS_KINDS)
    if pb.shape != gb.shape:
        raise ValueError(f"prediction and target cover different volumes: {tuple(pb.shape)} vs {tuple(gb.shape)}")
    B, D, H, W = pb.shape
    if D * H * W > 2**31 - 1:
        raise ValueError("volumes are limited to 2^31 - 1 voxels")
    dev = pb.device
    record = torch.zeros((B, K, _lib.METRIC_CLASS_NREC), dtype=torch.int64, device=dev)
    pbd, gbd = torch.empty_like(pb), torch.empty_like(gb)
    a = _lib.MetricClassCountArgs(pb.data_ptr(), gb.data_ptr(), pbd.data_ptr(), gbd.data_ptr(), record.data_ptr(), B, K, D, H, W)
    sp = _lib.stream_ptr(dev)
    _lib.call("smb_metric_class_count", (B, K), lambda: _lib.lib().smb_metric_class_count(ctypes.byref(a), sp), dev)
    rec = _readback(record)[0]                                                            # readback 1
    n = D * H * W
    te, tf, re, rf = existence(rec, n)
    dist = np.full((B, K, 4), np.nan)
    if any(m in DISTANCE_METRICS for m in names):
        plan = plan_edt(rec, (D, H, W))
        if len(plan.pairs):
            out, keep = _distances(plan, pbd, gbd, s, dev)
            host = _readback(out)[0]                                                      # readback 2
            dist[plan.pairs[:, 0], plan.pairs[:, 1]] = host
            del keep
    miss = float("NaN") if nan_for_nonexisting else 0
    table = {m: np.empty((B, K), dtype=np.float64) for m in names}
    for b in range(B):
        for k in range(K):
            p, g, tp = (int(v) for v in rec[b, k, :3])
            flags = (bool(te[b, k]), bool(tf[b, k]), bool(re[b, k]), bool(rf[b, k]))
            row = _confusion(tp, p - tp, n - p - g + tp, g - tp, *flags, nan_for_nonexisting)
            hd, hd95_, asd, assd = (miss,) * 4 if any(flags) else dist[b, k].tolist()
            row.update({"Hausdorff Distance": hd, "Hausdorff Distance 95": hd95_, "Avg. Surface Distance": asd,
                        "Avg. Symmetric Surface Distance": assd})
            for m in names:
                table[m][b, k] = row[m]
    return table
