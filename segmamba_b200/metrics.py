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
"""
from __future__ import annotations

import ctypes

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
    if x.dtype in _LABEL_KINDS:
        if x.dim() != 4:
            raise ValueError(f"a label map must be (B, D, H, W), got {tuple(x.shape)}")
        x = x.contiguous()
        B, vol = x.shape[0], x[0].numel()
        kind, dtype, classes, ss, cs, vs = _LABEL_KINDS[x.dtype], 0, 0, vol, 0, 1
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
