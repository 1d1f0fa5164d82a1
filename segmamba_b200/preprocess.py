"""Case preprocessing on the GPU (csrc/preprocess.cu): the reference's 2_preprocessing_mri.py step for one case --
MultiModalityPreprocessor.read_data's foreground intensities and DefaultPreprocessor.run_case_npy -- with the data on the device.

  * nonzero_mask: create_nonzero_mask -- OR over channels of data != 0 (NaN counts as nonzero), holes filled
    (scipy.ndimage.binary_fill_holes, via predict.fill_holes).
  * crop_to_nonzero: the bbox of that mask ([[lo, hi + 1]] per axis; an all-zero case raises ValueError), data and seg cropped
    to it, seg 0 outside the mask set to nonzero_label (without a seg: 0 inside, nonzero_label outside, int8).
  * zscore: ZScoreNormalization(use_mask_for_norm=False) per channel over the whole box, divisor max(std, 1e-8); mean and std
    are fp64 from an ordered reduction (smb_aug_stats), so the result is deterministic.
  * ct_normalize: CTNormalization per channel from the dataset's foreground statistics (plan.plan_dataset), clip to the
    0.5 / 99.5 percentiles then (x - mean) / max(std, 1e-8), in fp32 bit-equal to numpy.
  * compute_new_shape: the reference's, with Python round.
  * resample_case: skimage resize(order=3, mode='edge', anti_aliasing=False) of every channel, clipped to its range
    (smb_aug_stats + smb_aug_prefilter + smb_aug_resample, augment.py's low-resolution path), and batchgenerators
    resize_segmentation(order=1) of the labels.  An unchanged shape touches nothing.
  * sample_foreground_locations / foreground_intensities: the reference's RandomState(seed) draws, made on the host from
    counts read back from the device (choice(n, ...) depends only on n), over indices compacted on the device in raster
    order; the device gathers the drawn rows and intensities.
  * preprocess_case: all of it in the reference's order, returning (data, seg, properties); normalization="ct" runs the
    DefaultPreprocessor of the reference's CT pipelines instead of the z-score.

Bounds: labels must be integers in [0, 127] (the reference switches to int16 above 127; here that raises ValueError), volumes
below 2^31 voxels, and a resampled case needs crop axes of at least 4 voxels.

nonzero_mask, zscore, ct_normalize and resample_case never synchronise with the host.  Everything the host needs goes through `_readback`;
preprocess_case makes exactly READBACKS_PER_CASE (3) of them: the mask record (bbox, foreground count, NaN and label checks),
the label counts, and the drawn rows with the intensity samples and statistics.
"""
from __future__ import annotations

import ctypes
import math

import numpy as np
import torch

from . import _lib
from . import augment as A
from .predict import fill_holes

__all__ = ["nonzero_mask", "crop_to_nonzero", "zscore", "ct_normalize", "compute_new_shape", "resample_case", "sample_foreground_locations",
           "foreground_intensities", "preprocess_case", "READBACKS_PER_CASE"]

READBACKS_PER_CASE = 3
_readbacks = 0                   # device-to-host synchronisations made by _readback (tests count them)


def _readback(*tensors) -> list:
    """one synchronisation: every tensor copied to the host, as numpy arrays"""
    global _readbacks
    _readbacks += 1
    out = [t.to("cpu", non_blocking=True) for t in tensors]
    if any(t.is_cuda for t in tensors):
        torch.cuda.synchronize(tensors[0].device)
    return [o.numpy() for o in out]


def _call(name: str, args, device) -> None:
    fn = getattr(_lib.lib(), name)
    sp = _lib.stream_ptr(device)
    _lib.call(name, (), lambda: fn(ctypes.byref(args), sp), device)


def _data(data: torch.Tensor) -> torch.Tensor:
    _lib.require_cuda(data)
    if data.dim() != 4 or min(data.shape) == 0:
        raise ValueError(f"data must be a non-empty (C, D, H, W) tensor, got {tuple(data.shape)}")
    if math.prod(data.shape[1:]) >= 2 ** 31:
        raise ValueError(f"volumes are limited to 2^31 - 1 voxels, got {tuple(data.shape[1:])}")
    return data.to(torch.float32).contiguous()


def _seg(seg, shape) -> torch.Tensor | None:
    """(1, D, H, W) or (D, H, W), integer or integral float -> (D, H, W) fp32 (the reference reads labels as float32)"""
    if seg is None:
        return None
    _lib.require_cuda(seg)
    if seg.dim() == 4:
        if seg.shape[0] != 1:
            raise ValueError(f"seg must be (1, D, H, W) or (D, H, W), got {tuple(seg.shape)}")
        seg = seg[0]
    if tuple(seg.shape) != tuple(shape):
        raise ValueError(f"seg shape {tuple(seg.shape)} differs from the data's {tuple(shape)}")
    return seg.to(torch.float32).contiguous()


def _analyse(data: torch.Tensor, seg: torch.Tensor | None):
    """mask pass: (nonzero mask uint8, labels int8, int64 record of smb_prep_record)"""
    C, D, H, W = data.shape
    dev = data.device
    mask = torch.empty((D, H, W), dtype=torch.uint8, device=dev)
    seg8 = torch.empty((D, H, W), dtype=torch.int8, device=dev)
    rec = torch.empty(9, dtype=torch.int64, device=dev)
    _call("smb_prep_mask", _lib.PrepMaskArgs(data.data_ptr(), _lib.ptr(seg), mask.data_ptr(), seg8.data_ptr(), rec.data_ptr(),
                                             C, D, H, W), dev)
    return mask, seg8, rec


def _bbox(rec: np.ndarray) -> list:
    if rec[3] == 0:
        raise ValueError("the case has no nonzero voxel: there is no bounding box to crop to")
    return [[int(2 ** 31 - rec[q]), int(rec[3 + q])] for q in range(3)]


def _check(rec: np.ndarray, has_seg: bool) -> None:
    if rec[8]:
        raise ValueError(f"seg has {int(rec[8])} voxels that are not integer labels in [0, 127] (int8 labels only)")
    if has_seg and rec[7]:
        raise ValueError(f"data has {int(rec[7])} voxels with a NaN")


def _crop(data, filled, seg8, bbox, nonzero_label: int = -1):
    C, D, H, W = data.shape
    (z0, z1), (y0, y1), (x0, x1) = bbox
    box = (z1 - z0, y1 - y0, x1 - x0)
    dev = data.device
    out = torch.empty((C,) + box, dtype=torch.float32, device=dev)
    seg = torch.empty((1,) + box, dtype=torch.int8, device=dev)
    _call("smb_prep_crop", _lib.PrepCropArgs(data.data_ptr(), filled.data_ptr(), seg8.data_ptr(), out.data_ptr(), seg.data_ptr(),
                                             C, D, H, W, z0, y0, x0, *box, nonzero_label), dev)
    return out, seg


def nonzero_mask(data: torch.Tensor) -> torch.Tensor:
    """bool (D, H, W): the reference's create_nonzero_mask of a (C, D, H, W) case, on the device."""
    mask, _, _ = _analyse(_data(data), None)
    return fill_holes(mask)


def crop_to_nonzero(data: torch.Tensor, seg: torch.Tensor | None = None, nonzero_label: int = -1):
    """(data (C, d, h, w) fp32, seg (1, d, h, w) int8, bbox) as the reference's crop_to_nonzero; raises ValueError for a case
    without a nonzero voxel.  Reads the bbox back (one synchronisation)."""
    data = _data(data)
    seg = _seg(seg, data.shape[1:])
    mask, seg8, rec = _analyse(data, seg)
    filled = fill_holes(mask)
    rec = _readback(rec)[0]
    _check(rec, False)
    bbox = _bbox(rec)
    d, s = _crop(data, filled, seg8, bbox, nonzero_label)
    return d, s, bbox


def _stats(x: torch.Tensor) -> torch.Tensor:
    """(C, 4) fp64 sum, sum of squares, min, max of each channel of a contiguous (C, ...) fp32 tensor (smb_aug_stats)"""
    C, n = x.shape[0], x[0].numel()
    st = torch.empty((C, 4), dtype=torch.float64, device=x.device)
    scr = torch.empty((C, _lib.AUG_STATS_SCRATCH), dtype=torch.float64, device=x.device)
    A.stats([A.stats_job(x[c], st[c], scr[c], n) for c in range(C)], x.device)
    return st


def zscore(data: torch.Tensor):
    """(normalised (C, D, H, W) fp32, moments (C, 2) fp64 mean and std): ZScoreNormalization(use_mask_for_norm=False) of
    every channel, (x - mean) / max(std, 1e-8) in fp64 rounded to fp32.  No synchronisation."""
    data = _data(data)
    C, n = data.shape[0], data[0].numel()
    st = _stats(data)
    out = torch.empty_like(data)
    mom = torch.empty((C, 2), dtype=torch.float64, device=data.device)
    A._run("smb_prep_normalize", _lib.PrepNormJob,
           [_lib.PrepNormJob(data[c].data_ptr(), out[c].data_ptr(), st[c].data_ptr(), mom[c].data_ptr(), n) for c in range(C)],
           data.device)
    return out, mom


_CT_KEYS = ("mean", "std", "percentile_00_5", "percentile_99_5")


def ct_normalize(data: torch.Tensor, intensity_properties) -> torch.Tensor:
    """(C, D, H, W) fp32: CTNormalization(use_mask_for_norm=False) of every channel with intensity_properties[str(c)] (a dict
    with mean, std, percentile_00_5 and percentile_99_5, as plan.plan_dataset or the reference's data_analysis_result.txt give
    them): clip to [percentile_00_5, percentile_99_5], then (x - mean) / max(std, 1e-8), all in fp32 as numpy computes it for
    a float32 image.  Raises ValueError for a missing channel or key.  No synchronisation."""
    data = _data(data)
    C, n = data.shape[0], data[0].numel()
    f = np.float32
    jobs = []
    out = torch.empty_like(data)
    for c in range(C):
        try:
            p = intensity_properties[str(c)]
            mean, std, lo, hi = (p[k] for k in _CT_KEYS)
        except (KeyError, IndexError, TypeError) as e:
            raise ValueError(f"intensity_properties needs channel '{c}' with {', '.join(_CT_KEYS)}: {e!r}") from None
        jobs.append(_lib.PrepCtNormJob(data[c].data_ptr(), out[c].data_ptr(), n, f(lo), f(hi), f(mean), f(max(std, 1e-8))))
    A._run("smb_prep_ct_normalize", _lib.PrepCtNormJob, jobs, data.device)
    return out


def compute_new_shape(old_shape, old_spacing, new_spacing) -> np.ndarray:
    """the reference's compute_new_shape: int(round(old_spacing / new_spacing * old_shape)) per axis"""
    assert len(old_spacing) == len(old_shape)
    assert len(old_shape) == len(new_spacing)
    return np.array([int(round(i / j * k)) for i, j, k in zip(old_spacing, new_spacing, old_shape)])


def resample_case(data: torch.Tensor, seg: torch.Tensor | None, new_shape):
    """(data (C, *new_shape) fp32, seg (1, *new_shape) int8 or None): resample_data_or_seg_to_shape with
    force_separate_z=False -- skimage resize(order=3, mode='edge', anti_aliasing=False) of each channel clipped to its range,
    resize_segmentation(order=1) of the labels.  The inputs come back unchanged when the shape does not change.  Raises
    ValueError for a source axis below 4 voxels, an empty target axis or a volume of 2^31 voxels or more.  No
    synchronisation."""
    _lib.require_cuda(data, seg)
    new_shape = tuple(int(v) for v in new_shape)
    src = tuple(data.shape[1:])
    if len(new_shape) != 3 or data.dim() != 4:
        raise ValueError(f"data must be (C, D, H, W) and new_shape three axes, got {tuple(data.shape)} and {new_shape}")
    if new_shape == src:
        return data, seg
    if min(src) < 4 or min(new_shape) < 1:
        raise ValueError(f"resampling {src} -> {new_shape}: source axes need at least 4 voxels and target axes at least 1")
    if math.prod(v + 4 for v in src) >= 2 ** 31 or math.prod(new_shape) >= 2 ** 31:
        raise ValueError(f"resampling {src} -> {new_shape}: source (with a 2-voxel border) and target are limited to 2^31 - 1 "
                         f"voxels")
    data = data.to(torch.float32).contiguous()
    C, dev = data.shape[0], data.device
    st = _stats(data)
    coef = torch.empty((C, math.prod(v + 4 for v in src)), dtype=torch.float32, device=dev)
    out = torch.empty((C,) + new_shape, dtype=torch.float32, device=dev)
    A.prefilter([A.prefilter_job(data[c], coef[c], src, _lib.AUG_EDGE) for c in range(C)], dev)
    A.resample([A.resample_job(coef[c], out[c], src, new_shape, 3, zoom=True, clip=st[c]) for c in range(C)], dev)
    return out, (None if seg is None else _label_resize(seg.reshape(src), new_shape))


def _label_resize(seg: torch.Tensor, new_shape) -> torch.Tensor:
    """(1, *new_shape) int8: resize_segmentation(order=1) of a (d, h, w) int8 label volume"""
    s = seg.to(torch.int8).contiguous()
    out = torch.empty((1,) + tuple(new_shape), dtype=torch.int8, device=s.device)
    _call("smb_prep_label_resize", _lib.PrepLabelResizeArgs(s.data_ptr(), out.data_ptr(), *s.shape, *new_shape), s.device)
    return out


# ---- ordered compaction and gathers -------------------------------------------------------------------------------------------
def _label_set(labels) -> ctypes.Array:
    s = (ctypes.c_uint32 * 8)()
    for l in labels:
        if l == int(l) and -128 <= int(l) <= 127:                    # other values match no int8 voxel
            u = int(l) & 255
            s[u >> 5] |= 1 << (u & 31)
    return s


FOREGROUND = tuple(range(1, 128))                                      # seg > 0 of int8 labels


class _Compaction:
    """jobs over one int8 volume, one per label set: counts on the device after __init__, indices after write()"""

    def __init__(self, vol: torch.Tensor, sets: list):
        self.vol = vol.contiguous().reshape(-1)
        self.dev, self.n = vol.device, self.vol.numel()
        J = len(sets)
        self.chunk = torch.empty((max(J, 1), -(-self.n // _lib.PREP_CHUNK)), dtype=torch.int32, device=self.dev)
        self.counts = torch.zeros(J, dtype=torch.int64, device=self.dev)
        self.sets = [_label_set(s) for s in sets]
        A._run("smb_prep_count", _lib.PrepCompactJob, self._jobs([None] * J), self.dev)

    def _jobs(self, index):
        return [_lib.PrepCompactJob(self.vol.data_ptr(), self.chunk[j].data_ptr(), self.counts.data_ptr() + 8 * j, _lib.ptr(index[j]),
                                    self.n, self.sets[j]) for j in range(len(self.sets))]

    def write(self, counts) -> list:
        """int32 linear indices (raster order) per job, sized by the host copy of the counts"""
        index = [torch.empty(max(int(k), 1), dtype=torch.int32, device=self.dev) for k in counts]
        A._run("smb_prep_compact", _lib.PrepCompactJob, self._jobs(index), self.dev)
        return [ix[:int(k)] for ix, k in zip(index, counts)]


def _rows(index: torch.Tensor, select: torch.Tensor, shape) -> torch.Tensor:
    """(k, 4) int64 rows (0, z, y, x) of index[select] in a (d, h, w) volume"""
    rows = torch.empty((select.numel(), 4), dtype=torch.int64, device=index.device)
    ix = index if index.numel() else torch.zeros(1, dtype=torch.int32, device=index.device)
    _call("smb_prep_gather", _lib.PrepGatherArgs(index=ix.data_ptr(), select=select.data_ptr(), rows=rows.data_ptr(),
                                                 n=select.numel(), d=shape[0], h=shape[1], w=shape[2]), index.device)
    return rows


def _values(index: torch.Tensor, data: torch.Tensor, select: torch.Tensor | None, n: int) -> torch.Tensor:
    """(C, n) fp32: channel c at index[select[c, i]] (index[i] without select) of a contiguous (C, D, H, W) case"""
    C = data.shape[0]
    vals = torch.empty((C, n), dtype=torch.float32, device=data.device)
    ix = index if index.numel() else torch.zeros(1, dtype=torch.int32, device=data.device)
    _call("smb_prep_gather", _lib.PrepGatherArgs(index=ix.data_ptr(), select=_lib.ptr(select), data=data.data_ptr(),
                                                 values=vals.data_ptr(), n=n, channel_stride=data[0].numel(),
                                                 select_channel_stride=0 if select is None else select.shape[-1],
                                                 channels=C), data.device)
    return vals


def _location_draws(counts, seed: int) -> list:
    """_sample_foreground_locations' draws: one RandomState over the labels in order, none for an empty label"""
    rs = np.random.RandomState(seed)
    out = []
    for n in counts:
        n = int(n)
        if n == 0:
            out.append(None)
            continue
        k = max(min(10000, n), int(np.ceil(n * 0.01)))
        out.append(rs.choice(n, k, replace=False))
    return out


def _intensity_draws(n_fg: int, channels: int, seed: int, num_samples: int) -> list:
    """collect_foreground_intensities' draws: one RandomState over the channels, none without foreground"""
    rs = np.random.RandomState(seed)
    return [rs.choice(n_fg, num_samples, replace=True) if n_fg > 0 else None for _ in range(channels)]


def _percentile_ranks(n: int, q: float):
    """numpy.percentile(method='linear') of n float32 values, whose virtual index numpy computes in float32:
    (lower rank, upper rank, gamma)"""
    f = np.float32
    vi = f(f(q / 100) * f(n - 1))
    lo = int(np.floor(vi))
    return min(lo, n - 1), min(lo + 1, n - 1), f(vi - f(lo))


def _lerp(a, b, t):
    """numpy's _lerp in float32"""
    f = np.float32
    a, b = f(a), f(b)
    d = f(b - a)
    return f(b - d * f(f(1) - t)) if t >= 0.5 else f(a + d * t)


_STAT_Q = (50.0, 99.5, 0.5)


class _Intensities:
    """foreground intensities of a raw case: the device work, then the host assembly from one readback"""

    def __init__(self, data, seg8, n_fg: int, seed: int, num_samples: int):
        C, dev = data.shape[0], data.device
        self.n_fg, self.C = n_fg, C
        comp = _Compaction(seg8, [FOREGROUND])
        fg = comp.write([n_fg])[0]
        self.samples = self.stats = self.picks = None
        if n_fg == 0:
            return
        draws = _intensity_draws(n_fg, C, seed, num_samples)
        sel = torch.from_numpy(np.stack(draws)).to(dev)
        self.samples = _values(fg, data, sel, num_samples)
        vals = _values(fg, data, None, n_fg)
        self.stats = _stats(vals)
        ranks = []
        for q in _STAT_Q:
            lo, hi, _ = _percentile_ranks(n_fg, q)
            ranks += [lo, hi]
        ranks += [(n_fg - 1) // 2, n_fg // 2]                           # the median's middle pair
        ordered = torch.sort(vals, dim=1).values
        self.picks = ordered[:, torch.tensor(ranks, device=dev)]

    def tensors(self) -> list:
        return [] if self.n_fg == 0 else [self.samples, self.stats, self.picks]

    def result(self, host: list):
        """(intensities_per_channel, intensity_statistics_per_channel) from the host copies of tensors()"""
        if self.n_fg == 0:
            nan = float("nan")
            return [[] for _ in range(self.C)], [dict(mean=nan, median=nan, min=nan, max=nan, percentile_99_5=nan,
                                                      percentile_00_5=nan) for _ in range(self.C)]
        samples, st, picks = host
        stats = []
        for c in range(self.C):
            p = picks[c]
            pct = {}
            for i, q in enumerate(_STAT_Q):
                pct[q] = _lerp(p[2 * i], p[2 * i + 1], _percentile_ranks(self.n_fg, q)[2])
            median = p[6] if self.n_fg % 2 else np.float32((p[6] + p[7]) / np.float32(2))   # numpy's float32 mean of the pair
            stats.append(dict(mean=float(st[c, 0] / self.n_fg), median=float(median), min=float(st[c, 2]), max=float(st[c, 3]),
                              percentile_99_5=float(pct[99.5]), percentile_00_5=float(pct[0.5])))
        return [samples[c] for c in range(self.C)], stats


def _locations(comp: _Compaction, counts, classes, seed: int, shape):
    index = comp.write(counts)
    draws = _location_draws(counts, seed)
    rows = [None if d is None else _rows(ix, torch.from_numpy(d).to(ix.device), shape) for ix, d in zip(index, draws)]
    return rows


def _class_key(c):
    return tuple(c) if isinstance(c, list) else c


def _class_labels(c):
    return tuple(c) if isinstance(c, (tuple, list)) else (c,)


def sample_foreground_locations(seg: torch.Tensor, classes, seed: int = 1234) -> dict:
    """the reference's _sample_foreground_locations on a (1, d, h, w) or (d, h, w) int8 device seg: {label or region:
    (k, 4) int64 numpy rows (0, z, y, x), or [] for an empty label}.  Two synchronisations (counts, rows)."""
    _lib.require_cuda(seg)
    shape = tuple(seg.shape[-3:])
    classes = list(classes)
    comp = _Compaction(seg.to(torch.int8), [_class_labels(c) for c in classes])
    counts = _readback(comp.counts)[0]
    rows = _locations(comp, counts, classes, seed, shape)
    host = iter(_readback(*[r for r in rows if r is not None]))
    return {_class_key(c): ([] if r is None else next(host)) for c, r in zip(classes, rows)}


def foreground_intensities(data: torch.Tensor, seg: torch.Tensor, seed: int = 1234, num_samples: int = 10000):
    """the reference's collect_foreground_intensities on a raw (C, D, H, W) case and its labels (foreground: seg > 0):
    (per-channel samples drawn with replacement, per-channel statistics dicts).  Two synchronisations."""
    data = _data(data)
    seg = _seg(seg, data.shape[1:])
    if seg is None:
        raise ValueError("foreground_intensities needs a seg")
    _, seg8, rec = _analyse(data, seg)
    rec = _readback(rec)[0]
    _check(rec, True)
    fi = _Intensities(data, seg8, int(rec[6]), seed, num_samples)
    return fi.result(_readback(*fi.tensors()))


def preprocess_case(data: torch.Tensor, seg: torch.Tensor | None = None, spacing=(1.0, 1.0, 1.0), target_spacing=(1, 1, 1),
                    all_labels=(1, 2, 3), name=None, normalization: str = "zscore", intensity_properties=None):
    """(data (C, d, h, w) fp32, seg (1, d, h, w) int8, properties) of one raw case, as the reference's read_data +
    run_case_npy on the device: MultiModalityPreprocessor's (ZScoreNormalization, normalization="zscore") or
    DefaultPreprocessor's (CTNormalization, normalization="ct", with the dataset's intensity_properties).

    data      CUDA (C, D, H, W); other dtypes are converted to fp32
    seg       CUDA (1, D, H, W) or (D, H, W) integer labels in [0, 127] (integer or integral float dtype), or None
    spacing   SimpleITK (x, y, z) order, as properties["spacing"]
    target_spacing  the reference's output_spacing (array order)
    all_labels      labels or regions (tuples / lists of labels) for class_locations
    intensity_properties  normalization="ct" only: {"0": {mean, std, percentile_00_5, percentile_99_5}, ...} per channel,
                    plan.plan_dataset(...)["intensity_statistics_per_channel"]

    The output data and seg stay on the device; class_locations are numpy int64 (k, 4) arrays.  Makes exactly
    READBACKS_PER_CASE (3) synchronisations: the mask record, the label counts, the drawn rows and intensity statistics."""
    if normalization not in ("zscore", "ct"):
        raise ValueError(f"normalization must be 'zscore' or 'ct', got {normalization!r}")
    if normalization == "ct" and intensity_properties is None:
        raise ValueError("normalization='ct' needs the dataset's intensity_properties")
    data = _data(data)
    seg_in = _seg(seg, data.shape[1:])
    C, D, H, W = data.shape
    mask, seg8, rec = _analyse(data, seg_in)
    filled = fill_holes(mask)
    rec = _readback(rec)[0]                                                               # readback 1
    _check(rec, seg_in is not None)
    bbox = _bbox(rec)
    fi = _Intensities(data, seg8, int(rec[6]), 1234, 10000) if seg_in is not None else None
    crop, cseg = _crop(data, filled, seg8, bbox)
    crop_shape = tuple(crop.shape[1:])
    original_spacing_trans = list(spacing)[::-1]
    new_shape = compute_new_shape(crop_shape, original_spacing_trans, target_spacing)
    norm = ct_normalize(crop, intensity_properties) if normalization == "ct" else zscore(crop)[0]
    out, oseg = resample_case(norm, cseg, new_shape)
    classes = list(all_labels)
    comp = _Compaction(oseg, [_class_labels(c) for c in classes])
    counts = _readback(comp.counts)[0]                                                    # readback 2
    rows = _locations(comp, counts, classes, 1234, tuple(oseg.shape[1:]))
    live = [r for r in rows if r is not None]
    host = _readback(*live, *([] if fi is None else fi.tensors()))                       # readback 3
    it = iter(host[:len(live)])
    class_locations = {_class_key(c): ([] if r is None else next(it)) for c, r in zip(classes, rows)}
    if fi is None:
        intensities, statistics = [], []
    else:
        intensities, statistics = fi.result(host[len(live):])
    properties = {
        "spacing": tuple(spacing),
        "raw_size": (D, H, W),
        "name": name,
        "intensities_per_channel": intensities,
        "intensity_statistics_per_channel": statistics,
        "original_spacing_trans": original_spacing_trans,
        "target_spacing_trans": list(target_spacing),
        "shape_before_cropping": (D, H, W),
        "bbox_used_for_cropping": bbox,
        "shape_after_cropping_before_resample": crop_shape,
        "shape_after_resample": new_shape,
        "class_locations": class_locations,
    }
    return out, oseg, properties
