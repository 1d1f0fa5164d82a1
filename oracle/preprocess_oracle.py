"""CPU restatement (numpy / scipy) of the reference's case preprocessing -- MultiModalityPreprocessor.read_data's foreground
intensities and DefaultPreprocessor.run_case_npy with ZScoreNormalization -- for segmamba_b200/preprocess.py.  Test
infrastructure only: the product never imports it.

Each function follows the reference function it is named after; skimage's resize is augment_oracle.resize, and
batchgenerators' resize_segmentation(order=1) is the order-1 resize of every label's indicator, the label winning where it is
>= 0.5, later (higher) labels overwriting earlier ones.
"""
from __future__ import annotations

import numpy as np
import scipy.ndimage as ndi

from oracle.augment_oracle import resize


def create_nonzero_mask(data: np.ndarray) -> np.ndarray:
    mask = np.zeros(data.shape[1:], dtype=bool)
    for c in range(data.shape[0]):
        mask |= data[c] != 0
    return ndi.binary_fill_holes(mask)


def get_bbox_from_mask(mask: np.ndarray) -> list:
    """[[lo, hi + 1]] per axis; ValueError for an all-zero mask"""
    idx = np.argwhere(mask)
    if len(idx) == 0:
        raise ValueError("the case has no nonzero voxel")
    return [[int(idx[:, a].min()), int(idx[:, a].max()) + 1] for a in range(mask.ndim)]


def crop_to_nonzero(data: np.ndarray, seg: np.ndarray | None = None, nonzero_label: int = -1):
    mask = create_nonzero_mask(data)
    bbox = get_bbox_from_mask(mask)
    sl = tuple(slice(a, b) for a, b in bbox)
    data = data[(slice(None),) + sl]
    m = mask[sl][None]
    if seg is not None:
        seg = seg[(slice(None),) + sl].copy()
        seg[(seg == 0) & ~m] = nonzero_label
    else:
        seg = m.astype(np.int8)
        seg[seg == 0] = nonzero_label
        seg[seg > 0] = 0
    return data, seg, bbox


def zscore(image: np.ndarray) -> np.ndarray:
    """ZScoreNormalization(use_mask_for_norm=False).run of one channel, in float32 exactly as numpy computes it"""
    image = image.astype(np.float32)
    mean = image.mean()
    std = image.std()
    return (image - mean) / (max(std, 1e-8))


def compute_new_shape(old_shape, old_spacing, new_spacing) -> np.ndarray:
    return np.array([int(round(i / j * k)) for i, j, k in zip(old_spacing, new_spacing, old_shape)])


def resize_segmentation(seg: np.ndarray, new_shape):
    """(labels, distance of the nearest indicator to 0.5 per voxel, for tie tolerance)"""
    out = np.zeros(tuple(new_shape), dtype=seg.dtype)
    near = np.full(tuple(new_shape), np.inf)
    for c in np.unique(seg):
        ind = resize((seg == c).astype(float), new_shape, 1)
        out[ind >= 0.5] = c
        near = np.minimum(near, np.abs(ind - 0.5))
    return out, near


def resample(data: np.ndarray, seg: np.ndarray, new_shape):
    """resample_data_or_seg_to_shape (force_separate_z=False) of the data (order 3) and the seg (order 1); (data, seg, near)"""
    new_shape = tuple(int(v) for v in new_shape)
    if new_shape == tuple(data.shape[1:]):
        return data, seg, None
    d = np.stack([resize(data[c].astype(float), new_shape, 3) for c in range(data.shape[0])]).astype(data.dtype)
    s, near = resize_segmentation(seg[0].astype(float), new_shape)
    return d, s[None].astype(seg.dtype), near


def sample_foreground_locations(seg: np.ndarray, classes_or_regions, seed: int = 1234) -> dict:
    rs = np.random.RandomState(seed)
    out = {}
    for c in classes_or_regions:
        k = c if not isinstance(c, list) else tuple(c)
        if isinstance(c, (tuple, list)):
            mask = seg == c[0]
            for cc in c[1:]:
                mask = mask | (seg == cc)
        else:
            mask = seg == c
        locs = np.argwhere(mask)
        if len(locs) == 0:
            out[k] = []
            continue
        n = max(min(10000, len(locs)), int(np.ceil(len(locs) * 0.01)))
        out[k] = locs[rs.choice(len(locs), n, replace=False)]
    return out


def collect_foreground_intensities(seg: np.ndarray, images: np.ndarray, seed: int = 1234, num_samples: int = 10000):
    rs = np.random.RandomState(seed)
    fg = seg[0] > 0
    samples, stats = [], []
    for i in range(len(images)):
        px = images[i][fg]
        n = len(px)
        samples.append(rs.choice(px, num_samples, replace=True) if n > 0 else [])
        stats.append({"mean": np.mean(px) if n else np.nan, "median": np.median(px) if n else np.nan,
                      "min": np.min(px) if n else np.nan, "max": np.max(px) if n else np.nan,
                      "percentile_99_5": np.percentile(px, 99.5) if n else np.nan,
                      "percentile_00_5": np.percentile(px, 0.5) if n else np.nan})
    return samples, stats


def preprocess_case(data: np.ndarray, seg: np.ndarray | None, spacing, target_spacing=(1, 1, 1), all_labels=(1, 2, 3), name=None):
    """(data, seg int8, properties, near): read_data (float32 data and labels) + run_case_npy; near is the tie distance of
    the resampled labels (None when nothing was resampled)"""
    data = np.asarray(data, np.float32)
    if seg is not None:
        seg = np.asarray(seg, np.float32).reshape((1,) + data.shape[1:])
        inten, istats = collect_foreground_intensities(seg, data)
    else:
        inten, istats = [], []
    props = {"spacing": tuple(spacing), "raw_size": data.shape[1:], "name": name, "intensities_per_channel": inten,
             "intensity_statistics_per_channel": istats}
    props["original_spacing_trans"] = list(spacing)[::-1]
    props["target_spacing_trans"] = list(target_spacing)
    props["shape_before_cropping"] = data.shape[1:]
    data, seg, bbox = crop_to_nonzero(data, seg)
    props["bbox_used_for_cropping"] = bbox
    props["shape_after_cropping_before_resample"] = data.shape[1:]
    new_shape = compute_new_shape(data.shape[1:], props["original_spacing_trans"], target_spacing)
    data = np.stack([zscore(data[c]) for c in range(data.shape[0])])
    data, seg, near = resample(data, seg, new_shape)
    props["shape_after_resample"] = new_shape
    props["class_locations"] = sample_foreground_locations(seg, list(all_labels))
    return data, seg.astype(np.int8), props, near
