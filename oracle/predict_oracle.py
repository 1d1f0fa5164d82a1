"""Test-only restatement of what the reference does on the CPU after the sliding window: Predictor.predict_raw_probability
(torch's trilinear interpolate per channel in fp32, stored as fp16), argmax over classes, convert_labels_dim0, and
predict_noncrop_probability; and the connected-component post-processing of large_connected_domain in scipy
(skimage is not installed; scipy's 6-connected label numbers components the same way, in raster order of their first voxel)."""
from __future__ import annotations

import numpy as np
import torch
from scipy import ndimage

from .metrics_oracle import BRATS_REGIONS, regions_of

STRUCT6 = ndimage.generate_binary_structure(3, 1)


def resampled_scores(logits: torch.Tensor, crop_shape) -> torch.Tensor:
    """(C, d, h, w) logits -> (C, d', h', w') fp16 scores, channel by channel as predict_raw_probability does (CPU fp32)."""
    x = logits.detach().to("cpu", torch.float32)
    out = torch.zeros((x.shape[0],) + tuple(int(v) for v in crop_shape), dtype=torch.half)
    for c in range(x.shape[0]):
        out[c] = torch.nn.functional.interpolate(x[c][None, None], mode="trilinear", size=tuple(out.shape[1:]))[0, 0]
    return out


def uncrop(pred: np.ndarray, bbox_lo, crop_shape, full_shape) -> np.ndarray:
    """predict_noncrop_probability: (..., d', h', w') -> (..., D0, H0, W0) uint8, zero outside the box."""
    out = np.zeros(pred.shape[:-3] + tuple(full_shape), dtype=np.uint8)
    z, y, x = bbox_lo
    cd, ch, cw = crop_shape
    out[..., z:z + cd, y:y + ch, x:x + cw] = pred
    return out


def restore(logits: torch.Tensor, crop_shape, bbox_lo, full_shape, regions=BRATS_REGIONS) -> np.ndarray:
    """(C, d, h, w) logits -> uint8 (R, D0, H0, W0) region masks, or the (D0, H0, W0) label map for regions=None."""
    lab = resampled_scores(logits, crop_shape).argmax(dim=0).numpy()
    pred = lab.astype(np.uint8) if regions is None else regions_of(lab, regions).astype(np.uint8)
    return uncrop(pred, bbox_lo, crop_shape, full_shape)


def label(mask: np.ndarray):
    """scipy.ndimage.label with 6-connectivity: (int32 labels, count)."""
    lab, n = ndimage.label(np.asarray(mask, bool), structure=STRUCT6)
    return lab.astype(np.int32), int(n)


def fill_holes(mask: np.ndarray) -> np.ndarray:
    return ndimage.binary_fill_holes(np.asarray(mask, bool))


def largest_connected_domain(mask: np.ndarray) -> np.ndarray:
    """large_connected_domain with the tie rule made explicit: a stable argsort's last entry (the highest label of the
    largest size); an empty mask gives an empty result."""
    lab, n = label(mask)
    if n == 0:
        return np.zeros(lab.shape, bool)
    sizes = np.bincount(lab.ravel(), minlength=n + 1)[1:]
    keep = lab == (np.argsort(sizes, kind="stable")[-1] + 1)
    return fill_holes(keep)
