"""Case prediction on the GPU after the sliding window (csrc/predict.cu): what the reference's Predictor and 4_predict.py do on
the CPU between the blended logits and the saved segmentation.

  * restore_case: the trilinear resample of every class channel to `shape_after_cropping_before_resample`
    (F.interpolate(mode="trilinear", align_corners=False) in fp32, stored as fp16 as predict_raw_probability does), the
    argmax over classes (first maximum; a NaN is the maximum), the region conversion (TC / WT / ET for BRATS_REGIONS) and the
    copy into a zeroed `shape_before_cropping` volume at `bbox_used_for_cropping` (predict_noncrop_probability), in one pass
    that never materialises the resampled probabilities.
  * label_components: scipy.ndimage.label with 6-connectivity (generate_binary_structure(3, 1), skimage's connectivity=1),
    numbering included: component k is the k-th in raster order of its first voxel.
  * fill_holes: scipy.ndimage.binary_fill_holes with its default structure.
  * largest_connected_domain: the reference's large_connected_domain -- the largest 6-connected component, holes filled.
    Ties between equally large components go to the highest label (what a stable argsort(...)[-1] returns; the reference's
    default-kind argsort leaves the order of ties unspecified).  An empty mask gives an empty result (the reference raises
    IndexError).

Everything stays on the device; no call synchronises with the host, launch sizes depend on shapes only, and results are
bitwise deterministic.
"""
from __future__ import annotations

import ctypes
import operator

import numpy as np
import torch

from . import _lib
from .metrics import BRATS_REGIONS, _lut

__all__ = ["BRATS_REGIONS", "restore_case", "label_components", "fill_holes", "largest_connected_domain", "case_geometry"]


def _as_int(v, what: str) -> int:
    if isinstance(v, torch.Tensor):
        if v.numel() != 1:
            raise ValueError(f"{what}: expected one value, got a tensor of shape {tuple(v.shape)}")
        return int(v.reshape(-1)[0].item())
    if isinstance(v, np.ndarray):
        if v.size != 1:
            raise ValueError(f"{what}: expected one value, got an array of shape {v.shape}")
        v = v.reshape(-1)[0]
    try:
        return operator.index(v)
    except TypeError:
        raise ValueError(f"{what}: expected an integer, got {v!r}") from None


def _triple(v, what: str) -> tuple:
    if isinstance(v, torch.Tensor) and v.numel() == 3:
        v = v.reshape(-1).tolist()
    v = list(v)
    if len(v) != 3:
        raise ValueError(f"{what}: expected three axes, got {len(v)}")
    return tuple(_as_int(x, what) for x in v)


def case_geometry(properties) -> tuple:
    """(crop_shape, bbox_lower, shape_before_cropping) from the reference's per-case properties dict, whose values may be
    ints, numpy ints or one-element tensors (as a DataLoader collates them).  Raises ValueError when the bbox does not lie
    inside shape_before_cropping or its extent differs from shape_after_cropping_before_resample."""
    for k in ("shape_after_cropping_before_resample", "shape_before_cropping", "bbox_used_for_cropping"):
        if k not in properties:
            raise ValueError(f"properties lack {k!r}")
    crop = _triple(properties["shape_after_cropping_before_resample"], "shape_after_cropping_before_resample")
    full = _triple(properties["shape_before_cropping"], "shape_before_cropping")
    bbox = list(properties["bbox_used_for_cropping"])
    if len(bbox) != 3:
        raise ValueError(f"bbox_used_for_cropping: expected three axes, got {len(bbox)}")
    lo, hi = [], []
    for ax, pair in enumerate(bbox):
        pair = list(pair.reshape(-1)) if isinstance(pair, (torch.Tensor, np.ndarray)) else list(pair)
        if len(pair) != 2:
            raise ValueError(f"bbox_used_for_cropping[{ax}]: expected [lower, upper], got {pair!r}")
        lo.append(_as_int(pair[0], "bbox_used_for_cropping"))
        hi.append(_as_int(pair[1], "bbox_used_for_cropping"))
    for ax in range(3):
        if min(crop[ax], full[ax]) <= 0:
            raise ValueError(f"axis {ax}: shapes must be positive, got crop {crop} and original {full}")
        if not 0 <= lo[ax] <= hi[ax] <= full[ax]:
            raise ValueError(f"axis {ax}: bbox [{lo[ax]}, {hi[ax]}) is not inside shape_before_cropping {full}")
        if hi[ax] - lo[ax] != crop[ax]:
            raise ValueError(f"axis {ax}: bbox extent {hi[ax] - lo[ax]} differs from the crop shape {crop[ax]}")
    return crop, tuple(lo), full


def restore_case(logits: torch.Tensor, properties, regions=BRATS_REGIONS, postprocess: bool = False) -> torch.Tensor:
    """Blended logits (C, d, h, w) or (1, C, d, h, w) of one case, fp32 / bf16 / fp16, contiguous or channels_last_3d ->
    uint8 region masks (R, D0, H0, W0) in the geometry before cropping, or with regions=None the uint8 label map
    (D0, H0, W0).  postprocess=True applies largest_connected_domain to each region mask in 3-D; the reference's
    save_to_nii(postprocess=True) would instead label the stacked (R, D0, H0, W0) array as one 4-D volume (no reference
    script enables it), so masks are post-processed per region here.  Requires regions."""
    _lib.require_cuda(logits)
    if logits.dim() == 5:
        if logits.shape[0] != 1:
            raise ValueError(f"restore_case takes one case, got batch {logits.shape[0]}")
        logits = logits[0]
    if logits.dim() != 4:
        raise ValueError(f"logits must be (C, d, h, w) or (1, C, d, h, w), got {tuple(logits.shape)}")
    if logits.dtype not in (torch.float32, torch.float16, torch.bfloat16):
        raise TypeError(f"unsupported logit dtype {logits.dtype}")
    if postprocess and regions is None:
        raise ValueError("postprocess=True needs regions: the post-processing works on region masks")
    crop, lo, full = case_geometry(properties)
    C, d, h, w = logits.shape
    st = logits.stride()
    vs = st[3]
    if st[1:] != (h * w * vs, w * vs, vs) or vs <= 0:                  # neither NCDHW nor channels_last_3d
        logits = logits.contiguous()
        st, vs = logits.stride(), 1
    R = 0 if regions is None else len(regions)
    lut = _lut(regions if regions is not None else ((1,),))
    dev = logits.device
    out = torch.empty(((R,) if R else ()) + full, dtype=torch.uint8, device=dev)
    a = _lib.PredRestoreArgs(src=logits.data_ptr(), out=out.data_ptr(), class_stride=st[0], voxel_stride=vs,
                             dtype=_lib.dtype_code(logits.dtype), classes=C, regions=R, d=d, h=h, w=w,
                             cd=crop[0], ch=crop[1], cw=crop[2], z0=lo[0], y0=lo[1], x0=lo[2], D0=full[0], H0=full[1], W0=full[2])
    a.lut[:] = lut
    sp = _lib.stream_ptr(dev)
    _lib.call("smb_pred_restore", (C, d, h, w) + crop + full, lambda: _lib.lib().smb_pred_restore(ctypes.byref(a), sp), dev)
    if postprocess:
        _cc(out, _lib.PRED_LARGEST, out)
    return out


def _volumes(mask: torch.Tensor) -> torch.Tensor:
    _lib.require_cuda(mask)
    if mask.dim() not in (3, 4):
        raise ValueError(f"a mask must be (D, H, W) or (N, D, H, W), got {tuple(mask.shape)}")
    if mask.dtype == torch.bool:
        mask = mask.contiguous().view(torch.uint8)
    elif mask.dtype != torch.uint8:
        raise TypeError(f"masks must be bool or uint8, got {mask.dtype}")
    mask = mask.contiguous()
    if min(mask.shape) == 0:
        raise ValueError(f"empty volume {tuple(mask.shape)}")
    return mask


def _cc(mask: torch.Tensor, op: int, out: torch.Tensor, counts: torch.Tensor | None = None) -> None:
    """one smb_pred_cc call over the volumes of a (D, H, W) or (N, D, H, W) uint8 mask; `out` may alias `mask` for the
    mask-valued operations (the mask is read before the output is written)."""
    N = 1 if mask.dim() == 3 else mask.shape[0]
    D, H, W = mask.shape[-3:]
    dev = mask.device
    nbytes = int(_lib.lib().smb_pred_cc_workspace_bytes(N, D, H, W))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    a = _lib.PredCcArgs(mask.data_ptr(), out.data_ptr(), None if counts is None else counts.data_ptr(), ws.data_ptr(), nbytes,
                        N, D, H, W, op)
    sp = _lib.stream_ptr(dev)
    _lib.call("smb_pred_cc", (op, N, D, H, W), lambda: _lib.lib().smb_pred_cc(ctypes.byref(a), sp), dev)


def label_components(mask: torch.Tensor):
    """(labels, counts): int32 labels of the 6-connected components of each (D, H, W) volume (0: background, 1..count in
    raster order of each component's first voxel, as scipy.ndimage.label) and the int64 component count per volume (a
    0-d tensor for a single volume).  Both stay on the device."""
    m = _volumes(mask)
    labels = torch.empty(m.shape, dtype=torch.int32, device=m.device)
    counts = torch.empty((1 if m.dim() == 3 else m.shape[0],), dtype=torch.int64, device=m.device)
    _cc(m, _lib.PRED_LABEL, labels, counts)
    return labels, (counts[0] if m.dim() == 3 else counts)


def fill_holes(mask: torch.Tensor) -> torch.Tensor:
    """bool, same shape: scipy.ndimage.binary_fill_holes of each (D, H, W) volume -- every background component that does
    not touch the volume boundary (6-connectivity) becomes foreground."""
    m = _volumes(mask)
    out = torch.empty(m.shape, dtype=torch.bool, device=m.device)
    _cc(m, _lib.PRED_FILL_HOLES, out)
    return out


def largest_connected_domain(mask: torch.Tensor) -> torch.Tensor:
    """bool, same shape: per (D, H, W) volume, the largest 6-connected component with its holes filled (the reference's
    large_connected_domain); ties go to the highest label, an empty mask stays empty."""
    m = _volumes(mask)
    out = torch.empty(m.shape, dtype=torch.bool, device=m.device)
    _cc(m, _lib.PRED_LARGEST, out)
    return out
