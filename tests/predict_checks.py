"""Shared checks of the case-prediction kernels (segmamba_b200/predict.py) against oracle/predict_oracle.py, for the emulator
and the GPU."""
import numpy as np
import torch

from metrics_checks import nested_labels
from oracle import metrics_oracle as morc
from oracle import predict_oracle as orc
from segmamba_b200 import predict as P

FAMILIES = ("bernoulli", "serpentine", "checkerboard", "full", "empty", "brats")


def serpentine(shape) -> np.ndarray:
    """one simple 6-connected path through the whole volume: rows at even (z, y), walked in alternating x direction, joined
    by single voxels at odd y (inside a layer) or odd z (between layers, whose row order is reversed)."""
    D, H, W = shape
    m = np.zeros(shape, bool)
    rows = []
    for k, z in enumerate(range(0, D, 2)):
        ys = list(range(0, H, 2))
        rows += [(z, y) for y in (ys[::-1] if k % 2 else ys)]
    for i, (z, y) in enumerate(rows):
        m[z, y, :] = True
        if i:
            z0, y0 = rows[i - 1]
            x = W - 1 if i % 2 else 0                                   # where row i - 1 ended and row i starts
            m[(z0 + z) // 2, (y0 + y) // 2, x] = True
    return m


def family(name, shape, seed=0) -> np.ndarray:
    """(N, D, H, W) bool masks of one family (N = 3 for the BraTS regions plus the edema shell, else 1 or 2)."""
    rng = np.random.default_rng(seed)
    if name == "bernoulli":                                             # near the site-percolation threshold
        return rng.random((2,) + tuple(shape)) < 0.31
    if name == "serpentine":
        return serpentine(shape)[None]
    if name == "checkerboard":
        g = np.indices(shape).sum(0)
        return (g % 2 == 0)[None]
    if name == "full":
        return np.ones((1,) + tuple(shape), bool)
    if name == "empty":
        return np.zeros((1,) + tuple(shape), bool)
    lab = nested_labels(shape, seed=seed)[0]
    return np.concatenate([morc.regions_of(lab), (lab == 2)[None]])     # TC, WT, ET and the edema shell around the core


def check_cc(masks: np.ndarray, device) -> list:
    """mismatches of label_components / fill_holes / largest_connected_domain against scipy, one batched call each."""
    t = torch.from_numpy(masks).to(device)
    lab, cnt = P.label_components(t)
    fill = P.fill_holes(t).cpu().numpy()
    big = P.largest_connected_domain(t).cpu().numpy()
    lab, cnt = lab.cpu().numpy(), cnt.cpu().numpy()
    bad = []
    for b in range(masks.shape[0]):
        rl, rc = orc.label(masks[b])
        if not np.array_equal(lab[b], rl):
            bad.append((b, "labels", int((lab[b] != rl).sum())))
        if int(cnt[b]) != rc:
            bad.append((b, "count", int(cnt[b]), rc))
        if not np.array_equal(fill[b], orc.fill_holes(masks[b])):
            bad.append((b, "fill_holes"))
        if not np.array_equal(big[b], orc.largest_connected_domain(masks[b])):
            bad.append((b, "largest"))
    return bad


def case_properties(crop, lo, full):
    return {"shape_after_cropping_before_resample": list(crop), "shape_before_cropping": list(full),
            "bbox_used_for_cropping": [[lo[i], lo[i] + crop[i]] for i in range(3)]}


def logits_like(shape, C=4, seed=0) -> torch.Tensor:
    """smooth-ish (C, d, h, w) fp32 logits: nested-label one-hot scaled, plus noise, so the argmax has structure and ties."""
    rng = np.random.default_rng(seed)
    lab = nested_labels(shape, seed=seed)[0]
    x = 2.0 * np.eye(C, dtype=np.float32)[lab].transpose(3, 0, 1, 2) + rng.standard_normal((C,) + tuple(shape)).astype(np.float32)
    return torch.from_numpy(x)


def near_ties(logits: torch.Tensor, crop) -> np.ndarray:
    """voxels of the crop whose two best oracle fp16 scores are within one fp16 ulp of each other."""
    s = orc.resampled_scores(logits, crop).float().numpy()
    top = np.sort(s, axis=0)
    a, b = top[-1], top[-2]
    return (a - b) <= np.spacing(np.abs(a).astype(np.float16)).astype(np.float32)


def restore_variants(logits: torch.Tensor):
    """(name, tensor) of the layouts and dtypes restore_case accepts, each exactly representing `logits` where possible."""
    yield "f32", logits
    yield "f32_cl", logits[None].contiguous(memory_format=torch.channels_last_3d)
    yield "f16", logits.half()
    yield "bf16_cl", logits.bfloat16()[None].contiguous(memory_format=torch.channels_last_3d)


def check_restore(logits: torch.Tensor, crop, lo, full, device) -> dict:
    """per variant and output form: the number of voxels that differ from the oracle, and the near-tie voxels among them."""
    props = case_properties(crop, lo, full)
    ties = orc.uncrop(near_ties(logits, crop).astype(np.uint8), lo, crop, full).astype(bool)
    out = {}
    for name, t in restore_variants(logits):
        ref_in = t.float().reshape(t.shape[-4:]) if t.dim() == 5 else t.float()
        for regions in (P.BRATS_REGIONS, None):
            ref = orc.restore(ref_in, crop, lo, full, regions)
            got = P.restore_case(t.to(device), props, regions=regions).cpu().numpy()
            diff = got != ref
            if regions is not None:
                diff = diff.any(0)
            out[(name, regions is None)] = (int(diff.sum()), int((diff & ~ties).sum()))
    return out
