"""Shared cases and checks of the CT preprocessing path (preprocess_case(normalization="ct")) against
oracle/ct_preprocess_oracle.py, for the emulator, the GPU and the fixture generator."""
import numpy as np
import torch

from oracle import ct_preprocess_oracle as cto
from oracle import preprocess_oracle as orc
from preprocess_checks import compare_intensities, compare_locations
from segmamba_b200 import preprocess as PP


def ct_like(shape, seed, labels=True):
    """(data (1, D, H, W) float32, seg (1, D, H, W) float32 or None): a CT slab on a circular field of view"""
    rng = np.random.default_rng(seed)
    g = np.meshgrid(*[(np.arange(n) + 0.5) / n - 0.5 for n in shape], indexing="ij", sparse=True)
    fov = np.sqrt(g[1] ** 2 + g[2] ** 2) < 0.46
    body = np.sqrt((g[1] / 0.36) ** 2 + (g[2] / 0.4) ** 2) < 1.0
    data = np.where(fov, -1000.0, 0.0) + np.where(body, 1000.0 + rng.normal(40.0, 120.0, shape), 0.0)
    data = np.where(fov, np.round(np.clip(data, -1024, 3071)), 0.0).astype(np.float32)
    if not labels:
        return data[None], None
    t = np.sqrt((g[0] / 0.5) ** 2 + ((g[1] - 0.05) / 0.2) ** 2 + ((g[2] + 0.05) / 0.25) ** 2)
    seg = np.zeros(shape, np.float32)
    seg[(t < 1.0) & body] = 1
    seg[(t < 0.5) & body] = 2
    return data[None], seg[None]


def check_ct_case(data, seg, spacing, target, props, device, data_tol=1e-4):
    """(mismatches, label near-ties, device outputs) of preprocess_case(normalization="ct") against the oracle; labels may
    differ only where an oracle indicator lies within 1e-9 of 0.5"""
    d = torch.from_numpy(data).to(device)
    s = None if seg is None else torch.from_numpy(seg).to(device)
    od, os_, pp = PP.preprocess_case(d, s, spacing=spacing, target_spacing=target, all_labels=(1, 2), normalization="ct",
                                     intensity_properties=props)
    rd, rs, rp, near = cto.preprocess_case(data, seg, spacing, target, props, all_labels=(1, 2))
    od_h, os_h = od.cpu().numpy(), os_.cpu().numpy()
    bad = []
    for k in ("bbox_used_for_cropping", "shape_after_cropping_before_resample"):
        if list(np.asarray(pp[k]).ravel()) != list(np.asarray(rp[k]).ravel()):
            bad.append((k, pp[k], rp[k]))
    if od_h.shape != rd.shape or os_h.shape != rs.shape:
        return bad + [("shape", od_h.shape, rd.shape)], 0, (od, os_, pp)
    err = float(np.abs(od_h.astype(np.float64) - rd).max() / max(np.abs(rd).max(), 1e-30))
    if err > data_tol:
        bad.append(("data", err))
    diff = os_h != rs
    ties = int(diff.sum())
    if (diff & ((near[None] > 1e-9) if near is not None else True)).any():
        bad.append(("seg", ties))
    bad += compare_locations(pp["class_locations"], orc.sample_foreground_locations(os_h, [1, 2]))
    if seg is not None:
        bad += compare_intensities((pp["intensities_per_channel"], pp["intensity_statistics_per_channel"]),
                                   (rp["intensities_per_channel"], rp["intensity_statistics_per_channel"]))
    return bad, ties, (od, os_, pp)
