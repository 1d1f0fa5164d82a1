"""Shared cases and checks of the case-preprocessing path (segmamba_b200/preprocess.py) against oracle/preprocess_oracle.py,
for the emulator and the GPU."""
import numpy as np
import torch

from oracle import preprocess_oracle as orc
from segmamba_b200 import preprocess as PP


def brats_like(shape, channels=4, seed=0, labels=True):
    """(data (C, D, H, W) float32, seg (1, D, H, W) float32 or None): an ellipsoidal head on a zero background with an
    enclosed zero cavity, and nested labels 2 (edema) > 1 (core) > 3 (enhancing) inside.  Volumes too small for the head get
    a random nonzero pattern instead."""
    rng = np.random.default_rng(seed)
    D, H, W = shape
    g = np.stack(np.meshgrid(*[(np.arange(n) + 0.5) / n - 0.5 for n in shape], indexing="ij"))
    r = np.sqrt((g[0] / 0.42) ** 2 + (g[1] / 0.4) ** 2 + (g[2] / 0.38) ** 2)
    head = r < 1.0
    cavity = np.sqrt(((g[0] - 0.05) / 0.12) ** 2 + (g[1] / 0.1) ** 2 + ((g[2] + 0.1) / 0.1) ** 2) < 1.0
    if head.sum() < 8:
        head = rng.random(shape) < 0.6
        cavity = np.zeros(shape, bool)
    head &= ~cavity
    data = np.zeros((channels,) + tuple(shape), np.float32)
    for c in range(channels):
        data[c][head] = (rng.gamma(4.0, 100.0 * (c + 1), head.sum()) + 1).astype(np.float32)
    if not labels:
        return data, None
    t = np.sqrt(((g[0] + 0.1) / 0.2) ** 2 + ((g[1] - 0.1) / 0.22) ** 2 + ((g[2] - 0.05) / 0.18) ** 2)
    seg = np.zeros(shape, np.float32)
    seg[(t < 1.0) & head] = 2
    seg[(t < 0.6) & head] = 1
    seg[(t < 0.35) & head] = 3
    if seg.max() == 0:
        seg[head & (rng.random(shape) < 0.5)] = rng.integers(1, 4)
    return data, seg[None]


def dev_case(data, seg, device):
    return torch.from_numpy(data).to(device), (None if seg is None else torch.from_numpy(seg).to(device))


def compare_locations(got: dict, want: dict) -> list:
    bad = []
    for k in want:
        if k not in got:
            bad.append(("missing", k))
        elif isinstance(want[k], list) or isinstance(got[k], list):
            if not (isinstance(got[k], list) and len(got[k]) == 0 and isinstance(want[k], list) and len(want[k]) == 0):
                bad.append(("empty", k))
        elif got[k].dtype != np.int64 or not np.array_equal(got[k], want[k]):
            bad.append(("rows", k))
    if set(got) != set(want):
        bad.append(("keys", sorted(map(str, got)), sorted(map(str, want))))
    return bad


def compare_intensities(got, want, rel=1e-6) -> list:
    bad = []
    (gs, gst), (ws, wst) = got, want
    for c in range(len(ws)):
        if len(ws[c]) == 0:
            if len(gs[c]) != 0 or not all(np.isnan(v) for v in gst[c].values()):
                bad.append(("empty", c))
            continue
        if gs[c].dtype != np.float32 or not np.array_equal(gs[c], ws[c]):
            bad.append(("samples", c))
        for k in ("min", "max"):
            if gst[c][k] != float(wst[c][k]):
                bad.append((k, c, gst[c][k], float(wst[c][k])))
        for k in ("mean", "median", "percentile_99_5", "percentile_00_5"):
            w = float(wst[c][k])
            if abs(gst[c][k] - w) > rel * max(abs(w), 1e-30):
                bad.append((k, c, gst[c][k], w))
    return bad


def check_case(data, seg, spacing, target, device, data_tol=1e-5):
    """mismatches of preprocess_case against the oracle; labels may differ only where an oracle indicator lies within 1e-9
    of 0.5 (returned as the number of such voxels)"""
    d, s = dev_case(data, seg, device)
    od, os_, props = PP.preprocess_case(d, s, spacing=spacing, target_spacing=target, name="case")
    rd, rs, rp, near = orc.preprocess_case(data, seg, spacing, target, name="case")
    od, os_ = od.cpu().numpy(), os_.cpu().numpy()
    bad = []
    for k in ("spacing", "raw_size", "original_spacing_trans", "target_spacing_trans", "shape_before_cropping",
              "bbox_used_for_cropping", "shape_after_cropping_before_resample"):
        if list(np.asarray(props[k]).ravel()) != list(np.asarray(rp[k]).ravel()):
            bad.append((k, props[k], rp[k]))
    if not np.array_equal(props["shape_after_resample"], rp["shape_after_resample"]):
        bad.append(("shape_after_resample",))
    if od.shape != rd.shape or os_.shape != rs.shape or os_.dtype != np.int8:
        return bad + [("shape", od.shape, rd.shape, os_.shape, rs.shape)]
    err = float(np.abs(od.astype(np.float64) - rd).max() / max(np.abs(rd).max(), 1e-30))
    if err > data_tol:
        bad.append(("data", err))
    diff = os_ != rs
    ties = 0
    if near is None:
        if diff.any():
            bad.append(("seg", int(diff.sum())))
    else:
        ties = int(diff.sum())
        if (diff & (near[None] > 1e-9)).any():
            bad.append(("seg", int((diff & (near[None] > 1e-9)).sum())))
    want_loc = orc.sample_foreground_locations(os_, [1, 2, 3])     # the reference's sampling of the device's own seg
    bad += compare_locations(props["class_locations"], want_loc)
    if near is None:
        bad += compare_locations(props["class_locations"], rp["class_locations"])
    if seg is not None:
        bad += compare_intensities((props["intensities_per_channel"], props["intensity_statistics_per_channel"]),
                                   (rp["intensities_per_channel"], rp["intensity_statistics_per_channel"]))
    elif props["intensities_per_channel"] != [] or props["intensity_statistics_per_channel"] != []:
        bad.append(("intensities without seg",))
    return bad, ties
