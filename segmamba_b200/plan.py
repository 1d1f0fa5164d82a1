"""The dataset plan of the reference's CT pipelines (DefaultPreprocessor.run_plan), restated on the host.

plan_dataset(spacings, sizes, intensities) takes, per case, the SimpleITK (x, y, z) spacing, the raw array size (z, y, x) and
the foreground intensity samples per channel (preprocess.foreground_intensities(...)[0]), and returns the dict run_plan writes
to data_analysis_result.txt, with the values as they read back from that JSON file:

  intensity_statistics_per_channel  {"0": {mean, median, std, min, max, percentile_99_5, percentile_00_5}, ...}: numpy's
                                    statistics of the concatenated float32 samples of all cases, bit-equal to the reference's;
                                    preprocess.preprocess_case(normalization="ct") takes this dict as intensity_properties
  fullres spacing                   determine_fullres_target_spacing, in the (x, y, z) order of the spacings
  median_shape                      median over the cases of compute_new_shape at that spacing
  initial_patch_size                1 / spacing scaled to 256^3 voxels, rounded
  target medium patch size          get_pool_and_conv_props' patch size (min feature map 4), reversed

The reference's behaviour is restated, quirks included (DESIGN.md §3.14): determine_fullres_target_spacing compares an (x, y, z)
spacing with a (z, y, x) size axis by axis, and get_pool_and_conv_props indexes the spacings of the poolable axes with the full
axis number, which raises IndexError once fewer than three axes can still pool and a kernel size is not yet 3.
"""
from __future__ import annotations

import json

import numpy as np

__all__ = ["plan_dataset", "fullres_target_spacing", "pool_and_conv_props"]


def fullres_target_spacing(spacings, sizes) -> np.ndarray:
    """determine_fullres_target_spacing: the median spacing, with the worst axis lowered to its 10th percentile when that axis
    is both much coarser and much shorter than the others.  spacings and sizes are indexed by the same axis number."""
    target = np.percentile(np.vstack(spacings), 50, 0)
    target_size = np.percentile(np.vstack(sizes), 50, 0)
    worst = int(np.argmax(target))
    others = [i for i in range(len(target)) if i != worst]
    other_spacings = [target[i] for i in others]
    other_sizes = [target_size[i] for i in others]
    if target[worst] > 3 * max(other_spacings) and target_size[worst] * 3 < min(other_sizes):
        s = np.percentile(np.vstack(spacings)[:, worst], 10)
        if s < max(other_spacings):
            s = max(max(other_spacings), s) + 1e-5
        target[worst] = s
    return target


def _new_shape(size, spacing, target) -> np.ndarray:
    """DefaultPreprocessor.compute_new_shape: both spacings reversed to array order"""
    old, new = list(spacing)[::-1], list(target)[::-1]
    assert len(old) == len(size) == len(new)
    return np.array([int(round(i / j * k)) for i, j, k in zip(old, new, size)])


def _pad_shape(shape, divisor) -> np.ndarray:
    out = [shape[i] + divisor[i] - shape[i] % divisor[i] for i in range(len(shape))]
    for i in range(len(shape)):
        if shape[i] % divisor[i] == 0:
            out[i] -= divisor[i]
    return np.array(out).astype(int)


def pool_and_conv_props(spacing, patch_size, min_feature_map_size=4, max_numpool=999999):
    """get_pool_and_conv_props: (pools per axis, pool kernel sizes, conv kernel sizes, padded patch size, divisor)"""
    dim = len(spacing)
    spacing_now, size_now = list(spacing), list(patch_size)
    pool_kernels, conv_kernels = [[1] * dim], []
    pools, kernel = [0] * dim, [1] * dim
    while True:
        valid = [i for i in range(dim) if size_now[i] >= 2 * min_feature_map_size]
        if not valid:
            break
        valid_spacings = [spacing_now[i] for i in valid]
        smallest = min(valid_spacings)
        valid = [i for i in valid if spacing_now[i] / smallest < 2]
        valid = [i for i in valid if pools[i] < max_numpool]
        if len(valid) == 1 and size_now[valid[0]] < 3 * min_feature_map_size:
            break
        if not valid:
            break
        for d in range(dim):
            if kernel[d] != 3 and valid_spacings[d] / min(spacing_now) < 2:    # the reference's indexing, by full axis number
                kernel[d] = 3
        step = [0] * dim
        for v in range(dim):
            if v in valid:
                step[v] = 2
                pools[v] += 1
                spacing_now[v] *= 2
                size_now[v] = np.ceil(size_now[v] / 2)
            else:
                step[v] = 1
        pool_kernels.append(step)
        conv_kernels.append(list(kernel))
    divisor = 2 ** np.array(pools)
    conv_kernels.append([3] * dim)
    return pools, pool_kernels, conv_kernels, _pad_shape(patch_size, divisor), divisor


def _statistics(samples: np.ndarray) -> dict:
    return {"mean": float(np.mean(samples)), "median": float(np.median(samples)), "std": float(np.std(samples)),
            "min": float(np.min(samples)), "max": float(np.max(samples)),
            "percentile_99_5": float(np.percentile(samples, 99.5)), "percentile_00_5": float(np.percentile(samples, 0.5))}


def plan_dataset(spacings, sizes, intensities) -> dict:
    """run_plan's data_analysis_result.txt as a dict (JSON types, channel keys "0", "1", ...).

    spacings     per case, the SimpleITK (x, y, z) spacing
    sizes        per case, the raw array size (z, y, x)
    intensities  per case, a list of per-channel float32 sample arrays (preprocess.foreground_intensities(...)[0])"""
    spacings, sizes, intensities = list(spacings), list(sizes), list(intensities)
    if not (len(spacings) == len(sizes) == len(intensities)) or not spacings:
        raise ValueError(f"one spacing, size and intensity list per case, got {len(spacings)}, {len(sizes)}, {len(intensities)}")
    channels = len(intensities[0])
    per_channel = [np.concatenate([np.asarray(r[c]) for r in intensities]) for c in range(channels)]
    stats = {c: _statistics(per_channel[c]) for c in range(channels)}
    target = fullres_target_spacing(spacings, sizes)
    median_shape = np.median([_new_shape(size, sp, target) for sp, size in zip(spacings, sizes)], 0)
    inv = 1 / np.array(target)
    initial = [round(i) for i in inv * (256 ** 3 / np.prod(inv)) ** (1 / 3)]
    patch = pool_and_conv_props(target, initial, 4, 999999)[3]
    plan = {"intensity_statistics_per_channel": stats, "fullres spacing": target.tolist(), "median_shape": median_shape.tolist(),
            "initial_patch_size": initial, "target medium patch size": patch[::-1].tolist()}
    return json.loads(json.dumps(plan))
