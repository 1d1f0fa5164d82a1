"""CPU restatement (numpy / scipy) of the reference's CT case preprocessing -- DefaultPreprocessor.read_data +
run_case_npy with CTNormalization -- for preprocess_case(normalization="ct") in segmamba_b200/preprocess.py.  Test
infrastructure only: the product never imports it.

Everything but the normalisation is oracle/preprocess_oracle.py's restatement of the shared per-case step.
"""
from __future__ import annotations

import numpy as np

from oracle import preprocess_oracle as orc


def ct_normalize(image: np.ndarray, props: dict) -> np.ndarray:
    """CTNormalization(use_mask_for_norm=False).run of one channel with its intensity properties, in float32 as numpy
    computes it (Python-float bounds and scalars keep the float32 image in float32)"""
    image = image.astype(np.float32)
    image = np.clip(image, props["percentile_00_5"], props["percentile_99_5"])
    return (image - props["mean"]) / max(props["std"], 1e-8)


def preprocess_case(data: np.ndarray, seg: np.ndarray | None, spacing, target_spacing, intensity_properties,
                    all_labels=(1, 2), name=None):
    """(data, seg int8, properties, near): read_data (float32 data and labels) + run_case_npy with CTNormalization,
    intensity_properties[str(c)] per channel; near is the tie distance of the resampled labels (None when nothing was
    resampled)"""
    data = np.asarray(data, np.float32)
    if seg is not None:
        seg = np.asarray(seg, np.float32).reshape((1,) + data.shape[1:])
        inten, istats = orc.collect_foreground_intensities(seg, data)
    else:
        inten, istats = [], []
    props = {"spacing": tuple(spacing), "raw_size": data.shape[1:], "name": name, "intensities_per_channel": inten,
             "intensity_statistics_per_channel": istats}
    props["original_spacing_trans"] = list(spacing)[::-1]
    props["target_spacing_trans"] = list(target_spacing)
    props["shape_before_cropping"] = data.shape[1:]
    data, seg, bbox = orc.crop_to_nonzero(data, seg)
    props["bbox_used_for_cropping"] = bbox
    props["shape_after_cropping_before_resample"] = data.shape[1:]
    new_shape = orc.compute_new_shape(data.shape[1:], props["original_spacing_trans"], target_spacing)
    data = np.stack([ct_normalize(data[c], intensity_properties[str(c)]) for c in range(data.shape[0])])
    data, seg, near = orc.resample(data, seg, new_shape)
    props["shape_after_resample"] = new_shape
    props["class_locations"] = orc.sample_foreground_locations(seg, list(all_labels))
    return data, seg.astype(np.int8), props, near
