"""Generate tests/golden/preprocess_cases.npz from the REFERENCE's own preprocessing code (needs the reference checkout).

TEST INFRASTRUCTURE.  What runs is the reference's MultiModalityPreprocessor, unmodified: DefaultPreprocessor.run_case_npy,
MultiModalityPreprocessor._normalize (ZScoreNormalization), collect_foreground_intensities and _sample_foreground_locations.
Three third-party functions it calls are not installed here and are replaced in sys.modules by restatements of what they do
(as gen_golden.py replaces the CUDA extension modules):
  acvl_utils get_bbox_from_mask / bounding_box_to_slice   [[lo, hi + 1]] per axis and the matching slices
  skimage.transform.resize                                 oracle.augment_oracle.resize (zoom, grid_mode, 'nearest', clipped)
  batchgenerators resize_segmentation                      per label in np.unique order, order-n indicator resize >= 0.5
The imports of SimpleITK, the batchgenerators file helpers and monai's clip (used only by CTNormalization) are empty stubs.

    python oracle/gen_preprocess_golden.py     ->  tests/golden/preprocess_cases.npz

Three cases of 2 channels: identity spacing with seg, anisotropic spacing (z up, y down) with seg, and no seg.  Each has a zero
background, an enclosed zero cavity inside the nonzero region and labels 1 / 2 / 3.
"""
from __future__ import annotations

import os
import sys
import types
import typing

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
OUT = os.path.join(ROOT, "tests", "golden", "preprocess_cases.npz")
SHAPE = (16, 18, 20)
CASES = (("identity", (1.0, 1.0, 1.0), True), ("aniso", (1.0, 0.8, 1.25), True), ("noseg", (1.0, 0.8, 1.25), False))


def _module(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


def _install_stubs():
    sys.path.insert(0, ROOT)
    from oracle.augment_oracle import resize as zoom_resize

    def get_bbox_from_mask(mask):
        idx = np.argwhere(mask)
        if len(idx) == 0:
            raise ValueError("empty mask")
        return [[int(idx[:, a].min()), int(idx[:, a].max()) + 1] for a in range(mask.ndim)]

    def bounding_box_to_slice(bbox):
        return tuple(slice(a, b) for a, b in bbox)

    def resize(image, output_shape, order=None, mode="reflect", cval=0, clip=True, preserve_range=False, anti_aliasing=None):
        assert mode == "edge" and not anti_aliasing and clip
        return zoom_resize(image, tuple(output_shape), order)

    def resize_segmentation(segmentation, new_shape, order=3):
        out = np.zeros(tuple(new_shape), dtype=segmentation.dtype)
        for c in np.unique(segmentation):
            out[resize((segmentation == c).astype(float), new_shape, order, mode="edge", clip=True, anti_aliasing=False) >= 0.5] = c
        return out

    for n in ("acvl_utils", "acvl_utils.cropping_and_padding", "batchgenerators", "batchgenerators.utilities",
              "batchgenerators.augmentations", "skimage", "monai", "monai.transforms"):
        _module(n)
    _module("acvl_utils.cropping_and_padding.bounding_boxes", get_bbox_from_mask=get_bbox_from_mask,
            bounding_box_to_slice=bounding_box_to_slice, crop_to_bbox=None)
    # the reference takes `os` and typing's `List` from this module's star import
    _module("batchgenerators.utilities.file_and_folder_operations", os=os, List=typing.List)
    _module("batchgenerators.augmentations.utils", resize_segmentation=resize_segmentation)
    _module("skimage.transform", resize=resize)
    _module("monai.transforms.utils_pytorch_numpy_unification", clip=np.clip)
    _module("SimpleITK")
    sys.path.insert(0, REF)


def main():
    _install_stubs()
    from light_training.preprocessing.preprocessors.preprocessor_mri import MultiModalityPreprocessor   # reference module
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from preprocess_checks import brats_like

    out = {}
    for i, (name, spacing, with_seg) in enumerate(CASES):
        data, seg = brats_like(SHAPE, channels=2, seed=10 + i, labels=with_seg)
        p = MultiModalityPreprocessor(base_dir="", image_dir="")
        p.out_spacing, p.all_labels, p.foreground_intensity_properties_per_channel = [1.0, 1.0, 1.0], [1, 2, 3], {}
        if with_seg:
            inten, istats = p.collect_foreground_intensities(seg, data)
        else:
            inten, istats = [], []
        props = {"spacing": spacing, "raw_size": data.shape[1:], "name": name, "intensities_per_channel": inten,
                 "intensity_statistics_per_channel": istats}
        d, s = p.run_case_npy(data, None if seg is None else seg.copy(), props)
        k = f"{name}_"
        out[k + "data"], out[k + "spacing"] = data, np.asarray(spacing)
        if with_seg:
            out[k + "seg"] = seg
            out[k + "intensities"] = np.stack(inten)
            out[k + "intensity_stats"] = np.array([[st[f] for f in ("mean", "median", "min", "max", "percentile_99_5",
                                                                    "percentile_00_5")] for st in istats], np.float64)
        out[k + "out_data"], out[k + "out_seg"] = d, s
        out[k + "bbox"] = np.asarray(props["bbox_used_for_cropping"])
        out[k + "shape_after_cropping_before_resample"] = np.asarray(props["shape_after_cropping_before_resample"])
        out[k + "shape_after_resample"] = np.asarray(props["shape_after_resample"])
        for lab, rows in props["class_locations"].items():
            out[k + f"loc_{lab}"] = np.asarray(rows, np.int64).reshape(-1, 4)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
