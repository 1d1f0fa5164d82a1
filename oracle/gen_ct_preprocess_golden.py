"""Generate tests/golden/ct_preprocess_cases.npz from the REFERENCE's own CT preprocessing code (needs the reference checkout).

TEST INFRASTRUCTURE.  What runs is the reference's DefaultPreprocessor, unmodified except for a subclass that overrides
get_iterable_list / read_data so that synthetic arrays go in instead of NIfTI files: run_case_npy (crop, CTNormalization,
resampling, foreground locations), collect_foreground_intensities and run_plan (dataset statistics, target spacing, median
shape, patch size).  run_plan writes its data_analysis_result.txt into a temporary directory, from which it is read back.
The third-party stubs are gen_preprocess_golden.py's.

    python oracle/gen_ct_preprocess_golden.py     ->  tests/golden/ct_preprocess_cases.npz

Cases, one channel of integer HU values (air -1000 outside the body, zero outside a circular field of view so that the crop
cuts), labels 1 and 2, normalised with the statistics of the plan dataset "iso":
  resampled  8 x 10 x 300 at (0.7, 0.8, 2.5) -> [1.0, 0.768, 0.768]: axis 2 stays above 256 voxels after the crop
  identity   12 x 40 x 44 at (1, 1, 1) -> [1, 1, 1]
  noseg      8 x 30 x 32 at (0.9, 0.9, 1.5) -> [1.0, 0.768, 0.768], no seg
Plan datasets of three cases: "iso" (no anisotropic axis) and "aniso" (a coarse third spacing axis with a short third size
axis, which takes the anisotropic branch of determine_fullres_target_spacing).
"""
from __future__ import annotations

import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.gen_preprocess_golden import _install_stubs  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "ct_preprocess_cases.npz")
TARGET = [1.0, 0.768, 0.768]
CASES = (("resampled", (8, 10, 300), (0.7, 0.8, 2.5), TARGET, True),
         ("identity", (12, 40, 44), (1.0, 1.0, 1.0), [1.0, 1.0, 1.0], True),
         ("noseg", (8, 30, 32), (0.9, 0.9, 1.5), TARGET, False))
PLANS = {"iso": [((10, 24, 26), (0.8, 0.8, 1.0)), ((12, 22, 24), (0.75, 0.75, 1.25)), ((9, 26, 22), (0.7, 0.7, 1.5))],
         "aniso": [((30, 28, 8), (0.7, 0.7, 5.0)), ((28, 30, 7), (0.8, 0.8, 4.0)), ((32, 26, 9), (0.75, 0.75, 6.0))]}


def main():
    _install_stubs()
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from ct_checks import ct_like
    from light_training.preprocessing.preprocessors.default_preprocessor import DefaultPreprocessor   # reference module

    class ArrayPreprocessor(DefaultPreprocessor):
        """the reference's preprocessor on in-memory cases: {name: (data, seg, spacing)}"""

        def __init__(self, cases):
            super().__init__(base_dir="", image_dir="")
            self.cases = cases

        def get_iterable_list(self):
            return list(self.cases)

        def read_data(self, case_name):
            data, seg, spacing = self.cases[case_name]
            if seg is not None:
                inten, istats = self.collect_foreground_intensities(seg, data)
            else:
                inten, istats = [], []
            return data.copy(), None if seg is None else seg.copy(), {
                "spacing": spacing, "raw_size": data.shape[1:], "name": case_name, "intensities_per_channel": inten,
                "intensity_statistics_per_channel": istats}

    out = {}
    plans = {}
    for pname, members in PLANS.items():
        cases = {}
        for i, (shape, spacing) in enumerate(members):
            d, s = ct_like(shape, seed=100 + 10 * len(plans) + i)
            cases[f"{pname}{i}"] = (d, s, spacing)
        p = ArrayPreprocessor(cases)
        cwd = os.getcwd()
        with tempfile.TemporaryDirectory() as tmp:
            os.chdir(tmp)
            try:
                p.run_plan()
                text = open("data_analysis_result.txt").read()
            finally:
                os.chdir(cwd)
        plans[pname] = json.loads(text)
        k = f"plan_{pname}_"
        out[k + "json"] = np.array(text)
        out[k + "spacings"] = np.array([sp for _, sp in members], np.float64)
        out[k + "sizes"] = np.array([sh for sh, _ in members], np.int64)
        for i, name in enumerate(cases):
            out[k + f"intensities{i}"] = np.stack(p.read_data(name)[2]["intensities_per_channel"])
    props = plans["iso"]["intensity_statistics_per_channel"]
    for i, (name, shape, spacing, target, with_seg) in enumerate(CASES):
        data, seg = ct_like(shape, seed=10 + i, labels=with_seg)
        p = ArrayPreprocessor({name: (data, seg, spacing)})
        p.out_spacing, p.all_labels, p.foreground_intensity_properties_per_channel = target, [1, 2], props
        d, s, pr = p.read_data(name)
        d, s = p.run_case_npy(d, s, pr)
        k = f"{name}_"
        out[k + "data"], out[k + "spacing"], out[k + "target"] = data, np.asarray(spacing), np.asarray(target)
        if with_seg:
            out[k + "seg"] = seg
            out[k + "intensities"] = np.stack(pr["intensities_per_channel"])
            out[k + "out_seg"] = s
            for lab, rows in pr["class_locations"].items():
                out[k + f"loc_{lab}"] = np.asarray(rows, np.int64).reshape(-1, 4)
        out[k + "out_data"] = d
        out[k + "bbox"] = np.asarray(pr["bbox_used_for_cropping"])
        out[k + "shape_after_cropping_before_resample"] = np.asarray(pr["shape_after_cropping_before_resample"])
        out[k + "shape_after_resample"] = np.asarray(pr["shape_after_resample"])
    out["intensity_properties"] = np.array(json.dumps(props))
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
