"""CPU checks of case preprocessing: the oracle against the fixture made by the reference's own code, compute_new_shape,
the draw structure, the properties preprocess_case returns (on the emulator), and the ctypes layouts of the C ABI."""
import os
import re

import numpy as np
import pytest
import torch

from emu import emulated
from oracle import preprocess_oracle as orc
from preprocess_checks import brats_like
from segmamba_b200 import _lib
from segmamba_b200 import predict as P
from segmamba_b200 import preprocess as PP

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "preprocess_cases.npz"))
STATS = ("mean", "median", "min", "max", "percentile_99_5", "percentile_00_5")


@pytest.mark.parametrize("name", ["identity", "aniso", "noseg"])
def test_oracle_reproduces_reference_fixture(name):
    g = {k[len(name) + 1:]: GOLDEN[k] for k in GOLDEN.files if k.startswith(name + "_")}
    d, s, props, _ = orc.preprocess_case(g["data"], g.get("seg"), tuple(g["spacing"]))
    assert np.allclose(d, g["out_data"], rtol=0, atol=4 * np.finfo(np.float32).eps * np.abs(g["out_data"]).max())
    assert np.array_equal(s, g["out_seg"]) and s.dtype == np.int8
    assert props["bbox_used_for_cropping"] == [list(b) for b in g["bbox"]]
    assert tuple(props["shape_after_cropping_before_resample"]) == tuple(g["shape_after_cropping_before_resample"])
    assert np.array_equal(props["shape_after_resample"], g["shape_after_resample"])
    for lab in (1, 2, 3):
        assert np.array_equal(np.asarray(props["class_locations"][lab], np.int64).reshape(-1, 4), g[f"loc_{lab}"])
    if "seg" in g:
        assert np.array_equal(np.stack(props["intensities_per_channel"]), g["intensities"])
        st = np.array([[x[f] for f in STATS] for x in props["intensity_statistics_per_channel"]], np.float64)
        assert np.array_equal(st, g["intensity_stats"])


def test_compute_new_shape_rounds_like_python():
    assert list(PP.compute_new_shape((14, 14, 16), [1.25, 0.8, 1.0], [1, 1, 1])) == [18, 11, 16]   # 17.5 -> 18
    assert list(PP.compute_new_shape((10, 5, 3), [1.25, 0.5, 1.5], [1, 1, 1])) == [12, 2, 4]       # 12.5 -> 12, 2.5 -> 2, 4.5 -> 4
    assert list(PP.compute_new_shape((7, 9, 11), [2.0, 1.0, 0.5], [1.0, 1.0, 1.0])) == list(orc.compute_new_shape((7, 9, 11), [2.0, 1.0, 0.5], [1, 1, 1]))


def test_empty_label_consumes_no_draw():
    a = PP._location_draws([5000, 0, 300], 1234)
    b = PP._location_draws([5000, 300], 1234)
    assert a[1] is None and np.array_equal(a[0], b[0]) and np.array_equal(a[2], b[1])
    assert len(PP._location_draws([2_000_000], 1)[0]) == 20000                    # ceil(1 % of n) above 10000
    assert PP._intensity_draws(0, 3, 1234, 10) == [None] * 3


def test_draws_reproduce_the_reference_sampling():
    seg = brats_like((13, 17, 19), channels=1, seed=4)[1].astype(np.int8)
    classes = [1, (2, 3), [1, 3], 7]
    want = orc.sample_foreground_locations(seg, classes)
    masks = [np.isin(seg, PP._class_labels(c)) for c in classes]
    draws = PP._location_draws([int(m.sum()) for m in masks], 1234)
    for c, m, d in zip(classes, masks, draws):
        key = PP._class_key(c)
        assert key in want
        if d is None:
            assert want[key] == []
        else:
            assert np.array_equal(np.argwhere(m)[d], want[key])


def test_properties_keys_types_and_case_geometry():
    data, seg = brats_like((13, 17, 19), channels=2, seed=0)
    with emulated():
        d, s, props = PP.preprocess_case(torch.from_numpy(data), torch.from_numpy(seg), spacing=(1.0, 0.8, 1.25), name="c0")
    assert list(props) == ["spacing", "raw_size", "name", "intensities_per_channel", "intensity_statistics_per_channel",
                           "original_spacing_trans", "target_spacing_trans", "shape_before_cropping", "bbox_used_for_cropping",
                           "shape_after_cropping_before_resample", "shape_after_resample", "class_locations"]
    assert d.dtype == torch.float32 and s.dtype == torch.int8 and s.shape[0] == 1
    assert tuple(d.shape[1:]) == tuple(props["shape_after_resample"]) == tuple(s.shape[1:])
    assert props["original_spacing_trans"] == [1.25, 0.8, 1.0] and props["target_spacing_trans"] == [1, 1, 1]
    assert all(isinstance(v, int) for b in props["bbox_used_for_cropping"] for v in b)
    for k, v in props["class_locations"].items():
        assert isinstance(v, list) and v == [] or (isinstance(v, np.ndarray) and v.dtype == np.int64 and v.shape[1] == 4)
    assert all(x.dtype == np.float32 and x.shape == (10000,) for x in props["intensities_per_channel"])
    assert all(set(st) == set(STATS) for st in props["intensity_statistics_per_channel"])
    crop, lo, full = P.case_geometry(props)
    assert full == (13, 17, 19) and crop == props["shape_after_cropping_before_resample"]


def test_bad_inputs_raise():
    with emulated():
        with pytest.raises(ValueError):
            PP.preprocess_case(torch.zeros((2, 4, 5, 6)))
        data, seg = brats_like((13, 17, 19), channels=2, seed=0)
        with pytest.raises(ValueError):
            PP.preprocess_case(torch.from_numpy(data), torch.from_numpy(seg * 64))          # labels above 127
        with pytest.raises(ValueError):
            PP.preprocess_case(torch.from_numpy(data), torch.from_numpy(seg + 0.5))         # non-integral labels
        with pytest.raises(ValueError):
            PP.resample_case(torch.zeros((1, 3, 8, 8)), None, (4, 8, 8))                    # prefilter lines of 4..256


def _fields(name):
    src = open(os.path.join(ROOT, "include", "segmamba_b200.h")).read()
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), src, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    out = []
    for stmt in filter(None, (s.strip() for s in body.split(";"))):
        decl = re.sub(r"^(const\s+)?(void|float|double|uint8_t|int8_t|uint32_t|int32_t|int64_t|smb_prep_record)\s*", "", stmt)
        out += [re.sub(r"\[.*\]", "", p).replace("*", "").strip() for p in decl.split(",")]
    return out


@pytest.mark.parametrize("cname,pyname", [("smb_prep_record", "PrepRecord"), ("smb_prep_mask_args", "PrepMaskArgs"),
                                          ("smb_prep_crop_args", "PrepCropArgs"), ("smb_prep_norm_job", "PrepNormJob"),
                                          ("smb_prep_label_resize_args", "PrepLabelResizeArgs"),
                                          ("smb_prep_compact_job", "PrepCompactJob"), ("smb_prep_gather_args", "PrepGatherArgs")])
def test_prep_ctypes_structs_match_header(cname, pyname):
    assert [f[0] for f in getattr(_lib, pyname)._fields_] == _fields(cname)


def test_prep_constants_match_header():
    src = open(os.path.join(ROOT, "include", "segmamba_b200.h")).read()
    assert f"#define SMB_PREP_CHUNK {_lib.PREP_CHUNK}" in src and f"#define SMB_PREP_MAX_JOBS {_lib.PREP_MAX_JOBS}" in src
