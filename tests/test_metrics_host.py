"""CPU checks of the metric semantics: analytic cases of the oracle (oracle/metrics_oracle.py), the reference's two case
rules, numpy-percentile agreement, and the ctypes layouts of the metric C ABI against the header."""
import os
import re

import numpy as np
import pytest
import torch

from oracle import metrics_oracle as orc
from segmamba_b200 import _lib
from segmamba_b200 import metrics as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_single_voxels_anisotropic():
    p = np.zeros((9, 10, 11), bool)
    g = np.zeros_like(p)
    p[1, 2, 3] = True
    g[4, 6, 8] = True
    s = (2.5, 0.9, 0.7)
    want = np.sqrt(((3 * 2.5) ** 2 + (4 * 0.9) ** 2) + (5 * 0.7) ** 2)
    assert orc.hd_percentile(p, g, s) == want and orc.hd_percentile(p, g, s, q=100) == want


def test_cube_against_shifted_cube():
    p = np.zeros((12, 12, 12), bool)
    g = np.zeros_like(p)
    p[2:7, 2:7, 2:7] = True
    g[2:7, 2:7, 4:9] = True                                              # shifted by 2 along the last axis
    assert orc.dc(p, g) == 2.0 * 75 / 250
    assert orc.hd_percentile(p, g, q=100) == 2.0
    assert orc.hd_percentile(p, g, (1, 1, 3.0), q=100) == 6.0


def test_faces_are_border_and_full_volume():
    full = np.ones((4, 5, 6), bool)
    b = orc.border(full)
    assert b.sum() == full.size - 2 * 3 * 4 and not b[1:-1, 1:-1, 1:-1].any()
    assert orc.hd_percentile(full, full) == 0.0 and orc.dc(full, full) == 1.0


def test_voxel_inside_g_measures_to_the_border():
    g = np.zeros((11, 11, 11), bool)
    g[1:10, 1:10, 1:10] = True
    p = np.zeros_like(g)
    p[5, 5, 5] = True                                                    # 4 voxels from G's border on every axis
    d = orc.surface_distances(p, g)
    assert d.tolist() == [4.0]


def test_empty_masks():
    e = np.zeros((3, 3, 3), bool)
    f = e.copy()
    f[1, 1, 1] = True
    assert np.isnan(orc.hd_percentile(e, f)) and np.isnan(orc.hd_percentile(f, e)) and orc.dc(e, e) == 0.0


def test_case_rule_tables():
    e = np.zeros((1, 4, 4, 4), bool)
    f = e.copy()
    f[0, 1:3, 1:3, 1:3] = True
    assert orc.each_cases_metric(e, f).tolist() == [[0.0, 50.0]]
    assert orc.each_cases_metric(f, e).tolist() == [[0.0, 50.0]]
    assert orc.each_cases_metric(e, e).tolist() == [[0.0, 50.0]]
    assert orc.each_cases_metric(f, f).tolist() == [[1.0, 0.0]]
    z = np.zeros((2, 4, 4, 4), np.int64)
    lab = z.copy()
    lab[0, 1, 1, 1] = 3
    assert orc.validation_dices(z, z) == [1.0, 1.0, 1.0]
    assert orc.validation_dices(z, lab) == [0.0, 0.0, 0.0]
    assert orc.validation_dices(lab, lab) == [1.0, 1.0, 1.0]
    half = lab.copy()
    half[1, 2, 2, 2] = 3
    assert orc.validation_dices(half, lab) == [2 / 3, 2 / 3, 2 / 3]


@pytest.mark.parametrize("n", [1, 2, 3, 20, 21, 101, 1000])
def test_percentile_restatement(n):
    """the device's selection: numpy 'linear' as index (n - 1) q, its floor and numpy's two-branch lerp."""
    rng = np.random.default_rng(n)
    x = np.sqrt(rng.integers(0, 50, n).astype(np.float64))
    for q in (95.0, 100.0, 50.0, 0.0):
        s = np.sort(x)
        v = (n - 1) * (q / 100.0)
        if v >= n - 1:
            want = s[-1]
        else:
            k = int(np.floor(v))
            t = v - k
            a, b = s[k], s[k + 1]
            want = b - (b - a) * (1 - t) if t >= 0.5 else a + (b - a) * t
        assert np.percentile(x, q) == want


def test_regions_and_rejects_cpu():
    lab = np.array([0, 1, 2, 3, 4]).reshape(1, 1, 5)
    assert orc.regions_of(lab).astype(int).reshape(3, 5).tolist() == [[0, 1, 0, 1, 0], [0, 1, 1, 1, 0], [0, 0, 0, 1, 0]]
    with pytest.raises(RuntimeError):
        M.dice(torch.zeros(1, 4, 4, 4, dtype=torch.int64), torch.zeros(1, 4, 4, 4, dtype=torch.int64))
    with pytest.raises(ValueError):
        M._lut([(1,)] * 9)


def _fields(name):
    src = open(os.path.join(ROOT, "include", "segmamba_b200.h")).read()
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), src, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    out = []
    for stmt in filter(None, (s.strip() for s in body.split(";"))):
        decl = re.sub(r"^(const\s+)?(void|float|double|uint8_t|int32_t|int64_t)\s*", "", stmt)
        out += [re.sub(r"\[.*\]", "", p).replace("*", "").strip() for p in decl.split(",")]
    return out


@pytest.mark.parametrize("cname,pyname", [("smb_metric_bits_args", "MetricBitsArgs"), ("smb_metric_count_args", "MetricCountArgs"),
                                          ("smb_metric_edt_args", "MetricEdtArgs"), ("smb_metric_select_args", "MetricSelectArgs")])
def test_metric_ctypes_structs_match_header(cname, pyname):
    assert [f[0] for f in getattr(_lib, pyname)._fields_] == _fields(cname)


def test_metric_constants_match_header():
    src = open(os.path.join(ROOT, "include", "segmamba_b200.h")).read()
    for name, val in (("MAX_REGIONS", _lib.METRIC_MAX_REGIONS), ("MAX_AXIS", _lib.METRIC_MAX_AXIS), ("NCOUNTS", _lib.METRIC_NCOUNTS)):
        assert int(re.search(r"#define SMB_METRIC_%s (\d+)" % name, src).group(1)) == val
    assert "SMB_METRIC_I8 = 0, SMB_METRIC_U8 = 1, SMB_METRIC_I32 = 2, SMB_METRIC_I64 = 3, SMB_METRIC_LOGITS = 4" in src
