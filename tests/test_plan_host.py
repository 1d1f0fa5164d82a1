"""The dataset plan (segmamba_b200/plan.py) against run_plan of the reference, as recorded in tests/golden/ct_preprocess_cases.npz,
and the CT normalisation's ctypes record against the header.  Host only."""
import json
import os
import re

import numpy as np
import pytest

from segmamba_b200 import _lib
from segmamba_b200 import plan as PL

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "ct_preprocess_cases.npz"))


def _inputs(name):
    k = f"plan_{name}_"
    spacings = [tuple(float(v) for v in s) for s in GOLDEN[k + "spacings"]]
    sizes = [tuple(int(v) for v in s) for s in GOLDEN[k + "sizes"]]
    intensities = [list(GOLDEN[k + f"intensities{i}"]) for i in range(len(spacings))]
    return spacings, sizes, intensities


@pytest.mark.parametrize("name", ["iso", "aniso"])
def test_plan_matches_reference_run_plan(name):
    want = json.loads(str(GOLDEN[f"plan_{name}_json"]))
    got = PL.plan_dataset(*_inputs(name))
    assert got == want
    assert json.loads(json.dumps(got)) == want                          # the text round trip of data_analysis_result.txt


def test_plan_takes_both_target_spacing_branches():
    iso = PL.plan_dataset(*_inputs("iso"))["fullres spacing"]
    aniso = PL.plan_dataset(*_inputs("aniso"))["fullres spacing"]
    assert iso == list(np.percentile(GOLDEN["plan_iso_spacings"], 50, 0))       # the median spacing
    assert aniso[2] == np.percentile(GOLDEN["plan_aniso_spacings"][:, 2], 10)   # the coarse axis lowered to its 10th percentile


def test_plan_statistics_feed_ct_normalisation():
    props = PL.plan_dataset(*_inputs("iso"))["intensity_statistics_per_channel"]
    assert props == json.loads(str(GOLDEN["intensity_properties"]))
    assert set(props["0"]) == {"mean", "median", "std", "min", "max", "percentile_99_5", "percentile_00_5"}


def test_pool_and_conv_props_restates_the_reference():
    pools, pool_k, conv_k, patch, div = PL.pool_and_conv_props((1.0, 1.0, 1.0), [128, 128, 128])
    assert pools == [5, 5, 5] and list(patch) == [128, 128, 128] and list(div) == [32, 32, 32]
    assert len(pool_k) == 6 and conv_k[-1] == [3, 3, 3]
    with pytest.raises(IndexError):                                      # the reference's spacings_of_axes[d] with d a full axis
        PL.pool_and_conv_props((1, 2, 5), [20, 100, 7])


def test_plan_rejects_mismatched_inputs():
    spacings, sizes, intensities = _inputs("iso")
    with pytest.raises(ValueError):
        PL.plan_dataset(spacings, sizes[:2], intensities)


def test_ct_norm_job_matches_header():
    src = open(os.path.join(ROOT, "include", "segmamba_b200.h")).read()
    body = re.search(r"typedef struct smb_prep_ct_norm_job \{(.*?)\} smb_prep_ct_norm_job;", src, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for stmt in filter(None, (s.strip() for s in body.split(";"))):
        decl = re.sub(r"^(const\s+)?(float|int64_t)\s*", "", stmt)
        fields += [p.replace("*", "").strip() for p in decl.split(",")]
    assert [f[0] for f in _lib.PrepCtNormJob._fields_] == fields
    assert [f[1] for f in _lib.PrepCtNormJob._fields_][3:] == [__import__("ctypes").c_float] * 4
    assert "smb_prep_ct_normalize" in _lib.EXPORTS and "SMB_API int smb_prep_ct_normalize(" in src
