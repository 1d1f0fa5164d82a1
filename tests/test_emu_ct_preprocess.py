"""CT case preprocessing on the CPU SIMT emulator: the streaming prefilter of lines over 256 samples (csrc/augment.cu) through
resample_case against the oracle, smb_prep_ct_normalize bit-equal to numpy, and preprocess_case(normalization="ct") against
the fixture made by the reference's own DefaultPreprocessor."""
import json
import os

import numpy as np
import pytest
import torch

from emu import emulated
from oracle import ct_preprocess_oracle as cto
from oracle import preprocess_oracle as orc
from oracle.augment_oracle import resize
from segmamba_b200 import preprocess as PP

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "ct_preprocess_cases.npz"))
PROPS = json.loads(str(GOLDEN["intensity_properties"]))


@pytest.fixture(scope="module")
def emu():
    with emulated():
        yield "cpu"


def _smooth(shape, seed):
    rng = np.random.default_rng(seed)
    g = np.meshgrid(*[np.linspace(0, 1, n) for n in shape], indexing="ij")
    x = np.sin(7 * g[0] + 2 * g[1]) * np.cos(5 * g[2]) * 800 + rng.normal(0, 60, shape)
    return x.astype(np.float32)


@pytest.mark.parametrize("src,dst", [((300, 5, 6), (310, 5, 6)), ((5, 300, 6), (5, 150, 6)), ((5, 6, 300), (5, 6, 520)),
                                     ((2100, 4, 4), (1000, 4, 4))])
def test_emu_long_line_resample(emu, src, dst):
    x = _smooth(src, 3)
    seg = np.random.default_rng(4).integers(-1, 3, (1,) + src).astype(np.int8)
    out, oseg = PP.resample_case(torch.from_numpy(x[None]), torch.from_numpy(seg), dst)
    want = resize(x.astype(np.float64), dst, 3)
    err = np.abs(out[0].numpy().astype(np.float64) - want).max() / np.abs(want).max()
    assert out.shape == (1,) + dst and err <= 1e-4, err
    wseg, near = orc.resize_segmentation(seg[0].astype(float), dst)
    diff = oseg[0].numpy() != wseg
    assert not (diff & (near > 1e-9)).any(), int(diff.sum())


def test_emu_long_and_short_jobs_in_one_launch(emu):
    """a job whose axis 2 is short next to one whose axis 2 is long: each line goes to its own kernel"""
    a, b = _smooth((6, 7, 300), 5), _smooth((6, 7, 40), 6)
    ra, _ = PP.resample_case(torch.from_numpy(a[None]), None, (6, 7, 280))
    rb, _ = PP.resample_case(torch.from_numpy(b[None]), None, (6, 7, 50))
    from segmamba_b200 import _lib
    from segmamba_b200 import augment as A
    coef = [torch.empty(10 * 11 * (n + 4)) for n in (300, 40)]
    A.prefilter([A.prefilter_job(torch.from_numpy(x), c, x.shape, _lib.AUG_EDGE) for x, c in zip((a, b), coef)], "cpu")
    single = [torch.empty(10 * 11 * (n + 4)) for n in (300, 40)]
    for x, c in zip((a, b), single):
        A.prefilter([A.prefilter_job(torch.from_numpy(x), c, x.shape, _lib.AUG_EDGE)], "cpu")
    assert all(torch.equal(p, q) for p, q in zip(coef, single))
    assert ra.shape == (1, 6, 7, 280) and rb.shape == (1, 6, 7, 50)


def _ct_numpy(x, p):
    return cto.ct_normalize(x, p)


def test_emu_ct_normalize_bit_equal(emu):
    rng = np.random.default_rng(0)
    x = rng.normal(0, 600, (2, 9, 17, 23)).astype(np.float32)
    x[0, 0, 0, :4] = [-0.0, 0.0, np.inf, -np.inf]
    x[1, 1, 1, 1] = np.nan
    props = {"0": dict(mean=35.596134185791016, std=117.85196685791016, percentile_00_5=-267.0, percentile_99_5=334.0),
             "1": dict(mean=-12.3456789, std=3e-9, percentile_00_5=-281.0050048828125, percentile_99_5=1e3)}
    got = PP.ct_normalize(torch.from_numpy(x), props).numpy()
    want = np.stack([_ct_numpy(x[c], props[str(c)]) for c in range(2)])
    assert got.dtype == np.float32 and want.dtype == np.float32
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan)
    assert np.array_equal(got[~nan].view(np.uint32), want[~nan].view(np.uint32))
    assert (x[0] < -267).any() and (x[0] > 334).any()                   # both clip bounds are exercised


def test_emu_ct_normalize_rejects_missing_properties(emu):
    x = torch.ones((2, 4, 4, 4))
    with pytest.raises(ValueError):
        PP.ct_normalize(x, PROPS)                                        # no channel "1"
    with pytest.raises(ValueError):
        PP.ct_normalize(x[:1], {"0": {"mean": 0.0, "std": 1.0, "percentile_00_5": -1.0}})
    with pytest.raises(ValueError):
        PP.preprocess_case(x, normalization="ct")


@pytest.mark.parametrize("name", ["resampled", "identity", "noseg"])
def test_emu_ct_case_matches_reference_fixture(emu, name):
    g = {k[len(name) + 1:]: GOLDEN[k] for k in GOLDEN.files if k.startswith(name + "_")}
    seg = torch.from_numpy(g["seg"]) if "seg" in g else None
    od, os_, props = PP.preprocess_case(torch.from_numpy(g["data"]), seg, spacing=tuple(g["spacing"]),
                                        target_spacing=list(g["target"]), all_labels=(1, 2), normalization="ct",
                                        intensity_properties=PROPS)
    assert [list(b) for b in g["bbox"]] == props["bbox_used_for_cropping"]
    assert tuple(g["shape_after_cropping_before_resample"]) == props["shape_after_cropping_before_resample"]
    assert np.array_equal(g["shape_after_resample"], props["shape_after_resample"])
    od = od.numpy()
    if name == "identity":
        assert np.array_equal(od.view(np.uint32), g["out_data"].view(np.uint32))
    else:
        assert np.abs(od.astype(np.float64) - g["out_data"]).max() <= 1e-4 * np.abs(g["out_data"]).max()
    if seg is None:
        return
    assert np.array_equal(os_.numpy(), g["out_seg"])
    for lab in (1, 2):
        assert np.array_equal(props["class_locations"][lab], g[f"loc_{lab}"])
    assert np.array_equal(np.stack(props["intensities_per_channel"]), g["intensities"])
