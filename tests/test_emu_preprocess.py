"""The case-preprocessing kernels (csrc/preprocess.cu) on the CPU SIMT emulator against the oracle, at ragged shapes, and the
whole preprocess_case against the fixture made by the reference's own code."""
import numpy as np
import pytest
import torch

from emu import emulated
from oracle import preprocess_oracle as orc
from preprocess_checks import brats_like, check_case, compare_intensities, compare_locations
from segmamba_b200 import preprocess as PP

SHAPES = [(13, 17, 19), (1, 9, 7), (5, 1, 1), (1, 1, 1)]
GOLDEN = np.load(__import__("os").path.join(__import__("os").path.dirname(__file__), "golden", "preprocess_cases.npz"))


@pytest.fixture(scope="module")
def emu():
    with emulated():
        yield "cpu"


@pytest.mark.parametrize("shape", SHAPES)
def test_emu_mask_crop_zscore(emu, shape):
    data, seg = brats_like(shape, channels=3, seed=3)
    d, s = torch.from_numpy(data), torch.from_numpy(seg)
    assert np.array_equal(PP.nonzero_mask(d).numpy(), orc.create_nonzero_mask(data))
    for sg in (s, None):
        cd, cs, bbox = PP.crop_to_nonzero(d, sg)
        rd, rs, rb = orc.crop_to_nonzero(data, None if sg is None else seg)
        assert bbox == rb
        assert np.array_equal(cd.numpy(), rd) and np.array_equal(cs.numpy(), rs.astype(np.int8))
    z, mom = PP.zscore(cd)
    ref = np.stack([orc.zscore(rd[c]) for c in range(rd.shape[0])])
    assert np.abs(z.numpy() - ref).max() <= 1e-5 * max(np.abs(ref).max(), 1.0)
    x = rd.astype(np.float64).reshape(rd.shape[0], -1)
    assert np.allclose(mom.numpy(), np.stack([x.mean(1), x.std(1)], 1), rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("scale", [(1.3, 0.7, 1.0), (0.5, 2.0, 1.5)])
def test_emu_label_resize(emu, shape, scale):
    rng = np.random.default_rng(5)
    seg = rng.integers(-1, 4, shape).astype(np.int8)
    new = tuple(max(1, int(round(n * f))) for n, f in zip(shape, scale))
    got = PP._label_resize(torch.from_numpy(seg), new)[0].numpy()
    want, near = orc.resize_segmentation(seg.astype(float), new)
    diff = got != want
    assert not (diff & (near > 1e-9)).any(), int(diff.sum())


@pytest.mark.parametrize("shape", SHAPES)
def test_emu_locations_and_intensities(emu, shape):
    data, seg = brats_like(shape, channels=2, seed=7)
    lab = seg.astype(np.int8)
    classes = [1, 2, 3, (1, 3), [2, 3], 9]
    got = PP.sample_foreground_locations(torch.from_numpy(lab), classes)
    assert compare_locations(got, orc.sample_foreground_locations(lab, classes)) == []
    got = PP.foreground_intensities(torch.from_numpy(data), torch.from_numpy(seg))
    assert compare_intensities(got, orc.collect_foreground_intensities(seg, data)) == []


@pytest.mark.parametrize("shape", [(13, 17, 19), (1, 9, 7)])
@pytest.mark.parametrize("labels", [True, False])
def test_emu_case_identity(emu, shape, labels):
    data, seg = brats_like(shape, channels=2, seed=1, labels=labels)
    assert check_case(data, seg, (1.0, 1.0, 1.0), (1, 1, 1), emu) == ([], 0)


def test_emu_case_resampled(emu):
    data, seg = brats_like((13, 17, 19), channels=2, seed=2)
    bad, ties = check_case(data, seg, (0.8, 1.0, 1.3), (1, 1, 1), emu, data_tol=1e-4)
    assert bad == [] and ties <= 2, (bad, ties)


@pytest.mark.parametrize("name", ["identity", "aniso", "noseg"])
def test_emu_case_matches_reference_fixture(emu, name):
    g = {k[len(name) + 1:]: GOLDEN[k] for k in GOLDEN.files if k.startswith(name + "_")}
    seg = torch.from_numpy(g["seg"]) if "seg" in g else None
    od, os_, props = PP.preprocess_case(torch.from_numpy(g["data"]), seg, spacing=tuple(g["spacing"]))
    assert [list(b) for b in g["bbox"]] == props["bbox_used_for_cropping"]
    assert tuple(g["shape_after_cropping_before_resample"]) == props["shape_after_cropping_before_resample"]
    assert np.array_equal(g["shape_after_resample"], props["shape_after_resample"])
    assert np.abs(od.numpy() - g["out_data"]).max() <= 1e-4 * np.abs(g["out_data"]).max()
    assert np.array_equal(os_.numpy(), g["out_seg"])
    for lab in (1, 2, 3):
        want = g[f"loc_{lab}"]
        got = props["class_locations"][lab]
        assert (len(want) == 0 and len(got) == 0) or np.array_equal(got, want)
    if seg is not None:
        assert np.array_equal(np.stack(props["intensities_per_channel"]), g["intensities"])
        st = np.array([[s[f] for f in ("mean", "median", "min", "max", "percentile_99_5", "percentile_00_5")]
                       for s in props["intensity_statistics_per_channel"]])
        assert np.allclose(st, g["intensity_stats"], rtol=1e-6, atol=0)
