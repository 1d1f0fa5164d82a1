"""CT case preprocessing on the H100 against the oracle (oracle/ct_preprocess_oracle.py): 512 x 512 slices resampled with axes over
256 voxels (the streaming prefilter of csrc/augment.cu), CT normalisation with the statistics of plan.plan_dataset, and the
preprocessed case feeding restore_case and the patch loader."""
import numpy as np
import pytest
import torch

from ct_checks import check_ct_case, ct_like
from oracle import ct_preprocess_oracle as cto
from oracle import preprocess_oracle as orc
from segmamba_b200 import plan as PL
from segmamba_b200 import predict as P
from segmamba_b200 import preprocess as PP
from segmamba_b200.patch_loader import GpuPatchLoader

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LITS_SHAPE, LITS_SPACING, LITS_TARGET = (48, 512, 512), (0.7, 0.7, 2.5), [1.0, 0.76757812, 0.76757812]


def _props(data, seg, spacing):
    """the dataset statistics of a one-case dataset, through foreground_intensities and plan_dataset"""
    samples, _ = PP.foreground_intensities(torch.from_numpy(data).to(DEV), torch.from_numpy(seg).to(DEV))
    return PL.plan_dataset([spacing], [data.shape[1:]], [samples])["intensity_statistics_per_channel"]


@pytest.fixture(scope="module")
def lits():
    data, seg = ct_like(LITS_SHAPE, seed=1)
    return data, seg, _props(data, seg, LITS_SPACING)


def test_lits_like_resampled(lits):
    data, seg, props = lits
    bad, ties, (od, _, pp) = check_ct_case(data, seg, LITS_SPACING, LITS_TARGET, props, DEV)
    print("label near-ties that differ:", ties, "output", tuple(od.shape))
    assert max(pp["shape_after_cropping_before_resample"][1:]) > 256 and max(od.shape[2:]) > 256
    assert bad == [], bad
    assert ties <= 50, ties


def test_long_axis_0():
    data, seg = ct_like((300, 160, 160), seed=2)
    bad, ties, (od, _, pp) = check_ct_case(data, seg, (1.0, 1.0, 0.8), [1, 1, 1], _props(data, seg, (1.0, 1.0, 0.8)), DEV)
    assert pp["shape_after_cropping_before_resample"][0] > 256
    assert bad == [] and ties <= 50, (bad, ties)


def test_identity_bit_equal_and_restore_round_trip(lits):
    _, _, props = lits
    data, seg = ct_like((64, 512, 512), seed=3)
    d, s = torch.from_numpy(data).to(DEV), torch.from_numpy(seg).to(DEV)
    od, oseg, pp = PP.preprocess_case(d, s, spacing=(1.0, 1.0, 1.0), target_spacing=[1, 1, 1], all_labels=(1, 2),
                                      normalization="ct", intensity_properties=props)
    crop, _, _ = orc.crop_to_nonzero(data, seg)
    want = cto.ct_normalize(crop[0], props["0"])[None]
    assert np.array_equal(od.cpu().numpy().view(np.uint32), want.view(np.uint32))
    lab = oseg[0].long().clamp(min=0)
    logits = torch.nn.functional.one_hot(lab, 3).permute(3, 0, 1, 2).float().contiguous()
    out = P.restore_case(logits, pp, regions=None)
    assert np.array_equal(out.cpu().numpy(), seg[0].astype(np.uint8))


def test_two_runs_bitwise_equal(lits):
    data, seg, props = lits
    d, s = torch.from_numpy(data).to(DEV), torch.from_numpy(seg).to(DEV)
    run = lambda: PP.preprocess_case(d, s, spacing=LITS_SPACING, target_spacing=LITS_TARGET, all_labels=(1, 2),
                                     normalization="ct", intensity_properties=props)
    a, b = run(), run()
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    for k in a[2]["class_locations"]:
        assert np.array_equal(a[2]["class_locations"][k], b[2]["class_locations"][k])


def test_no_sync_and_readbacks(lits):
    data, seg, props = lits
    d, s = torch.from_numpy(data).to(DEV), torch.from_numpy(seg).to(DEV)
    crop, cs, _ = PP.crop_to_nonzero(d, s)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        z = PP.ct_normalize(crop, props)
        PP.resample_case(z, cs, (100, 300, 520))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    n0 = PP._readbacks
    PP.preprocess_case(d, s, spacing=LITS_SPACING, target_spacing=LITS_TARGET, all_labels=(1, 2), normalization="ct",
                       intensity_properties=props)
    assert PP._readbacks - n0 == PP.READBACKS_PER_CASE == 3


def test_patch_loader_draws_from_a_ct_case(lits):
    data, seg, props = lits
    d, s = torch.from_numpy(data).to(DEV), torch.from_numpy(seg).to(DEV)
    od, oseg, pp = PP.preprocess_case(d, s, spacing=LITS_SPACING, target_spacing=LITS_TARGET, all_labels=(1, 2),
                                      normalization="ct", intensity_properties=props)
    loader = GpuPatchLoader([{"data": od, "seg": oseg, "class_locations": pp["class_locations"]}], (128, 128, 128),
                            batch_size=2, augmentation=False, device=DEV)
    image, label = next(loader)
    torch.cuda.synchronize()
    assert tuple(image.shape) == (2, 1, 128, 128, 128) and tuple(label.shape) == (2, 128, 128, 128)
    assert torch.isfinite(image).all() and (label > 0).any()
