"""Case preprocessing on the H100 against the oracle (oracle/preprocess_oracle.py), at the BraTS size 4 x 155 x 240 x 240."""
import numpy as np
import pytest
import torch

from oracle import preprocess_oracle as orc
from preprocess_checks import brats_like, check_case, dev_case
from segmamba_b200 import predict as P
from segmamba_b200 import preprocess as PP

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SHAPE = (155, 240, 240)
RESAMPLED = (1.0, 0.8, 1.25)             # SimpleITK (x, y, z): z up by 1.25, y down by 0.8, x unchanged


@pytest.fixture(scope="module")
def case():
    return brats_like(SHAPE, channels=4, seed=0)


def test_identity_spacing(case):
    data, seg = case
    bad, ties = check_case(data, seg, (1.0, 1.0, 1.0), (1, 1, 1), DEV, data_tol=1e-5)
    assert bad == [] and ties == 0, bad


def test_resampled(case):
    data, seg = case
    bad, ties = check_case(data, seg, RESAMPLED, (1, 1, 1), DEV, data_tol=1e-4)
    print("label near-ties that differ:", ties)
    assert bad == [], bad
    assert ties <= 50, ties                                         # near ties are rare: count them, not a share


def test_no_seg(case):
    data, _ = case
    bad, ties = check_case(data, None, RESAMPLED, (1, 1, 1), DEV, data_tol=1e-4)
    assert bad == [], bad


def test_mask_crop_and_moments(case):
    data, seg = case
    d, s = dev_case(data, seg, DEV)
    assert np.array_equal(PP.nonzero_mask(d).cpu().numpy(), orc.create_nonzero_mask(data))
    cd, cs, bbox = PP.crop_to_nonzero(d, s)
    rd, rs, rb = orc.crop_to_nonzero(data, seg)
    assert bbox == rb and np.array_equal(cd.cpu().numpy(), rd) and np.array_equal(cs.cpu().numpy(), rs.astype(np.int8))
    z, mom = PP.zscore(cd)
    x = rd.astype(np.float64).reshape(rd.shape[0], -1)
    mean = x.mean(1)
    std = np.sqrt(((x - mean[:, None]) ** 2).mean(1))
    got = mom.cpu().numpy()
    assert np.all(np.abs(got[:, 0] - mean) <= 1e-10 * np.abs(mean)) and np.all(np.abs(got[:, 1] - std) <= 1e-10 * std), (got, mean, std)
    ref = np.stack([orc.zscore(rd[c]) for c in range(rd.shape[0])])
    assert np.abs(z.cpu().numpy() - ref).max() <= 1e-5 * np.abs(ref).max()


def test_all_zero_raises():
    with pytest.raises(ValueError):
        PP.preprocess_case(torch.zeros((2, 9, 10, 11), device=DEV), torch.zeros((9, 10, 11), device=DEV))


def test_bad_labels_raise(case):
    data, seg = case
    d, s = dev_case(data, seg, DEV)
    with pytest.raises(ValueError):
        PP.preprocess_case(d, s * 100)                              # labels up to 300 need int16 in the reference


def test_two_runs_bitwise_equal(case):
    data, seg = case
    d, s = dev_case(data, seg, DEV)
    a = PP.preprocess_case(d, s, spacing=RESAMPLED)
    b = PP.preprocess_case(d, s, spacing=RESAMPLED)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    for k in a[2]["class_locations"]:
        assert np.array_equal(a[2]["class_locations"][k], b[2]["class_locations"][k])
    assert all(np.array_equal(x, y) for x, y in zip(a[2]["intensities_per_channel"], b[2]["intensities_per_channel"]))


def test_device_functions_do_not_sync_and_readbacks_are_counted(case):
    data, seg = case
    d, s = dev_case(data, seg, DEV)
    cd, cs, _ = PP.crop_to_nonzero(d, s)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        PP.nonzero_mask(d)
        z, _ = PP.zscore(cd)
        PP.resample_case(z, cs, (150, 140, 170))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    n0 = PP._readbacks
    PP.preprocess_case(d, s, spacing=RESAMPLED)
    assert PP._readbacks - n0 == PP.READBACKS_PER_CASE == 3


def test_round_trip_through_restore_case(case):
    """a one-hot 'prediction' of the preprocessed seg (-1 -> 0), restored with the case's properties, is the raw label map"""
    data, seg = case
    d, s = dev_case(data, seg, DEV)
    _, oseg, props = PP.preprocess_case(d, s)
    lab = oseg[0].long().clamp(min=0)
    logits = torch.nn.functional.one_hot(lab, 4).permute(3, 0, 1, 2).float().contiguous()
    out = P.restore_case(logits, props, regions=None)
    assert np.array_equal(out.cpu().numpy(), seg[0].astype(np.uint8))
