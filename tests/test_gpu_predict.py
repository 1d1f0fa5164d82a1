"""Case restore and 6-connected component post-processing on the H100 against the oracle (oracle/predict_oracle.py), at the
BraTS size 155 x 240 x 240."""
import numpy as np
import pytest
import torch

from metrics_checks import nested_labels
from oracle import metrics_oracle as morc
from oracle import predict_oracle as orc
from predict_checks import FAMILIES, case_properties, check_cc, check_restore, family, logits_like
from segmamba_b200 import metrics as M
from segmamba_b200 import predict as P

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SHAPE = (155, 240, 240)


@pytest.mark.parametrize("name", FAMILIES)
def test_components_fullsize(name):
    assert check_cc(family(name, SHAPE), DEV) == []


def test_restore_identity_is_exact():
    lg = logits_like((128, 160, 144), seed=1)
    r = check_restore(lg, (128, 160, 144), (14, 40, 48), SHAPE, DEV)
    assert all(v == (0, 0) for v in r.values()), r


def test_restore_resampled():
    """crop shape != logit shape and a margin on every side: labels differ from the oracle only where its two best fp16
    scores are within one fp16 ulp (the kernel rounds the same fp32 products in its own order)."""
    lg = logits_like((128, 128, 128), seed=2)
    r = check_restore(lg, (137, 161, 150), (9, 40, 45), SHAPE, DEV)
    for k, (diff, off_tie) in r.items():
        assert off_tie == 0, (k, r)
        assert diff <= 50, (k, r)                                        # near ties are rare: count them, not a share


def test_batch_equals_single_calls():
    m = torch.from_numpy(family("bernoulli", (64, 80, 72), seed=5)[:1].repeat(3, 0)).to(DEV)
    m[1] = torch.from_numpy(family("brats", (64, 80, 72), seed=6)[0])
    m[2] = torch.from_numpy(family("serpentine", (64, 80, 72))[0])
    lab, cnt = P.label_components(m)
    one = [P.label_components(m[b]) for b in range(3)]
    assert torch.equal(lab, torch.stack([o[0] for o in one])) and torch.equal(cnt, torch.stack([o[1] for o in one]))
    for fn in (P.fill_holes, P.largest_connected_domain):
        assert torch.equal(fn(m), torch.stack([fn(m[b]) for b in range(3)]))


def test_runs_are_bitwise_equal():
    m = torch.from_numpy(family("bernoulli", SHAPE, seed=7)).to(DEV)
    a = P.label_components(m), P.largest_connected_domain(m), P.fill_holes(m)
    b = P.label_components(m), P.largest_connected_domain(m), P.fill_holes(m)
    assert torch.equal(a[0][0], b[0][0]) and torch.equal(a[0][1], b[0][1])
    assert torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])
    lg = logits_like((128, 128, 128), seed=3).to(DEV)
    props = case_properties((137, 161, 150), (9, 40, 45), SHAPE)
    assert torch.equal(P.restore_case(lg, props, postprocess=True), P.restore_case(lg, props, postprocess=True))


def test_no_host_synchronisation():
    lg = torch.randn((1, 4, 128, 128, 128), device=DEV)
    props = case_properties((137, 161, 150), (9, 40, 45), SHAPE)
    m = torch.rand((3,) + SHAPE, device=DEV) < 0.31
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        P.restore_case(lg, props)
        P.restore_case(lg, props, regions=None)
        P.restore_case(lg, props, postprocess=True)
        P.label_components(m)
        P.fill_holes(m)
        P.largest_connected_domain(m)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def test_restore_then_case_metrics():
    """restore_case -> metrics.case_metrics against a raw-geometry ground truth, as the oracle chain computes it (at the
    1 mm BraTS geometry, where the resample is the identity and the restore is exact)."""
    crop, lo = (128, 160, 144), (14, 40, 48)
    lg = logits_like(crop, seed=9)
    gt = nested_labels(SHAPE, seed=9)[0]
    props = case_properties(crop, lo, SHAPE)
    ref_lab = orc.restore(lg, crop, lo, SHAPE, regions=None)
    ref = morc.each_cases_metric(morc.regions_of(ref_lab), morc.regions_of(gt))
    tg = torch.from_numpy(gt[None]).to(DEV)
    got = M.case_metrics(P.restore_case(lg.to(DEV), props, regions=None)[None], tg)
    assert np.array_equal(got, ref), (got, ref)
    got_masks = M.case_metrics(P.restore_case(lg.to(DEV), props).bool()[None], tg)
    assert np.array_equal(got_masks, ref), (got_masks, ref)
    # post-processed regions against the oracle's per-region rule
    pp = P.restore_case(lg.to(DEV), props, postprocess=True).cpu().numpy()
    want = np.stack([orc.largest_connected_domain(r) for r in morc.regions_of(ref_lab)]).astype(np.uint8)
    assert np.array_equal(pp, want)
