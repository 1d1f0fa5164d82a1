"""Dice / HD95 on the H100 against the oracle (oracle/metrics_oracle.py) on synthetic BraTS-sized cases."""
import numpy as np
import pytest
import torch

from metrics_checks import check_labels_and_logits, nested_labels, oracle_case, perturb, run_case
from oracle import metrics_oracle as orc
from segmamba_b200 import metrics as M

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SHAPE = (155, 240, 240)


@pytest.fixture(scope="module")
def case():
    gt = nested_labels(SHAPE, seed=0)
    return perturb(gt, seed=1), gt


def test_fullsize_against_oracle():
    r = check_labels_and_logits(SHAPE, DEV)
    unit, aniso = r[(1.0, 1.0, 1.0)], r[(2.5, 0.9, 0.9)]
    assert unit["dice_exact"] and unit["hd_exact"] and unit["hd100_exact"], unit
    assert aniso["dice_exact"] and aniso["hd_err"] <= 1e-12 and aniso["hd100_err"] <= 1e-12, aniso
    assert all(r["logits"].values()), r["logits"]


def test_edge_cases():
    shape = (24, 20, 22)
    gt = nested_labels(shape, seed=5)
    empty = np.zeros_like(gt)
    single = np.zeros_like(gt)
    single[0, 3, 4, 5] = 3
    full = np.full_like(gt, 3)
    for p, g in ((empty, gt), (gt, empty), (empty, empty), (single, gt), (gt, single), (full, gt), (full, full), (single, single)):
        for s in ((1.0, 1.0, 1.0), (2.5, 0.9, 0.9)):
            d_ref, h_ref = oracle_case(p, g, s)
            d, h = run_case(p, g, s, DEV)
            assert np.array_equal(d, d_ref), (d, d_ref)
            assert np.allclose(h, h_ref, rtol=1e-12, atol=0, equal_nan=True), (h, h_ref)


def test_batch_equals_single_calls():
    shape = (40, 48, 44)
    gt = nested_labels(shape, seed=2, batch=2)
    pred = perturb(gt, seed=3)
    tp, tg = torch.from_numpy(pred).to(DEV), torch.from_numpy(gt).to(DEV)
    for fn in (M.dice, lambda a, b: M.hd95(a, b, spacing=(2.5, 0.9, 0.9))):
        both = fn(tp, tg)
        one = torch.cat([fn(tp[b:b + 1], tg[b:b + 1]) for b in range(2)])
        assert torch.equal(both, one)


def test_runs_are_bitwise_equal(case):
    pred, gt = case
    a = run_case(pred, gt, (2.5, 0.9, 0.9), DEV)
    b = run_case(pred, gt, (2.5, 0.9, 0.9), DEV)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def test_no_host_synchronisation(case):
    pred, gt = case
    tp, tg = torch.from_numpy(pred).to(DEV), torch.from_numpy(gt).to(DEV)
    lg = torch.randn((1, 4) + SHAPE, device=DEV)
    masks = torch.stack([torch.isin(tp, torch.tensor(r, device=DEV)) for r in M.BRATS_REGIONS], dim=1)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        M.region_bits(tp)
        M.region_bits(lg)
        M.region_bits(masks)
        M.dice(lg, tg)
        M.hd95(tp, tg)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def test_case_metrics_and_validation_dices(case):
    pred, gt = case
    P, G = orc.regions_of(pred[0]), orc.regions_of(gt[0])
    ref = orc.each_cases_metric(P, G, (1.0, 1.0, 1.0))
    got = M.case_metrics(torch.from_numpy(P[None]).to(DEV), torch.from_numpy(G[None]).to(DEV), (1.0, 1.0, 1.0))
    assert got.shape == (3, 2) and np.array_equal(got, ref), (got, ref)
    empty = np.zeros_like(P)
    got = M.case_metrics(torch.from_numpy(empty[None]).to(DEV), torch.from_numpy(G[None]).to(DEV))
    assert np.array_equal(got, orc.each_cases_metric(empty, G)), got
    # validation_step: logits of a batch of two against the label map, Dice pooled over the batch
    gt2 = nested_labels((64, 64, 64), seed=7, batch=2)
    pr2 = perturb(gt2, seed=8)
    pr2[1] = 0                                                           # one region empty in one sample only
    lg = torch.from_numpy(np.eye(4, dtype=np.float32)[pr2]).permute(0, 4, 1, 2, 3).to(DEV)
    assert M.validation_dices(lg, torch.from_numpy(gt2).to(DEV)) == orc.validation_dices(pr2, gt2)
    z = np.zeros_like(gt2)
    lz = torch.from_numpy(np.eye(4, dtype=np.float32)[z]).permute(0, 4, 1, 2, 3).to(DEV)
    assert M.validation_dices(lz, torch.from_numpy(z).to(DEV)) == orc.validation_dices(z, z) == [1.0, 1.0, 1.0]
    assert M.validation_dices(lz, torch.from_numpy(gt2).to(DEV)) == orc.validation_dices(z, gt2) == [0.0, 0.0, 0.0]
