"""CPU checks of the training-patch loader's host side and of its oracle: the parameter sampler's rates and ranges, the crop
box rules of the reference loader, analytic properties of the oracle (oracle/augment_oracle.py), Philox known answers, and the
ctypes layouts of the smb_aug_* records."""
import math
import os
import re

import numpy as np
import pytest

from oracle import augment_oracle as orc
from segmamba_b200 import _lib
from segmamba_b200 import augment as aug
from segmamba_b200.patch_loader import class_locations_from_seg, get_bbox

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 20000


def _rate_ok(k, n, p):
    return abs(k - n * p) <= 4 * math.sqrt(n * p * (1 - p)) + 1e-9


def _draws(pipeline=True, n=N, C=4):
    s = aug.AugmentSampler(C, pipeline, seed=123)
    return [s.sample() for _ in range(n)]


def test_sampler_rates_and_ranges():
    recs = _draws()
    P = aug.PROBABILITIES
    for key in ("rot", "scale", "noise", "blur", "bright", "contrast", "lowres", "gamma_inv", "gamma"):
        k = sum(r[key] is not None for r in recs)
        assert _rate_ok(k, N, P[key]), (key, k)
    for key, pc in (("blur", P["blur_channel"]), ("lowres", P["lowres_channel"])):
        ch = [v for r in recs if r[key] is not None for v in r[key]]
        assert _rate_ok(sum(v is not None for v in ch), len(ch), pc), key
    mir = np.array([r["mirror"] for r in recs])
    for a in range(3):
        assert _rate_ok(int(mir[:, a].sum()), N, 0.5)
    ang = np.array([r["rot"] for r in recs if r["rot"] is not None])
    assert np.all(np.abs(ang) <= math.pi / 6) and ang.min() < -0.5 and ang.max() > 0.5
    sc = np.array([r["scale"] for r in recs if r["scale"] is not None])
    assert sc.min() >= 0.7 and sc.max() <= 1.4
    assert _rate_ok(int((sc < 1).sum()), len(sc), 0.5)                 # the half/half rule
    nz = np.array([r["noise"] for r in recs if r["noise"] is not None])
    assert nz.min() >= 0 and nz.max() <= 0.1
    for key, lo, hi in (("blur", 0.5, 1.0), ("bright", 0.75, 1.25), ("contrast", 0.75, 1.25), ("lowres", 0.5, 1.0),
                        ("gamma_inv", 0.7, 1.5), ("gamma", 0.7, 1.5)):
        v = np.array([x for r in recs if r[key] is not None for x in r[key] if x is not None])
        assert v.min() >= lo and v.max() <= hi, key
    for key in ("contrast", "gamma"):
        v = np.array([x for r in recs if r[key] is not None for x in r[key]])
        assert _rate_ok(int((v < 1).sum()), len(v), 0.5), key


@pytest.mark.parametrize("pipeline,groups", [(True, {"spatial", "intensity", "mirror"}), ("nomirror", {"spatial", "intensity"}),
                                             ("onlymirror", {"intensity", "mirror"}), ("onlyspatial", {"spatial", "mirror"}),
                                             (False, set())])
def test_pipeline_subsets(pipeline, groups):
    recs = _draws(pipeline, n=3000)
    seen = set()
    for r in recs:
        if r["rot"] is not None or r["scale"] is not None:
            seen.add("spatial")
        if any(r[k] is not None for k in ("noise", "blur", "bright", "contrast", "lowres", "gamma_inv", "gamma")):
            seen.add("intensity")
        if any(r["mirror"]):
            seen.add("mirror")
    assert seen == groups


def test_forced_sampler_draws_everything():
    r = aug.AugmentSampler(4, True, seed=1, force=True).sample()
    assert all(r[k] is not None for k in ("rot", "scale", "noise", "blur", "bright", "contrast", "lowres", "gamma_inv", "gamma"))
    assert all(v is not None for v in r["blur"] + r["lowres"]) and all(r["mirror"])


def test_bbox_bounds_and_foreground():
    rng = np.random.default_rng(0)
    shape, patch = (40, 50, 60), (32, 32, 32)
    seg = np.zeros((1,) + shape, np.int8)
    seg[0, 3:6, 40:44, 50:58] = 2
    locs = class_locations_from_seg(seg, max_per_class=50, seed=0)
    assert list(locs) == [2] and locs[2].shape[1] == 4
    for _ in range(500):
        lbs, ubs = get_bbox(rng, shape, patch, False, locs)
        assert all(0 <= lbs[d] <= shape[d] - patch[d] and ubs[d] - lbs[d] == patch[d] for d in range(3))
        lbs, ubs = get_bbox(rng, shape, patch, True, locs)
        assert any(all(lbs[d] <= v[d + 1] < ubs[d] for d in range(3)) for v in locs[2])
        # the chosen voxel is inside: the crop is centred on it unless that leaves the lower bound
        assert all(lbs[d] >= 0 for d in range(3))


def test_bbox_small_volume_pads_symmetrically():
    rng = np.random.default_rng(0)
    shape, patch = (20, 31, 64), (32, 32, 32)
    for _ in range(200):
        lbs, _ = get_bbox(rng, shape, patch, False, None)
        assert lbs[0] == -(12 // 2)                     # need_to_pad 12: 6 before, 6 after
        assert lbs[1] == 0                              # need_to_pad 1: lower bound 0, upper 0 (the odd voxel goes after)
        assert 0 <= lbs[2] <= 32
    d, s = orc.crop(np.ones((2,) + shape), np.ones(shape, np.int8), [-6, 0, 5], patch)
    assert d.shape == (2,) + patch and d[:, :6].sum() == 0 and d[:, 26:].sum() == 0 and d[:, 6:26, :31].min() == 1
    assert s[:, 31:].sum() == 0


def test_bbox_no_foreground_falls_back_to_random():
    rng = np.random.default_rng(0)
    lbs, _ = get_bbox(rng, (40, 40, 40), (32, 32, 32), True, {1: np.zeros((0, 4), np.int64)})
    assert all(0 <= v <= 8 for v in lbs)


def test_philox_known_answers():
    # Random123 kat_vectors, philox4x32_10
    kat = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
           ((0xffffffff,) * 4, (0xffffffff, 0xffffffff), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
           ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in kat:
        got = orc.philox4x32_10([[v] for v in ctr], key)[:, 0]
        assert tuple(int(v) for v in got) == want


def test_oracle_identity_is_the_crop():
    rng = np.random.default_rng(1)
    x = rng.standard_normal((2, 9, 10, 11))
    s = rng.integers(-1, 4, (9, 10, 11)).astype(np.int8)
    rec = aug.AugmentSampler(2, False).sample()
    img, lab, _ = orc.augment_sample(x, s, rec, 0, 0, 0, aug.spatial_affine)
    assert np.array_equal(img, x) and np.array_equal(lab, np.where(s == -1, 0, s))
    # an identity affine map through the spline path reproduces the volume
    assert np.allclose(orc.resample_data(x[0], np.eye(3, 4)), x[0], atol=1e-12)


def test_oracle_rotation_by_90_degrees_is_a_permutation():
    rng = np.random.default_rng(2)
    P = 15
    x = rng.standard_normal((P, P, P))
    s = rng.integers(0, 4, (P, P, P)).astype(np.int8)
    rec = {"rot": (math.pi / 2, 0.0, 0.0), "scale": None}
    A = aug.spatial_affine(rec, (P, P, P))
    y = orc.resample_data(x, A)
    # src = R^T (o - c) + c with Rx(90): src_y = o_z', src_z = -(o_y - c) + c  ->  y[i, j, k] = x[i, k, P-1-j]
    want = np.transpose(x, (0, 2, 1))[:, ::-1, :]
    assert np.abs(y - want).max() < 1e-9
    ys, _ = orc.resample_seg(s, A)
    assert np.array_equal(ys, np.transpose(s, (0, 2, 1))[:, ::-1, :])


def test_oracle_gamma_retains_mean_and_std():
    rng = np.random.default_rng(3)
    x = rng.standard_normal((8, 9, 10)) * 3 + 1
    for inv in (False, True):
        y = orc.gamma(x, 1.3, inv)
        assert abs(y.mean() - x.mean()) < 1e-9 and abs(y.std() - x.std()) < 1e-6


def test_oracle_noise_is_standard_normal():
    v = orc.normals(200000, 7, 3, 1, 2)
    assert abs(v.mean()) < 0.01 and abs(v.std() - 1) < 0.01
    assert not np.array_equal(v[:100], orc.normals(100, 7, 3, 1, 3))


def _fields(name):
    src = open(os.path.join(ROOT, "include", "segmamba_b200.h")).read()
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), src, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    out = []
    for stmt in filter(None, (s.strip() for s in body.split(";"))):
        decl = re.sub(r"^(const\s+)?(void|float|double|int32_t|int64_t|size_t|smb_aug_\w+)\s*", "", stmt)
        out += [p.replace("*", "").strip() for p in decl.split(",")]
    return out


@pytest.mark.parametrize("cname,pyname", [("smb_aug_case", "AugCase"), ("smb_aug_crop_args", "AugCropArgs"),
                                          ("smb_aug_prefilter_job", "AugPrefilterJob"), ("smb_aug_resample_job", "AugResampleJob"),
                                          ("smb_aug_blur_job", "AugBlurJob"), ("smb_aug_stats_job", "AugStatsJob"),
                                          ("smb_aug_point_job", "AugPointJob"), ("smb_aug_emit_sample", "AugEmitSample"),
                                          ("smb_aug_emit_args", "AugEmitArgs")])
def test_aug_ctypes_structs_match_header(cname, pyname):
    assert [f[0] for f in getattr(_lib, pyname)._fields_] == _fields(cname)
