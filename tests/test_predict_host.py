"""CPU checks of the prediction semantics: analytic cases of the oracle (oracle/predict_oracle.py), the parsing of the
reference's per-case properties, and the ctypes layouts of the prediction C ABI against the header."""
import os
import re

import numpy as np
import pytest
import torch

from oracle import predict_oracle as orc
from segmamba_b200 import _lib
from segmamba_b200 import predict as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _shell(n=9):
    m = np.zeros((n, n, n), bool)
    m[1:-1, 1:-1, 1:-1] = True
    m[3:-3, 3:-3, 3:-3] = False                                          # a closed cavity
    return m


def test_hole_is_filled():
    m = _shell()
    f = orc.fill_holes(m)
    assert f[1:-1, 1:-1, 1:-1].all() and f.sum() == 7 ** 3
    assert orc.largest_connected_domain(m).sum() == 7 ** 3


def test_tunnel_to_the_border_is_not_a_hole():
    m = _shell()
    m[4, 4, :3] = False                                                  # the cavity opens through the wall to the border
    f = orc.fill_holes(m)
    assert np.array_equal(f, m)


def test_equal_components_keep_the_highest_label():
    m = np.zeros((4, 6, 6), bool)
    m[0, 0, :3] = True                                                   # label 1, three voxels
    m[3, 5, 3:] = True                                                   # label 2, three voxels
    lab, n = orc.label(m)
    assert n == 2 and lab[3, 5, 5] == 2
    assert np.array_equal(orc.largest_connected_domain(m), lab == 2)


def test_diagonal_contact_is_two_components():
    m = np.zeros((3, 3, 3), bool)
    m[0, 0, 0] = m[1, 1, 0] = m[2, 2, 2] = True                           # edge and corner contacts only
    lab, n = orc.label(m)
    assert n == 3 and lab[0, 0, 0] == 1 and lab[1, 1, 0] == 2 and lab[2, 2, 2] == 3
    e = np.zeros((2, 2, 2), bool)
    assert orc.label(e)[1] == 0 and not orc.largest_connected_domain(e).any()


def test_restore_oracle_identity_and_uncrop():
    lg = torch.randn(4, 3, 4, 5)
    lab = orc.restore(lg, (3, 4, 5), (1, 0, 2), (5, 4, 9), regions=None)
    assert lab.shape == (5, 4, 9) and lab.dtype == np.uint8
    assert np.array_equal(lab[1:4, :, 2:7], lg.half().argmax(0).numpy())
    assert lab[0].sum() == 0 and lab[4].sum() == 0 and lab[:, :, :2].sum() == 0
    masks = orc.restore(lg, (3, 4, 5), (1, 0, 2), (5, 4, 9))
    assert masks.shape == (3, 5, 4, 9) and np.array_equal(masks[2], (lab == 3).astype(np.uint8))


def _props(crop=(3, 4, 5), full=(5, 6, 9), bbox=((1, 4), (2, 6), (0, 5))):
    return {"shape_after_cropping_before_resample": crop, "shape_before_cropping": full, "bbox_used_for_cropping": bbox}


def test_properties_accept_collated_values():
    want = ((3, 4, 5), (1, 2, 0), (5, 6, 9))
    assert P.case_geometry(_props()) == want
    collated = _props(crop=[torch.tensor([3]), np.int64(4), np.array([5])], full=[torch.tensor([5]), torch.tensor([6]), torch.tensor([9])],
                      bbox=[[torch.tensor([1]), torch.tensor([4])], [np.int32(2), 6], torch.tensor([0, 5])])
    assert P.case_geometry(collated) == want
    assert P.case_geometry(_props(crop=torch.tensor([3, 4, 5]))) == want


@pytest.mark.parametrize("props", [
    _props(bbox=((1, 4), (2, 6), (5, 10))),                              # past the upper edge
    _props(bbox=((-1, 2), (2, 6), (0, 5))),                              # below zero
    _props(bbox=((1, 5), (2, 6), (0, 5))),                               # extent differs from the crop shape
    _props(crop=(3, 4)),
    _props(crop=(3, 4, 5.5)),
    _props(crop=(3, torch.tensor([4, 4]), 5)),
    {"shape_before_cropping": (5, 6, 9), "bbox_used_for_cropping": ((1, 4), (2, 6), (0, 5))},
])
def test_properties_errors(props):
    with pytest.raises(ValueError):
        P.case_geometry(props)


def test_rejects_cpu_and_bad_arguments():
    with pytest.raises(RuntimeError):
        P.label_components(torch.zeros(2, 3, 4, dtype=torch.bool))
    with pytest.raises(RuntimeError):
        P.restore_case(torch.zeros(4, 3, 4, 5), _props())


def _fields(name):
    src = open(os.path.join(ROOT, "include", "segmamba_b200.h")).read()
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), src, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    out = []
    for stmt in filter(None, (s.strip() for s in body.split(";"))):
        decl = re.sub(r"^(const\s+)?(void|uint8_t|int32_t|int64_t|size_t)\s*", "", stmt)
        out += [re.sub(r"\[.*\]", "", p).replace("*", "").strip() for p in decl.split(",")]
    return out


@pytest.mark.parametrize("cname,pyname", [("smb_pred_restore_args", "PredRestoreArgs"), ("smb_pred_cc_args", "PredCcArgs")])
def test_pred_ctypes_structs_match_header(cname, pyname):
    assert [f[0] for f in getattr(_lib, pyname)._fields_] == _fields(cname)


def test_pred_constants_match_header():
    src = open(os.path.join(ROOT, "include", "segmamba_b200.h")).read()
    assert "SMB_PRED_LABEL = 0, SMB_PRED_FILL_HOLES = 1, SMB_PRED_LARGEST = 2" in src
    assert (_lib.PRED_LABEL, _lib.PRED_FILL_HOLES, _lib.PRED_LARGEST) == (0, 1, 2)
