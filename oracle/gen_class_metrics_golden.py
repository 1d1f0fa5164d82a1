"""Generate tests/golden/class_metrics_cases.npz from the REFERENCE's own evaluation module (needs the reference checkout).

TEST INFRASTRUCTURE.  What runs is light_training/evaluation/metric.py, unmodified: every ALL_METRICS function on
test = (pred == c), reference = (target == c) per class c, with nan_for_nonexisting True and False.  medpy is not installed, so
`medpy.metric` is stubbed with oracle/class_metrics_oracle.py's hd / hd95 / asd / assd; every confusion-matrix value and every
empty / full rule comes from the reference's code.

    python oracle/gen_class_metrics_golden.py     ->  tests/golden/class_metrics_cases.npz

Cases (labels 0..9 unless noted, classes 1..9):
  organs       1 x 24 x 28 x 30, nine ellipsoid organs, prediction perturbed, unit spacing
  organs_aniso the same volumes at spacing (2.5, 0.9, 0.9), batch 2 with a second seed
  absent       1 x 14 x 16 x 18: class 4 missing from the prediction, 5 from the target, 6 and 7 from both
  full         1 x 6 x 7 x 8: class 1 fills the target, class 2 fills the prediction of a second sample
  wide         1 x 12 x 13 x 14 int16 labels: classes (1, 200, 255), label 300 belongs to no class
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
OUT = os.path.join(ROOT, "tests", "golden", "class_metrics_cases.npz")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _install_medpy_stub():
    from oracle import class_metrics_oracle as orc
    medpy = types.ModuleType("medpy")
    metric = types.ModuleType("medpy.metric")
    metric.hd, metric.hd95, metric.asd, metric.assd = orc.hd, orc.hd95, orc.asd, orc.assd
    medpy.metric = metric
    sys.modules["medpy"], sys.modules["medpy.metric"] = medpy, metric


def cases():
    from class_metrics_checks import organ_labels, perturb_organs
    out = {}
    gt = organ_labels((24, 28, 30), seed=0)
    out["organs"] = (perturb_organs(gt, seed=1), gt, (1.0, 1.0, 1.0), tuple(range(1, 10)))
    gt2 = np.concatenate([gt, organ_labels((24, 28, 30), seed=2)])
    out["organs_aniso"] = (perturb_organs(gt2, seed=3), gt2, (2.5, 0.9, 0.9), tuple(range(1, 10)))
    gt = organ_labels((14, 16, 18), seed=4)
    pred = perturb_organs(gt, seed=5)
    pred[pred == 4] = 0
    gt[gt == 5] = 0
    pred[(pred == 6) | (pred == 7)] = 0
    gt[(gt == 6) | (gt == 7)] = 0
    out["absent"] = (pred, gt, (1.0, 1.0, 1.0), tuple(range(1, 10)))
    rng = np.random.default_rng(6)
    gt = np.stack([np.ones((6, 7, 8), np.int64), rng.integers(0, 3, (6, 7, 8))])
    pred = np.stack([rng.integers(0, 3, (6, 7, 8)), np.full((6, 7, 8), 2, np.int64)])
    out["full"] = (pred, gt, (1.0, 1.0, 1.0), (1, 2))
    gt = organ_labels((12, 13, 14), seed=7)
    wide = np.array([0, 1, 200, 255, 300, 1, 200, 255, 300, 0], dtype=np.int16)
    gt = wide[gt]
    pred = wide[perturb_organs(organ_labels((12, 13, 14), seed=7), seed=8)]
    out["wide"] = (pred, gt, (1.0, 1.0, 1.0), (1, 200, 255))
    return out


def main():
    _install_medpy_stub()
    sys.path.insert(0, REF)
    from light_training.evaluation import metric as ref          # reference module
    data = {}
    for name, (pred, gt, spacing, classes) in cases().items():
        data[f"{name}/pred"], data[f"{name}/gt"] = pred, gt
        data[f"{name}/spacing"], data[f"{name}/classes"] = np.array(spacing), np.array(classes)
        for nan in (True, False):
            vals = np.empty((len(ref.ALL_METRICS), pred.shape[0], len(classes)))
            for b in range(pred.shape[0]):
                for k, c in enumerate(classes):
                    cm = ref.ConfusionMatrix(pred[b] == c, gt[b] == c)
                    for i, fn in enumerate(ref.ALL_METRICS.values()):
                        vals[i, b, k] = fn(confusion_matrix=cm, nan_for_nonexisting=nan, voxel_spacing=spacing)
            data[f"{name}/values_nan{int(nan)}"] = vals
    data["metric_names"] = np.array(list(ref.ALL_METRICS))
    np.savez_compressed(OUT, **data)
    print(f"wrote {OUT}")


if __name__ == "__main__":
    main()
