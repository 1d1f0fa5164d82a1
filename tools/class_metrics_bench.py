"""Time per-class evaluation (metrics.class_metrics, all 19 metrics) on the GPU: an AbdomenAtlas-like nine-organ case at
1 x 400 x 512 x 512, spacing (1.0, 0.8, 0.8), and the BraTS-size case (labels 1, 2, 3 as classes at 155 x 240 x 240) beside
tools/metrics_bench.py.

    python tools/class_metrics_bench.py [--iters 10] [--oracle] [--out class_metrics_bench.json]

Prints the card name and power limit read in the same run; ms per call on the host clock around the whole call (both readbacks
included); per-stage CUDA-event times from one profiled call; the peak device memory the call allocates beyond its inputs; and,
with --oracle, the CPU oracle's seconds on the same case."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

from class_metrics_checks import ct_organs  # noqa: E402
from metrics_bench import card  # noqa: E402
from metrics_checks import nested_labels, perturb  # noqa: E402
from oracle import class_metrics_oracle as orc  # noqa: E402
from segmamba_b200 import _lib  # noqa: E402
from segmamba_b200 import metrics as M  # noqa: E402


def bench(name, pred, gt, classes, spacing, iters, oracle):
    dev = "cuda:0"
    tp, tg = torch.from_numpy(pred).to(dev), torch.from_numpy(gt).to(dev)
    call = lambda: M.class_metrics(tp, tg, classes=classes, spacing=spacing)
    for _ in range(2):                                                     # warm-up: module load, allocator
        call()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        t0 = time.perf_counter()
        call()                                                             # ends in its second readback
        times.append((time.perf_counter() - t0) * 1e3)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    with _lib.profile() as prof:
        call()
    stages = {op: round(sum(v), 3) for (op, _), v in prof.durations().items()}
    peak = torch.cuda.max_memory_allocated() - base
    res = {"case": name, "shape": list(pred.shape), "classes": list(classes), "spacing": list(spacing),
           "ms_per_call": {"min": round(min(times), 2), "median": round(float(np.median(times)), 2), "max": round(max(times), 2)},
           "stage_ms": stages, "workspace_peak_MB": round(peak / 2**20, 1)}
    if oracle:
        t0 = time.perf_counter()
        orc.class_table(pred, gt, classes, spacing)
        res["oracle_s"] = round(time.perf_counter() - t0, 2)
        res["oracle_threads"] = os.cpu_count()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--oracle", action="store_true")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    res = {"card": card(), "cases": []}
    pred, gt = ct_organs((400, 512, 512), seed=3)
    res["cases"].append(bench("ct_9_organs", pred, gt, tuple(range(1, 10)), (1.0, 0.8, 0.8), args.iters, args.oracle))
    gt = nested_labels((155, 240, 240), seed=0)
    res["cases"].append(bench("brats_3_classes", perturb(gt, seed=1), gt, (1, 2, 3), (1.0, 1.0, 1.0), args.iters, args.oracle))
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
