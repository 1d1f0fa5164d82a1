"""Time case restore and connected-component post-processing on the GPU (segmamba_b200/predict.py) for one BraTS-sized
case, with CUDA events after warm-up, and the CPU oracle on the same work.

    python tools/predict_bench.py [--iters 20] [--out predict_bench.json]

The case: synthetic fp32 logits (4, 155, 240, 240) (nested BraTS-like labels, one-hot scaled by 2, plus unit Gaussian noise,
so the region masks carry speckle and many small components), restored at identity size and into a (140, 200, 190) crop
at a margin of a 155 x 240 x 240 volume.  Prints the card name and power limit read in the same run, ms per stage with the
algorithmic bytes of the streaming restore pass, and the oracle's seconds with the CPU thread count."""
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

from metrics_bench import card, timed  # noqa: E402
from oracle import predict_oracle as orc  # noqa: E402
from predict_checks import case_properties, logits_like  # noqa: E402
from segmamba_b200 import predict as P  # noqa: E402

SHAPE = (155, 240, 240)
CROP, LO = (140, 200, 190), (7, 20, 25)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    dev = "cuda:0"
    lg_cpu = logits_like(SHAPE, seed=0)
    lg = lg_cpu.to(dev)
    C, n = lg.shape[0], int(np.prod(SHAPE))
    ident = case_properties(SHAPE, (0, 0, 0), SHAPE)
    resized = case_properties(CROP, LO, SHAPE)
    masks = P.restore_case(lg, ident)
    R = masks.shape[0]
    stages = {
        # logits read once, R uint8 masks written
        "restore identity": (lambda: P.restore_case(lg, ident), C * 4 * n + R * n),
        "restore resized": (lambda: P.restore_case(lg, resized), C * 4 * n + R * n),
        "label_components x3": (lambda: P.label_components(masks), None),
        "largest_connected_domain x3": (lambda: P.largest_connected_domain(masks), None),
        "restore + postprocess (identity)": (lambda: P.restore_case(lg, ident, postprocess=True), None),
        "restore + postprocess (resized)": (lambda: P.restore_case(lg, resized, postprocess=True), None),
    }
    for fn, _ in stages.values():                                          # warm-up: module load, allocator
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    res = {"card": card(), "shape": SHAPE, "classes": C, "regions": R, "crop": CROP, "stages": {}}
    for name, (fn, nbytes) in stages.items():
        ms = timed(fn, args.iters)
        res["stages"][name] = {"ms": round(ms, 4), "algorithmic_bytes": nbytes,
                               "GB_per_s": round(nbytes / ms / 1e6, 1) if nbytes else None}
    res["components_per_region"] = P.label_components(masks)[1].tolist()
    # the same work on the CPU: oracle restore, then label and largest_connected_domain per region
    m = masks.cpu().numpy()
    t0 = time.perf_counter()
    ref = orc.restore(lg_cpu, SHAPE, (0, 0, 0), SHAPE)
    t1 = time.perf_counter()
    for r in range(R):
        orc.label(ref[r])
    t2 = time.perf_counter()
    big = np.stack([orc.largest_connected_domain(ref[r]) for r in range(R)])
    t3 = time.perf_counter()
    res["oracle_cpu_s"] = {"restore identity": round(t1 - t0, 3), "label x3": round(t2 - t1, 3),
                           "largest_connected_domain x3": round(t3 - t2, 3)}
    res["cpu_threads"] = os.cpu_count()
    res["matches_oracle"] = bool(np.array_equal(m, ref)
                                 and np.array_equal(P.largest_connected_domain(masks).cpu().numpy(), big))
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
