"""Time Dice + HD95 of one BraTS-sized case (155 x 240 x 240, regions TC / WT / ET) on the GPU, stage by stage, with CUDA
events after warm-up, and the scipy oracle on the same case on the CPU.

    python tools/metrics_bench.py [--iters 20] [--oracle-reps 1] [--out metrics_bench.json]

Prints the card name and power limit read in the same run, ms per stage with the algorithmic bytes each stage must move, and
the oracle's seconds with the CPU thread count."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from metrics_checks import nested_labels, perturb  # noqa: E402
from oracle import metrics_oracle as orc  # noqa: E402
from segmamba_b200 import metrics as M  # noqa: E402

SHAPE = (155, 240, 240)


def card() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, clk = [v.strip() for v in q.split(",")]
        return {"name": name, "power_limit": pl, "max_sm_clock": clk}
    except Exception as e:                                                # report, do not guess
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"unknown ({e})"}


def timed(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--oracle-reps", type=int, default=1)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    dev = "cuda:0"
    gt = nested_labels(SHAPE, seed=0)
    pred = perturb(gt, seed=1)
    tp, tg = torch.from_numpy(pred).to(dev), torch.from_numpy(gt).to(dev)
    R, n = 3, int(np.prod(SHAPE))
    pb, gb = M._prepare(tp, tg, M.BRATS_REGIONS)
    counts, pbd, gbd = M._counts(pb, gb, R)
    stages = {
        "region_bits x2 (int64 labels)": (lambda: M._prepare(tp, tg, M.BRATS_REGIONS), 2 * n * (8 + 1)),
        "counts + borders": (lambda: M._counts(pb, gb, R), n * 4),
        "edt + select (6 jobs)": (lambda: M._hd_from(counts.clone(), pbd, gbd, (1.0, 1.0, 1.0), 95.0),
                                  2 * R * n * (1 + 4 + 4 + 4 + 4 + 4 + 1)),
        "dice + hd95 end to end": (lambda: (M.dice(tp, tg), M.hd95(tp, tg)), None),
    }
    for fn, _ in stages.values():                                          # warm-up: module load, allocator
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    res = {"card": card(), "shape": SHAPE, "regions": R, "stages": {}}
    for name, (fn, nbytes) in stages.items():
        ms = timed(fn, args.iters)
        res["stages"][name] = {"ms": round(ms, 4), "algorithmic_bytes": nbytes,
                               "GB_per_s": round(nbytes / ms / 1e6, 1) if nbytes else None}
    case = lambda: M.case_metrics(torch.stack([torch.isin(tp, torch.tensor(r, device=dev)) for r in M.BRATS_REGIONS], 1),
                                  torch.stack([torch.isin(tg, torch.tensor(r, device=dev)) for r in M.BRATS_REGIONS], 1))
    case()
    t0 = time.perf_counter()
    for _ in range(args.iters):
        case()
    res["case_metrics_ms_incl_readback"] = round((time.perf_counter() - t0) / args.iters * 1e3, 3)
    P, G = orc.regions_of(pred[0]), orc.regions_of(gt[0])
    t0 = time.perf_counter()
    for _ in range(args.oracle_reps):
        ref = orc.each_cases_metric(P, G, (1.0, 1.0, 1.0))
    res["oracle_cpu_s_per_case"] = round((time.perf_counter() - t0) / args.oracle_reps, 3)
    res["cpu_threads"] = os.cpu_count()
    res["matches_oracle"] = bool(np.array_equal(case(), ref))
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
