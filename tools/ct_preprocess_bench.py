"""Time CT case preprocessing on the GPU (preprocess_case(normalization="ct")) for two 512 x 512-slice cases, with CUDA events
after warm-up, and optionally the CPU oracle (oracle/ct_preprocess_oracle.py) on the same case.

    python tools/ct_preprocess_bench.py [--iters 10] [--oracle] [--out ct_preprocess_bench.json]

Workloads (synthetic, one channel of integer HU values on a circular field of view, labels 1 and 2; tests/ct_checks.py):
  lits   1 x 400 x 512 x 512 at (0.7, 0.7, 1.0) -> [1.0, 0.76757812, 0.76757812]
  aiib   1 x 320 x 512 x 512 at (0.7041, 0.7041, 1.0) -> [0.5, 0.70410156, 0.70410156]
Prints the card name and power limit read in the same run and, per workload: ms per whole preprocess_case (readbacks and
host draws included), ms per C-ABI stage from one profiled pass, host ms (the RandomState draws, the readback waits and the
rest), the kernel time and algorithmic GB/s (one read of the line samples, one write of the coefficients) of each prefilter
axis pass from torch.profiler, and with --oracle the oracle's seconds."""
from __future__ import annotations

import argparse
import json
import os
import re
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

from ct_checks import ct_like  # noqa: E402
from metrics_bench import card, timed  # noqa: E402
from segmamba_b200 import _lib  # noqa: E402
from segmamba_b200 import augment as A  # noqa: E402
from segmamba_b200 import plan as PL  # noqa: E402
from segmamba_b200 import preprocess as PP  # noqa: E402

WORKLOADS = {"lits": ((400, 512, 512), (0.7, 0.7, 1.0), [1.0, 0.76757812, 0.76757812]),
             "aiib": ((320, 512, 512), (0.7041, 0.7041, 1.0), [0.5, 0.70410156, 0.70410156])}
GOALS = {"lits_ms": 100.0, "prefilter_gbs": 1000.0}


def prefilter_passes(crop: torch.Tensor, reps: int = 10) -> list:
    """[(kernel, ms, algorithmic GB/s)] of the three axis passes of the edge prefilter of a (n0, n1, n2) crop"""
    n = tuple(crop.shape)
    coef = torch.empty((n[0] + 4) * (n[1] + 4) * (n[2] + 4), device=crop.device)
    job = [A.prefilter_job(crop, coef, n, _lib.AUG_EDGE)]
    A.prefilter(job, crop.device)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            A.prefilter(job, crop.device)
        torch.cuda.synchronize()
    kernels = sorted((e for e in prof.events() if "prefilter" in e.name), key=lambda e: e.time_range.start)
    # whole (axis 0, 1, 2) triples: the trace may miss the first launches, so anchor on the axis-2 kernel of long rows
    rows = [i for i, e in enumerate(kernels) if "rows" in e.name]
    first = rows[0] - 2 if rows[0] >= 2 else rows[0] + 1
    kernels = kernels[first:first + 3 * ((len(kernels) - first) // 3)]
    lines = [n[1] * n[2], (n[0] + 4) * n[2], (n[0] + 4) * (n[1] + 4)]
    out = []
    for axis in range(3):
        ev = kernels[axis::3]
        ms = sum(getattr(e, "device_time", 0.0) or e.cuda_time for e in ev) / len(ev) / 1e3
        nbytes = 4 * lines[axis] * (2 * n[axis] + 4)
        out.append({"axis": axis, "kernel": re.search(r"prefilter\w*", ev[0].name).group(0), "line": n[axis], "ms": round(ms, 4),
                    "gbs": round(nbytes / ms / 1e6, 1)})
    return out


def host_split(run) -> dict:
    """ms of one call spent in the RandomState draws, in the readbacks (waiting for the device) and elsewhere on the host"""
    spent = {"draws": 0.0, "readbacks": 0.0}
    orig = (PP._location_draws, PP._intensity_draws, PP._readback)

    def wrap(fn, key):
        def f(*a, **k):
            t = time.perf_counter()
            try:
                return fn(*a, **k)
            finally:
                spent[key] += time.perf_counter() - t
        return f
    PP._location_draws, PP._intensity_draws, PP._readback = wrap(orig[0], "draws"), wrap(orig[1], "draws"), wrap(orig[2], "readbacks")
    try:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        run()
        torch.cuda.synchronize()
        total = time.perf_counter() - t0
    finally:
        PP._location_draws, PP._intensity_draws, PP._readback = orig
    return {"wall_ms": round(total * 1e3, 2), "draws_ms": round(spent["draws"] * 1e3, 2),
            "readbacks_ms": round(spent["readbacks"] * 1e3, 2),
            "rest_ms": round((total - spent["draws"] - spent["readbacks"]) * 1e3, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--oracle", action="store_true")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ct_preprocess_bench needs a CUDA device")
    dev = "cuda:0"
    res = {"card": card(), "iters": args.iters, "goals": GOALS, "workloads": {}}
    print("card", json.dumps(res["card"]), flush=True)
    for name, (shape, spacing, target) in WORKLOADS.items():
        data, seg = ct_like(shape, seed=7)
        d, s = torch.from_numpy(data).to(dev), torch.from_numpy(seg).to(dev)
        samples, _ = PP.foreground_intensities(d, s)
        props = PL.plan_dataset([spacing], [shape], [samples])["intensity_statistics_per_channel"]
        run = lambda: PP.preprocess_case(d, s, spacing=spacing, target_spacing=target, all_labels=(1, 2), normalization="ct",
                                         intensity_properties=props)
        for _ in range(3):
            out = run()
        ms = timed(run, args.iters)
        host = host_split(run)
        with _lib.profile() as prof:
            run()
        stages = {}
        for (op, _), v in prof.durations().items():
            stages[op] = stages.get(op, 0.0) + sum(v)
        crop, _, _ = PP.crop_to_nonzero(d, s)
        passes = prefilter_passes(PP.ct_normalize(crop, props)[0])
        r = {"shape": (1,) + shape, "spacing": spacing, "target": target, "crop": tuple(crop.shape[1:]),
             "out_shape": tuple(out[0].shape), "ms_per_case": round(ms, 3),
             "stages_ms": {k: round(v, 4) for k, v in sorted(stages.items())}, "host": host, "prefilter": passes}
        if name == "lits":
            r["goal_ms_met"] = ms <= GOALS["lits_ms"]
        r["goal_gbs_met"] = all(p["gbs"] >= GOALS["prefilter_gbs"] for p in passes if p["line"] > 256)
        if args.oracle:
            from oracle import ct_preprocess_oracle as cto
            t0 = time.perf_counter()
            cto.preprocess_case(data, seg, spacing, target, props, all_labels=(1, 2))
            r["oracle_s"] = round(time.perf_counter() - t0, 2)
            r["cpu_threads"] = torch.get_num_threads()
        res["workloads"][name] = r
        print(name, json.dumps(r), flush=True)
        del out, d, s, crop
        torch.cuda.empty_cache()
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
