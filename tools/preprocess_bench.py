"""Time case preprocessing on the GPU (segmamba_b200/preprocess.py) for one BraTS-sized case, with CUDA events after warm-up,
and the CPU oracle (oracle/preprocess_oracle.py, numpy / scipy as the reference runs it) on the same case.

    python tools/preprocess_bench.py [--iters 20] [--out preprocess_bench.json]

The case: synthetic 4 x 155 x 240 x 240 fp32 (an ellipsoidal head on a zero background with an enclosed cavity, nested
labels 2 > 1 > 3), in two modes: identity spacing, and spacing (1.0, 0.8, 1.25) (x, y, z) to 1 mm, which resamples up along z
and down along y.  Prints the card name and power limit read in the same run, ms per case (the whole preprocess_case,
readbacks and host draws included), ms per C-ABI stage from one profiled pass, and the oracle's seconds."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

from metrics_bench import card, timed  # noqa: E402
from oracle import preprocess_oracle as orc  # noqa: E402
from preprocess_checks import brats_like  # noqa: E402
from segmamba_b200 import _lib  # noqa: E402
from segmamba_b200 import preprocess as PP  # noqa: E402

SHAPE = (155, 240, 240)
MODES = {"identity": (1.0, 1.0, 1.0), "resampled": (1.0, 0.8, 1.25)}
GOALS_MS = {"identity": 10.0, "resampled": 25.0}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("preprocess_bench needs a CUDA device")
    dev = "cuda:0"
    data, seg = brats_like(SHAPE, channels=4, seed=0)
    d, s = torch.from_numpy(data).to(dev), torch.from_numpy(seg).to(dev)
    res = {"card": card(), "shape": (4,) + SHAPE, "iters": args.iters, "modes": {}}
    for mode, spacing in MODES.items():
        run = lambda: PP.preprocess_case(d, s, spacing=spacing)
        for _ in range(3):
            run()
        ms = timed(run, args.iters)
        with _lib.profile() as prof:
            out = run()
        stages = {}
        for (op, _), v in prof.durations().items():
            stages[op] = stages.get(op, 0.0) + sum(v)
        t0 = time.perf_counter()
        orc.preprocess_case(data, seg, spacing)
        cpu = time.perf_counter() - t0
        res["modes"][mode] = {"ms_per_case": ms, "goal_ms": GOALS_MS[mode], "goal_met": ms <= GOALS_MS[mode],
                              "out_shape": tuple(out[0].shape), "stages_ms": {k: round(v, 4) for k, v in sorted(stages.items())},
                              "oracle_s": cpu, "cpu_threads": torch.get_num_threads()}
        print(mode, json.dumps(res["modes"][mode]), flush=True)
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
