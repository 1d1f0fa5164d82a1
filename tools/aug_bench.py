"""Measure the GPU patch loader (segmamba_b200/patch_loader.py) and print one JSON line.

    python tools/aug_bench.py [--batches 20] [--steps 10] [--skip-oracle]

* ms per batch (B=2, 4x128^3, fp32) at the reference probabilities and with every transform forced, with a CUDA-event time per
  C-ABI stage (the whole job list of one call) and the HBM bytes each stage needs;
* ms per TrainStep (the README's SegMamba, bf16) fed by the loader with and without augmentation, on synthetic BraTS-sized
  cases (4x155x240x240, blob labels, seeded), against the same step fed from a fixed batch;
* seconds per forced sample of the CPU oracle (numpy / scipy, float64) on this host, with its thread and core counts.
The card's name and power limit are read in the same run.
"""
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
sys.path.insert(0, ROOT)

from segmamba_b200 import _lib  # noqa: E402
from segmamba_b200.patch_loader import GpuPatchLoader, class_locations_from_seg  # noqa: E402

PATCH = (128, 128, 128)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as e:                                           # noqa: BLE001
        return torch.cuda.get_device_name(0), f"unknown ({e})"


def brats_cases(n, seed, device):
    rng = np.random.default_rng(seed)
    shape = (155, 240, 240)
    g = np.meshgrid(*[np.arange(s, dtype=np.float32) for s in shape], indexing="ij")
    cases = []
    for i in range(n):
        ctr = np.array([rng.uniform(50, 105), rng.uniform(80, 160), rng.uniform(80, 160)])
        r = np.sqrt(sum(((g[d] - ctr[d]) / (30 + 10 * rng.random())) ** 2 for d in range(3)))
        seg = np.where(r < 0.4, 3, np.where(r < 0.7, 1, np.where(r < 1.0, 2, 0))).astype(np.int8)[None]
        data = (rng.standard_normal((4,) + shape, dtype=np.float32) * 0.3 + seg.astype(np.float32))
        cases.append({"data": torch.from_numpy(data).to(device), "seg": torch.from_numpy(seg).to(device),
                      "class_locations": class_locations_from_seg(seg, 10000, seed=i)})
    return cases


def stage_bytes():
    """HBM bytes one call of each C-ABI stage needs in a forced batch (B=2, C=4, 128^3): reads + writes of every pass, fp32 = 4 B,
    labels 1 B; gathered taps counted once (their lines are reused out of L1 / L2)."""
    v = PATCH[0] * PATCH[1] * PATCH[2]
    e = (PATCH[0] + 4) * (PATCH[1] + 4) * (PATCH[2] + 4)
    B, C = 2, 4
    bc = B * C
    return {
        "smb_aug_crop": B * v * (4 * C * 2 + 2),
        "smb_aug_prefilter": bc * 4 * (v + e) + bc * 4 * 2 * 2 * e,           # axis 0 read src + write coef, axes 1, 2 in place
        "smb_aug_resample": bc * 4 * (e + v) + B * 2 * v,                      # one cubic pass (coef read once from L2-resident lines)
        "smb_aug_blur": bc * 3 * 2 * 4 * v,
        "smb_aug_stats": bc * 4 * v,
        "smb_aug_pointwise": bc * 2 * 4 * v,
        "smb_aug_emit": B * v * (4 * C * 2 + 1 + 8),
    }


def time_batches(loader, n):
    for _ in range(3):
        next(loader)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        next(loader)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / n * 1e3


def breakdown(loader, n):
    with _lib.profile() as prof:
        for _ in range(n):
            next(loader)
    d = prof.durations()
    per = {}
    for (op, _), ts in d.items():
        per.setdefault(op, []).extend(ts)
    return {op: {"ms_per_batch": sum(ts) / n, "calls_per_batch": len(ts) / n} for op, ts in per.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=20)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--skip-oracle", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("aug_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    name, power = card()
    res = {"card": name, "power_limit": power, "batch": 2, "channels": 4, "patch": list(PATCH)}
    cases = brats_cases(4, 0, dev)

    for label, force in (("reference_p", False), ("forced", True)):
        ld = GpuPatchLoader(cases, PATCH, batch_size=2, seed=1, force=force, device=dev)
        res[f"ms_per_batch_{label}"] = time_batches(ld, args.batches)
        res[f"stages_{label}"] = breakdown(ld, max(5, args.batches // 2))
    nbytes = stage_bytes()
    for op, rec in res["stages_forced"].items():
        if op in nbytes:
            per_call = nbytes[op]                                     # every call of a forced batch covers all pairs
            rec["bytes_per_batch"] = per_call * rec["calls_per_batch"]
            rec["GBps"] = rec["bytes_per_batch"] / (rec["ms_per_batch"] * 1e-3) / 1e9
    res["ms_per_batch_crop_only"] = time_batches(GpuPatchLoader(cases, PATCH, batch_size=2, seed=1, augmentation=False, device=dev),
                                                 args.batches)

    # TrainStep fed by the loader
    from segmamba_b200.segmamba import SegMamba
    from segmamba_b200.train_step import TrainStep, reference_optimizer
    torch.manual_seed(0)
    m = SegMamba(in_chans=4, out_chans=4, depths=[2, 2, 2, 2], feat_size=[48, 96, 192, 384]).to(dev)
    step = TrainStep(m, reference_optimizer(m), torch.nn.CrossEntropyLoss())
    fixed = next(GpuPatchLoader(cases, PATCH, batch_size=2, seed=2, augmentation=False, device=dev))

    def run(feed, n):
        for _ in range(2):
            step(*feed())
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(n):
            step(*feed())
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / n * 1e3

    la = GpuPatchLoader(cases, PATCH, batch_size=2, seed=3, device=dev)
    ln = GpuPatchLoader(cases, PATCH, batch_size=2, seed=3, augmentation=False, device=dev)
    lf = GpuPatchLoader(cases, PATCH, batch_size=2, seed=3, force=True, device=dev)
    res["ms_per_step_fixed_batch"] = run(lambda: fixed, args.steps)
    res["ms_per_step_loader_augmented"] = run(lambda: next(la), args.steps)
    res["ms_per_step_loader_forced"] = run(lambda: next(lf), args.steps)
    res["ms_per_step_loader_no_aug"] = run(lambda: next(ln), args.steps)
    res["ms_per_step_fixed_batch_again"] = run(lambda: fixed, args.steps)

    if not args.skip_oracle:
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        from oracle import augment_oracle as orc
        from segmamba_b200 import augment as aug
        sampler = aug.AugmentSampler(4, True, seed=0, force=True)
        rec = sampler.sample()
        x = np.random.default_rng(0).standard_normal((4,) + PATCH).astype(np.float32)
        s = (np.random.default_rng(1).random(PATCH) * 4).astype(np.int8)
        t0 = time.perf_counter()
        orc.augment_sample(x, s, rec, 0, 0, 0, aug.spatial_affine)
        res["oracle_s_per_forced_sample"] = time.perf_counter() - t0
        res["oracle_host"] = {"cpu_count": os.cpu_count(), "torch_threads": torch.get_num_threads(),
                              "omp_num_threads": os.environ.get("OMP_NUM_THREADS")}
    res["target_ms_forced"] = 17.0
    print(json.dumps(res))


if __name__ == "__main__":
    main()
