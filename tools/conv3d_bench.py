"""Native 3x3x3 convolution (smb_conv3d / smb_conv3d_wgrad) against cuDNN, per model shape and pass, at batch 2 in bf16.

    python tools/conv3d_bench.py [--reps 20] [--edges 128,64,32,16,8] [--out bench_out/conv3d_bench.json]

For every 3x3x3 convolution shape of the default SegMamba, times the forward, data-gradient and weight-gradient pass of
  native        the implicit-GEMM kernel of libsegmamba_b200
  cudnn         cuDNN with torch.backends.cudnn.benchmark = False (the heuristic plan the training step runs)
  cudnn_tuned   cuDNN with benchmark = True (the library's best plan for the shape)
as the median of CUDA-event timings after warm-up, rotating over enough input copies that the inputs exceed the 50 MB L2.
Reports TFLOP/s (2 x voxels x 27 x C_in x C_out per pass) and the fraction of the H100 SXM data sheet's 989 dense bf16
TFLOP/s, with the card name and power limit read in the same run.  conv3d.NATIVE_PASSES is set from this table."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK = 989.0
# (C_in, C_out, edge, count in one forward of the default model)
SHAPES = [(48, 48, 128, 4), (96, 48, 128, 1),
          (48, 48, 64, 2), (48, 96, 64, 1), (96, 96, 64, 2), (192, 96, 64, 1),
          (96, 96, 32, 2), (96, 192, 32, 1), (192, 192, 32, 2), (384, 192, 32, 1),
          (192, 192, 16, 2), (192, 384, 16, 1), (384, 384, 16, 2), (768, 384, 16, 1),
          (384, 384, 8, 2), (384, 768, 8, 1), (768, 768, 8, 1)]


def card() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, clk = [v.strip() for v in q.split(",")]
        return {"name": name, "power_limit": pl, "max_sm_clock": clk}
    except Exception as e:                                                # report, do not guess
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"unknown ({e})"}


def median_ms(fn, n_bufs, reps, warmup=3):
    for i in range(warmup):
        fn(i % n_bufs)
    torch.cuda.synchronize()
    times = []
    for i in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn(i % n_bufs)
        e.record()
        times.append((s, e))
    torch.cuda.synchronize()
    return statistics.median(s.elapsed_time(e) for s, e in times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--edges", default="128,64,32,16,8")
    ap.add_argument("--out", default=os.path.join(ROOT, "bench_out", "conv3d_bench.json"))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "conv3d_bench.py needs a CUDA device"
    from segmamba_b200 import conv3d as C
    edges = {int(e) for e in args.edges.split(",")}
    dt, cl = torch.bfloat16, torch.channels_last_3d
    rows = []
    for ci, co, edge, count in SHAPES:
        if edge not in edges:
            continue
        vox = 2 * edge ** 3
        flop = 2.0 * vox * 27 * ci * co
        n_bufs = max(1, -(-(100 << 20) // (vox * (ci + co) * 2)))
        g = torch.Generator(device="cuda").manual_seed(0)
        xs = [torch.randn(2, ci, edge, edge, edge, device="cuda", generator=g).to(dt).contiguous(memory_format=cl) for _ in range(n_bufs)]
        dys = [torch.randn(2, co, edge, edge, edge, device="cuda", generator=g).to(dt).contiguous(memory_format=cl) for _ in range(n_bufs)]
        w = (torch.randn(co, ci, 3, 3, 3, device="cuda", generator=g) / (27 * ci) ** 0.5).to(dt).contiguous(memory_format=cl)
        x5s = [x.permute(0, 2, 3, 4, 1) for x in xs]
        dy5s = [d.permute(0, 2, 3, 4, 1) for d in dys]
        w5 = w.permute(0, 2, 3, 4, 1)
        native = {"fprop": lambda i: C.conv3d_fwd(x5s[i], w5), "dgrad": lambda i: C.conv3d_dgrad(dy5s[i], w5),
                  "wgrad": lambda i: C.conv3d_wgrad(x5s[i], dy5s[i])}

        def lib(i, mask):
            return torch.ops.aten.convolution_backward(dys[i], xs[i], w, None, [1, 1, 1], [1, 1, 1], [1, 1, 1], False, [0, 0, 0], 1, mask)
        cudnn = {"fprop": lambda i: F.conv3d(xs[i], w, None, 1, 1), "dgrad": lambda i: lib(i, [True, False, False]),
                 "wgrad": lambda i: lib(i, [False, True, False])}
        for ps in ("fprop", "dgrad", "wgrad"):
            r = {"c_in": ci, "c_out": co, "edge": edge, "batch": 2, "count": count, "pass": ps, "gflop": flop / 1e9}
            r["native_ms"] = median_ms(native[ps], n_bufs, args.reps)
            torch.backends.cudnn.benchmark = False
            r["cudnn_ms"] = median_ms(cudnn[ps], n_bufs, args.reps)
            torch.backends.cudnn.benchmark = True
            r["cudnn_tuned_ms"] = median_ms(cudnn[ps], n_bufs, args.reps)
            torch.backends.cudnn.benchmark = False
            for k in ("native", "cudnn", "cudnn_tuned"):
                r[k + "_tflops"] = flop / (r[k + "_ms"] * 1e-3) / 1e12
                r[k + "_frac_peak"] = r[k + "_tflops"] / PEAK
            rows.append(r)
        del xs, dys, x5s, dy5s
        torch.cuda.empty_cache()
    c = card()
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump({"card": c, "peak_tflops_datasheet": PEAK, "rows": rows}, f, indent=1)
    print(f"card: {c['name']}, power limit {c['power_limit']}, max SM clock {c.get('max_sm_clock')}; "
          f"fractions of the {PEAK:.0f} TFLOP/s data-sheet peak")
    print(f"{'shape':>18} {'pass':>6} {'native ms':>10} {'TF/s':>6} {'frac':>5} | {'cudnn ms':>9} {'TF/s':>6} | {'tuned ms':>9} {'TF/s':>6}")
    for r in rows:
        print(f"{r['c_in']:>4}->{r['c_out']:<4} @{r['edge']:>3}^3 {r['pass']:>6} {r['native_ms']:10.3f} {r['native_tflops']:6.0f} "
              f"{r['native_frac_peak']:5.2f} | {r['cudnn_ms']:9.3f} {r['cudnn_tflops']:6.0f} | {r['cudnn_tuned_ms']:9.3f} {r['cudnn_tuned_tflops']:6.0f}")


if __name__ == "__main__":
    main()
