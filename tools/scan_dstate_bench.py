"""Timing of the selective scan at 16 / 32 / 64 states on one H100, plus the bf16 training step with d_state 32 / 64.

1. `selective_scan_cuda.fwd` / `.bwd` at the stage-0 mixer shape (batch 2, 96 channels, L = 262144, bf16): the native drop-in
   against the reference's own extension (oracle/_ref/selective_scan_cuda.so, oracle/build_ref.py).  The arms run alternately,
   one block of `--iters` calls per arm and round, each block timed with CUDA events; the JSON reports the median block over
   `--rounds`.  The native "model path" row times what the mixer runs: the forward keeping the 256-position and the dense
   checkpoints, and the backward that consumes them.
2. One bf16 training step (the bench.py step: SegMamba 128^3 patch, batch 2, cross entropy, clip, SGD) with every MambaLayer at
   d_state 16 / 32 / 64: median ms/step over `--steps` steps and the peak of torch.cuda.max_memory_allocated.

usage: python tools/scan_dstate_bench.py [--iters 5] [--rounds 5] [--steps 10] [--out result.json]
"""
import argparse
import importlib.util
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def load_ref():
    path = os.path.join(ROOT, "oracle", "_ref", "selective_scan_cuda.so")
    if not os.path.exists(path):
        return None
    spec = importlib.util.spec_from_file_location("selective_scan_cuda", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def block_ms(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / iters


def scan_inputs(N, batch=2, dim=96, L=262144, dtype=torch.bfloat16):
    g = torch.Generator(device="cuda").manual_seed(N)
    r = lambda *s: torch.randn(*s, generator=g, device="cuda")
    d = dict(u=r(batch, dim, L).to(dtype), delta=(0.5 * r(batch, dim, L) - 4.0).to(dtype), z=r(batch, dim, L).to(dtype),
             dout=r(batch, dim, L).to(dtype), B=r(batch, 1, N, L).to(dtype), C=r(batch, 1, N, L).to(dtype),
             A=-torch.arange(1, N + 1, dtype=torch.float32, device="cuda").repeat(dim, 1).contiguous(), D=r(dim),
             bias=0.1 * r(dim))
    return d


def scan_timings(states, iters, rounds):
    from segmamba_b200 import selective_scan_cuda as ssc
    ref = load_ref()
    rows = {}
    for N in states:
        d = scan_inputs(N)
        a = (d["u"], d["delta"], d["A"], d["B"], d["C"], d["D"], d["z"], d["bias"], True)
        mo = ssc.fwd(*a)
        arms = {"native_fwd": lambda: ssc.fwd(*a),
                "native_bwd": lambda: ssc.bwd(*a[:8], d["dout"], mo[1], mo[0], None, True, False)}
        _, _, _, hst, hd = ssc.fwd_ex(*a, want_out=False, want_x=False, want_hstates=True, want_hdense=True)
        arms["native_model_fwd"] = lambda: ssc.fwd_ex(*a, want_out=False, want_x=False, want_hstates=True, want_hdense=True)
        arms["native_model_bwd"] = lambda: ssc.bwd_ex(*a[:8], d["dout"], None, True, False, hstates=hst, hdense=hd)
        if ref is not None:
            ro = ref.fwd(*a)
            arms["ref_fwd"] = lambda: ref.fwd(*a)
            arms["ref_bwd"] = lambda: ref.bwd(*a[:8], d["dout"], ro[1], ro[0], None, True, False)
        for fn in arms.values():                           # warm-up: module load, allocator, first launches
            fn()
        times = {k: [] for k in arms}
        for _ in range(rounds):
            for k, fn in arms.items():
                times[k].append(block_ms(fn, iters))
        row = {k: statistics.median(v) for k, v in times.items()}
        row["dense_checkpoints"] = hd is not None
        if ref is not None:
            row["fwd_speedup_vs_ref"] = row["ref_fwd"] / row["native_fwd"]
            row["bwd_speedup_vs_ref"] = row["ref_bwd"] / row["native_bwd"]
        rows[N] = row
        print(json.dumps({"N": N, **row}), flush=True)
        del d, a, mo, hst, hd, arms
        torch.cuda.empty_cache()
    return rows


def train_step(N, steps, warmup):
    import segmamba_b200.segmamba as sm
    defaults = sm.MambaLayer.__init__.__defaults__
    sm.MambaLayer.__init__.__defaults__ = (N,) + defaults[1:]           # every MambaLayer the model builds takes d_state N
    try:
        torch.manual_seed(0)
        model = sm.SegMamba(in_chans=4, out_chans=4, depths=[2, 2, 2, 2], feat_size=[48, 96, 192, 384]).cuda().train()
    finally:
        sm.MambaLayer.__init__.__defaults__ = defaults
    opt = torch.optim.SGD(model.parameters(), lr=1e-2, weight_decay=3e-5, momentum=0.99, nesterov=True)
    g = torch.Generator().manual_seed(42)
    x = torch.rand(2, 4, 128, 128, 128, generator=g).cuda()
    y = torch.randint(0, 4, (2, 128, 128, 128), generator=g).cuda()

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = torch.nn.functional.cross_entropy(model(x).float(), y)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(model.parameters(), 12.0)
        opt.step()
        return loss

    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    ms = [block_ms(step, 1) for _ in range(steps)]
    loss = float(step())
    row = {"d_state": N, "ms_per_step": statistics.median(ms), "peak_gb": torch.cuda.max_memory_allocated() / 1e9, "loss": loss}
    print(json.dumps(row), flush=True)
    del model, opt
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--states", default="16,32,64")
    ap.add_argument("--no-train", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print("gpu:", q, flush=True)
    states = [int(s) for s in args.states.split(",")]
    res = {"gpu": q, "scan": scan_timings(states, args.iters, args.rounds)}
    if not args.no_train:
        res["train"] = [train_step(N, args.steps, args.warmup) for N in states]
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
