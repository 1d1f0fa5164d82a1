"""Device time per kernel of one bench.py training step, grouped by who owns the kernel.

    python tools/step_kernels.py [--steps 3] [--out bench_out/step_kernels.json]

Runs the step bench.py measures (default SegMamba, seed 0, batch 2 of 4x128^3, bf16 autocast, cudnn.benchmark = False,
SGD nesterov + clip at 12) under torch.profiler with CUDA activities, in a run of its own, and sums kernel time per step in
these groups:
  conv        kernels under a convolution op, per pass (fprop / dgrad / wgrad / other) and per shape (weight shape,
              spatial size); 3^3 convolutions (all of them stride 1 in this model) are grouped apart
  cublas      GEMM kernels outside a convolution op
  aten        ATen kernels: elementwise, reduce, foreach, other
  native      kernels of libsegmamba_b200 (namespace smb), per kernel name
  other       everything else
Prints the card name and power limit read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, clk = [v.strip() for v in q.split(",")]
        return {"name": name, "power_limit": pl, "max_sm_clock": clk}
    except Exception as e:                                                # report, do not guess
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"unknown ({e})"}


CONV_OPS = ("aten::cudnn_convolution", "aten::convolution_backward", "aten::cudnn_convolution_transpose", "aten::convolution")


def conv_key(evt):
    """(op name, shape string, is_3cube_s1) of the nearest convolution op above a kernel's launching op, else None."""
    e = evt
    while e is not None:
        if e.name in ("aten::convolution", "aten::convolution_backward", "aten::_convolution") and e.input_shapes:
            sh = e.input_shapes
            if e.name == "aten::convolution_backward":
                x, w = sh[1], sh[2]
            else:
                x, w = sh[0], sh[1]
            if len(x) == 5 and len(w) == 5:
                k = tuple(w[2:])
                name = f"w{list(w)} @ {'x'.join(map(str, x[2:]))} (N={x[0]})"     # transposed convolutions: w = (C_in, C_out, k)
                return e.name, name, k == (3, 3, 3)
        e = e.cpu_parent
    return None


def classify(kname: str, evt):
    if "smb::" in kname:
        short = kname.split("(")[0].split("<")[0].replace("void ", "").strip()
        return ("native", short)
    ck = conv_key(evt)
    if ck is not None:
        op, shape, cube3 = ck
        low = kname.lower()
        if op == "aten::convolution_backward":
            ps = "wgrad" if "wgrad" in low else "dgrad" if "dgrad" in low else "bwd_other"
        else:
            ps = "fprop" if ("fprop" in low or "conv" in low or "xmma" in low or "implicit" in low) else "fwd_other"
        return ("conv3x3x3_s1" if cube3 else "conv_other", f"{ps} {shape}")
    low = kname.lower()
    if "gemm" in low or "cublas" in low or "cutlass" in low or ("xmma" in low and "conv" not in low):
        return ("cublas", kname[:90])
    if "multi_tensor_apply" in low or "foreach" in low:
        return ("aten_foreach", kname[:90])
    if "reduce_kernel" in low or "reduce" in low:
        return ("aten_reduce", kname[:90])
    if "elementwise" in low or "vectorized" in low or "at::native" in low:
        return ("aten_elementwise", kname[:90])
    return ("other", kname[:90])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "bench_out", "step_kernels.json"))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "step_kernels.py needs a CUDA device"
    from torch.profiler import ProfilerActivity, profile
    from segmamba_b200.segmamba import SegMamba
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    torch.backends.cudnn.benchmark = False                        # what bench.py runs: cuDNN's heuristic plans
    model = SegMamba(in_chans=4, out_chans=4, depths=[2, 2, 2, 2], feat_size=[48, 96, 192, 384]).to(dev).train()
    opt = torch.optim.SGD(model.parameters(), lr=1e-2, weight_decay=3e-5, momentum=0.99, nesterov=True)
    g = torch.Generator().manual_seed(42)
    x = torch.rand(2, 4, 128, 128, 128, generator=g).to(dev)
    y = torch.randint(0, 4, (2, 128, 128, 128), generator=g).to(dev)

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = torch.nn.functional.cross_entropy(model(x).float(), y)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(model.parameters(), 12.0)
        opt.step()

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(args.steps):
        step()
    e.record()
    torch.cuda.synchronize()
    step_ms = s.elapsed_time(e) / args.steps                      # unprofiled, for scale
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA], record_shapes=True) as prof:
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()

    from torch.autograd import DeviceType
    launches = []                                                 # (kernel name, launching CPU op, us)
    for evt in prof.profiler.function_events:
        if evt.device_type == DeviceType.CPU and not getattr(evt, "is_legacy", False):
            launches.extend((k.name, evt, k.duration) for k in evt.kernels)
    groups, items = {}, {}
    for name, evt, us in launches:
        grp, item = classify(name, evt)
        ms = us / 1e3 / args.steps
        groups[grp] = groups.get(grp, 0.0) + ms
        items[(grp, item)] = items.get((grp, item), 0.0) + ms
    c = card()
    total = sum(groups.values())
    res = {"card": c, "step_ms_unprofiled": step_ms, "kernel_ms_per_step": total, "groups_ms": groups,
           "items_ms": [{"group": gk, "item": ik, "ms": v} for (gk, ik), v in sorted(items.items(), key=lambda t: -t[1])]}
    big = {"128": 0.0, "64": 0.0}
    for (gk, ik), v in items.items():
        if gk == "conv3x3x3_s1":
            sp = ik.split("@ ")[1].split("x")[0]
            if sp in big:
                big[sp] += v
    res["conv3x3x3_s1_ms_at_128_and_64"] = big["128"] + big["64"]
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print(f"card: {c['name']}, power limit {c['power_limit']}, max SM clock {c.get('max_sm_clock')}")
    print(f"step {step_ms:.2f} ms unprofiled; kernel time {total:.2f} ms/step under the profiler")
    for gk, v in sorted(groups.items(), key=lambda t: -t[1]):
        print(f"  {gk:18s} {v:8.2f} ms")
    print(f"3^3 stride-1 convolutions at 128^3 and 64^3: {res['conv3x3x3_s1_ms_at_128_and_64']:.2f} ms/step")
    for r in res["items_ms"][:60]:
        print(f"  {r['ms']:8.3f}  {r['group']:16s} {r['item']}")


if __name__ == "__main__":
    main()
