"""Per-op, per-shape device time of the native calls inside one training step (CUDA events around every C-ABI call)."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    from segmamba_b200 import _lib
    from segmamba_b200.segmamba import SegMamba
    dev = "cuda"
    torch.manual_seed(0)
    torch.backends.cudnn.benchmark = True
    m = SegMamba(in_chans=4, out_chans=4, depths=[2, 2, 2, 2], feat_size=[48, 96, 192, 384]).to(dev).train()
    opt = torch.optim.SGD(m.parameters(), lr=1e-2, momentum=0.99, nesterov=True, weight_decay=3e-5)
    x = torch.rand(2, 4, 128, 128, 128, device=dev)
    y = torch.randint(0, 4, (2, 128, 128, 128), device=dev)

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = torch.nn.functional.cross_entropy(m(x).float(), y)
        loss.backward()
        opt.step()
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    with _lib.profile() as prof:
        for _ in range(3):
            step()
        durs = prof.durations()
    hbm = 3350.0     # H100 SXM data sheet, GB/s
    rows = []
    for (op, meta), d in durs.items():
        ms = sum(d) / 3
        rows.append((ms, op, meta, len(d) // 3, sum(d) / len(d)))
    rows.sort(reverse=True)
    print(f"{'ms/step':>8} {'calls':>5} {'avg ms':>8}  op meta  [GB/s for instnorm: 3 passes fwd (x2 if two operands), 5 bwd]")
    for ms, op, meta, n, avg in rows:
        extra = ""
        if op.startswith("instnorm"):
            B, C, S, eb, mode2 = meta
            t = B * C * S * eb
            passes = (3 if mode2 == 0 else 5 if mode2 == 1 else 6) if op.endswith("fwd") else (5 if mode2 == 0 else 8)
            extra = f"  {passes * t / avg / 1e6:7.0f} GB/s ({100 * passes * t / avg / 1e6 / hbm:4.1f}% of {hbm})"
        print(f"{ms:8.3f} {n:5d} {avg:8.4f}  {op} {meta}{extra}")
    print("total native ms/step", sum(r[0] for r in rows))


if __name__ == "__main__":
    main()
