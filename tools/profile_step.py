"""Run ONE training step (or one op set) inside a cudaProfilerStart/Stop range, for ncu --profile-from-start off.

    ncu --profile-from-start off --metrics gpu__time_duration.sum --clock-control none --csv --log-file bench_out/launches.csv \
        python tools/profile_step.py --what step
    ncu --profile-from-start off --set full --clock-control none --import-source on -k regex:scan_ -o bench_out/scan_full \
        python tools/profile_step.py --what scan
"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--what", default="step", choices=["step", "scan", "fwd"])
    ap.add_argument("--batch", type=int, default=2)
    ap.add_argument("--dtype", default="bf16")
    args = ap.parse_args()
    dev = "cuda"
    if args.what in ("step", "fwd"):
        from segmamba_b200.segmamba import SegMamba
        torch.manual_seed(0)
        torch.backends.cudnn.benchmark = True
        m = SegMamba(in_chans=4, out_chans=4, depths=[2, 2, 2, 2], feat_size=[48, 96, 192, 384]).to(dev).train()
        opt = torch.optim.SGD(m.parameters(), lr=1e-2, momentum=0.99, nesterov=True, weight_decay=3e-5)
        x = torch.rand(args.batch, 4, 128, 128, 128, device=dev)
        y = torch.randint(0, 4, (args.batch, 128, 128, 128), device=dev)

        def step():
            opt.zero_grad(set_to_none=True)
            with torch.autocast("cuda", dtype=torch.bfloat16):
                out = m(x)
                if args.what == "fwd":
                    return
                loss = torch.nn.functional.cross_entropy(out.float(), y)
            loss.backward()
            torch.nn.utils.clip_grad_norm_(m.parameters(), 12.0)
            opt.step()
        for _ in range(3):
            step()
        torch.cuda.synchronize()
        torch.cuda.profiler.start()
        step()
        torch.cuda.synchronize()
        torch.cuda.profiler.stop()
    else:
        from segmamba_b200 import selective_scan_cuda as ssc
        dt = {"f32": torch.float32, "bf16": torch.bfloat16}[args.dtype]
        batch, D, L, N = args.batch, 96, 262144, 16
        u = torch.randn(batch, D, L, device=dev).to(dt)
        delta = (0.5 * torch.randn(batch, D, L, device=dev)).to(dt)
        z = torch.randn(batch, D, L, device=dev).to(dt)
        dout = torch.randn(batch, D, L, device=dev).to(dt)
        A = -torch.arange(1, N + 1, dtype=torch.float32, device=dev).repeat(D, 1).contiguous()
        B = torch.randn(batch, 1, N, L, device=dev).to(dt)
        C = torch.randn(batch, 1, N, L, device=dev).to(dt)
        Dp = torch.ones(D, device=dev)
        bias = torch.log(torch.expm1(0.001 + 0.1 * torch.rand(D, device=dev)))

        def run():
            _, _, _, hst, hd = ssc.fwd_ex(u, delta, A, B, C, Dp, z, bias, True, want_out=False, want_x=False, want_hstates=True, want_hdense=True)
            ssc.bwd_ex(u, delta, A, B, C, Dp, z, bias, dout, None, True, False, hstates=hst, hdense=hd)
        for _ in range(2):
            run()
        torch.cuda.synchronize()
        torch.cuda.profiler.start()
        run()
        torch.cuda.synchronize()
        torch.cuda.profiler.stop()


if __name__ == "__main__":
    main()
