"""Per-shape timing of the native tensor-core GEMM (smb_gemm) against the library product of the same views, for every
pointwise contraction of one mixer direction at the four stages (batch 2, 128^3 patch).  Measurement tool, not product.

    python tools/gemm_bench.py [--iters 10] [--stages 0,1,2,3]
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def timeit(fn, iters, flush):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(iters):
        flush.fill_(1.0)
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--stages", default="0,1,2,3")
    ap.add_argument("--out", default=os.path.join(ROOT, "bench_out", "gemm_bench.json"))
    args = ap.parse_args()
    from segmamba_b200 import gemm as G
    dev, bf = "cuda", torch.bfloat16
    flush = torch.empty(128 * 1024 * 1024, device=dev)
    rows = []
    for s in [int(v) for v in args.stages.split(",")]:
        C = 48 * 2 ** s
        d = 2 * C
        T = 2 * (64 // 2 ** s) ** 3
        R8 = {0: 8, 1: 8, 2: 16, 3: 24}[s]
        J = R8 + 32
        r = lambda *sh: torch.randn(*sh, device=dev).to(bf)
        W_in, X, Wx, U, Wdt, Xd, Wo, Y = r(2 * d, C), r(T, C), r(J, d), r(d, T), r(d, R8), r(J, T), r(C, d), r(d, T)
        dxz, dD, ddl, dXd = r(2 * d, T), r(T, C), r(d, T), r(J, T)
        acc = r(d, T)
        cases = [
            ("in_proj      xz = W X^T", W_in, X, {}),
            ("x_proj       x_dbl = Wx u", Wx, U.t(), {}),
            ("dt_proj      delta = Wdt x_dbl[:R]", Wdt, Xd[:R8].t(), {}),
            ("out_proj     y Wo^T", Y.t(), Wo, {}),
            ("in_proj dW   (split-K)", dxz, X.t(), {"split": True}),
            ("in_proj dX", dxz.t(), W_in.t(), {}),
            ("out_proj dY  (channel-major)", Wo.t(), dD, {}),
            ("out_proj dW  (split-K)", dD.t(), Y, {"split": True}),
            ("dt_proj dW   (split-K)", ddl, Xd[:R8], {"split": True}),
            ("dt_proj dx_dbl[:R]", Wdt.t(), ddl.t(), {}),
            ("x_proj dW    (split-K)", dXd, U, {"split": True}),
            ("x_proj du    (+= )", Wx.t(), dXd.t(), {"acc": True}),
        ]
        for name, a, b, kw in cases:
            M, K = a.shape
            N = b.shape[0]
            if kw.get("split"):
                sk = G._split_k_for(K)
                nat = lambda: G.gemm(a, b, out_dtype=torch.float32, split_k=sk)
                lib = lambda: (a @ b.t())
            elif kw.get("acc"):
                nat = lambda: G.gemm(a, b, out=acc, accumulate=True)
                lib = lambda: torch.addmm(acc, a, b.t())
            else:
                nat = lambda: G.gemm(a, b)
                lib = lambda: (a @ b.t())
            t_n, t_l = timeit(nat, args.iters, flush), timeit(lib, args.iters, flush)
            by = 2 * (M * K + N * K + M * N)
            row = {"stage": s, "op": name, "M": M, "N": N, "K": K, "native_ms": t_n, "library_ms": t_l, "ratio_lib_over_native": t_l / t_n,
                   "native_GBs": by / t_n / 1e6}
            rows.append(row)
            print(json.dumps(row), flush=True)
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    json.dump(rows, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
