"""Op-level timing on H100: native scan / conv1d vs the REFERENCE's own CUDA kernels (oracle/_ref, compiled for sm_90a).

Measurement tool (not product, not a bench.py value).  CUDA events on the launching stream, >= 3 warm-ups, L2 flushed
between iterations by writing a 512 MB buffer.  Also cross-checks the two implementations against each other (the
reference extension is a second, GPU-side oracle).  Writes bench_out/microbench.json and a markdown table.

    python tools/microbench.py [--iters 10] [--dtypes f32,bf16] [--batches 1,2]
"""
import argparse
import importlib.util
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

STAGES = [(96, 262144), (192, 32768), (384, 4096), (768, 512)]   # (d_inner, L) of the default model at 128^3 (SURVEY 8)
N = 16


def load_ref(name):
    path = os.path.join(ROOT, "oracle", "_ref", name + ".so")
    if not os.path.exists(path):
        return None
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


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


def rel(a, b):
    return float((a.float() - b.float()).abs().max() / b.float().abs().max().clamp_min(1e-30))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--dtypes", default="f32,bf16")
    ap.add_argument("--batches", default="1,2")
    ap.add_argument("--out", default=os.path.join(ROOT, "bench_out", "microbench.json"))
    ap.add_argument("--stages", default="0,1,2,3")
    ap.add_argument("--no-ref", action="store_true")
    ap.add_argument("--no-dense", action="store_true", help="A/B: 256-position checkpoints only (warp-scan main backward pass)")
    args = ap.parse_args()
    from segmamba_b200 import causal_conv1d_cuda as cc
    from segmamba_b200 import selective_scan_cuda as ssc
    ssc.DENSE_STATES = not args.no_dense
    ref_ss, ref_cc = (None, None) if args.no_ref else (load_ref("selective_scan_cuda"), load_ref("causal_conv1d_cuda"))
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    hbm = float(peaks.get("hbm_gbs", 3350.0))     # H100 SXM data sheet unless a measured peak is given
    dev = "cuda"
    flush = torch.empty(128 * 1024 * 1024, device=dev)
    rows = []
    dts = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}
    for dname in args.dtypes.split(","):
        dt = dts[dname]
        s = torch.empty(0, dtype=dt).element_size()
        for batch in [int(b) for b in args.batches.split(",")]:
            for D, L in [STAGES[int(i)] for i in args.stages.split(",")]:
                torch.manual_seed(0)
                u = torch.randn(batch, D, L, device=dev).to(dt)
                delta = (0.5 * torch.randn(batch, D, L, device=dev)).to(dt)
                z = torch.randn(batch, D, L, device=dev).to(dt)
                dout = torch.randn(batch, D, L, device=dev).to(dt)
                A = -torch.arange(1, N + 1, dtype=torch.float32, device=dev).repeat(D, 1).contiguous()
                B = torch.randn(batch, 1, N, L, device=dev).to(dt)
                C = torch.randn(batch, 1, N, L, device=dev).to(dt)
                Dp = torch.ones(D, device=dev)
                bias = torch.log(torch.expm1(0.001 + 0.1 * torch.rand(D, device=dev)))
                w = torch.randn(D, 4, device=dev) * 0.5
                cb = torch.randn(D, device=dev) * 0.1
                nck = (L + 255) // 256
                fwd_bytes = s * batch * L * (4 * D + 2 * N) + 4 * batch * (nck + 1) * N * D
                bwd_bytes = s * batch * L * (7 * D + 2 * N) + 8 * batch * N * L + 4 * batch * (nck + 1) * N * D
                conv_bytes = 2 * s * batch * D * L
                r = {"dtype": dname, "batch": batch, "dim": D, "L": L}
                _, _, _, hst, hd = ssc.fwd_ex(u, delta, A, B, C, Dp, z, bias, True, want_out=False, want_x=False, want_hstates=True,
                                              want_hdense=True)
                r["scan_fwd_ms"] = timeit(lambda: ssc.fwd_ex(u, delta, A, B, C, Dp, z, bias, True, want_out=False, want_x=False,
                                                             want_hstates=True, want_hdense=True), args.iters, flush)
                r["scan_bwd_ms"] = timeit(lambda: ssc.bwd_ex(u, delta, A, B, C, Dp, z, bias, dout, None, True, False, hstates=hst,
                                                             hdense=hd), args.iters, flush)
                r["conv_fwd_ms"] = timeit(lambda: cc.causal_conv1d_fwd(u, w, cb, True), args.iters, flush)
                r["conv_bwd_ms"] = timeit(lambda: cc.causal_conv1d_bwd(u, w, cb, dout, None, True), args.iters, flush)
                ns = {262144: 64, 32768: 32, 4096: 16, 512: 8}.get(L, 8)
                xz = torch.randn(2 * D, batch, L, device=dev).to(dt).permute(1, 0, 2)      # channel-major xz, as in the mixer
                r["permute_ms"] = timeit(lambda: cc.seq_permute(xz, ns), args.iters, flush)
                r["permute_gbs"] = 2 * s * batch * 2 * D * L / r["permute_ms"] / 1e6
                del xz
                r["scan_fwd_gbs"] = fwd_bytes / r["scan_fwd_ms"] / 1e6
                r["scan_bwd_gbs"] = bwd_bytes / r["scan_bwd_ms"] / 1e6
                r["conv_fwd_gbs"] = conv_bytes / r["conv_fwd_ms"] / 1e6
                r["scan_fwd_frac"] = r["scan_fwd_gbs"] / hbm
                r["scan_bwd_frac"] = r["scan_bwd_gbs"] / hbm
                r["conv_fwd_frac"] = r["conv_fwd_gbs"] / hbm
                if ref_ss is not None:
                    ro = ref_ss.fwd(u, delta, A, B, C, Dp, z, bias, True)
                    mo = ssc.fwd(u, delta, A, B, C, Dp, z, bias, True)
                    r["parity_out_z_vs_refcuda"] = rel(mo[2], ro[2])
                    r["ref_scan_fwd_ms"] = timeit(lambda: ref_ss.fwd(u, delta, A, B, C, Dp, z, bias, True), args.iters, flush)
                    rg = ref_ss.bwd(u, delta, A, B, C, Dp, z, bias, dout, ro[1], ro[0], None, True, False)
                    mg = ssc.bwd(u, delta, A, B, C, Dp, z, bias, dout, mo[1], mo[0], None, True, False)
                    for i, nm in enumerate(["du", "ddelta", "dA", "dB", "dC", "dD", "ddelta_bias", "dz"]):
                        r["parity_" + nm + "_vs_refcuda"] = rel(mg[i], rg[i])
                    r["ref_scan_bwd_ms"] = timeit(lambda: ref_ss.bwd(u, delta, A, B, C, Dp, z, bias, dout, ro[1], ro[0], None, True, False),
                                                  args.iters, flush)
                    r["scan_fwd_speedup"] = r["ref_scan_fwd_ms"] / r["scan_fwd_ms"]
                    r["scan_bwd_speedup"] = r["ref_scan_bwd_ms"] / r["scan_bwd_ms"]
                if ref_cc is not None:
                    r["ref_conv_fwd_ms"] = timeit(lambda: ref_cc.causal_conv1d_fwd(u, w, cb, True), args.iters, flush)
                    r["ref_conv_bwd_ms"] = timeit(lambda: ref_cc.causal_conv1d_bwd(u, w, cb, dout, None, True), args.iters, flush)
                    r["parity_conv_vs_refcuda"] = rel(cc.causal_conv1d_fwd(u, w, cb, True), ref_cc.causal_conv1d_fwd(u, w, cb, True))
                rows.append(r)
                print(json.dumps(r), flush=True)
                del u, delta, z, dout, B, C, hst, hd
                torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    json.dump({"hbm_peak_gbs": hbm, "rows": rows}, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
