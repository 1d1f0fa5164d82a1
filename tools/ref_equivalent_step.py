"""Training step with the REFERENCE's op sequence on the reference's own CUDA kernels -- the denominator of the
"x times the reference CUDA path" target (BASELINE.md section 3a).  Measurement tool, not product, not a bench.py value.

The reference checkout is not needed at run time, so the reference model is not imported.  What is used instead:
  * oracle/_ref/{selective_scan_cuda,causal_conv1d_cuda}.so -- the reference's kernels, compiled for sm_90a from its sources
    (oracle/build_ref.py);
  * oracle/oracle.py -- the restatement of the reference's Python (SegMamba.forward, Mamba.forward v3,
    MambaInnerFnNoOutProj.forward with its flips / stack / rearrange copies, NCDHW layout, ATen InstanceNorm3d / LayerNorm),
    pinned against the reference's own outputs by tests/test_oracle_golden.py.
This tool runs that restatement on the GPU with the two kernel entry points bound to the reference extensions.  Differences
from the real reference step: plain autograd through conv1d / x_proj / dt_proj instead of MambaInnerFnNoOutProj's
recompute-in-backward (saves the reference one conv1d + one GEMM per direction in backward, costs it memory), bf16 autocast
instead of fp16 + GradScaler.  Both arms get the same treatment of everything else (cuDNN benchmark mode, SGD, clip).

    python tools/ref_equivalent_step.py [--steps 5] [--batch 2] [--patch 128] [--native] [--dry-run-cpu]
"""
import argparse
import importlib.util
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def load_ref(name):
    path = os.path.join(ROOT, "oracle", "_ref", name + ".so")
    if not os.path.exists(path):
        raise SystemExit(f"{path} is missing: run `python oracle/build_ref.py` where the reference checkout is present first")
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def bind_reference_kernels(orc):
    """orc.selective_scan / orc.causal_conv1d <- autograd functions on the reference extensions (ssi.py:14-74,
    causal_conv1d_interface.py:10-34)."""
    ss, cc = load_ref("selective_scan_cuda"), load_ref("causal_conv1d_cuda")

    class RefScan(torch.autograd.Function):
        @staticmethod
        def forward(ctx, u, delta, A, B, C, D, z, delta_bias, delta_softplus):
            u, delta, B, C = (t if t.stride(-1) == 1 else t.contiguous() for t in (u, delta, B, C))
            z = z if z is None or z.stride(-1) == 1 else z.contiguous()
            out, x, *rest = ss.fwd(u, delta, A, B, C, D, z, delta_bias, delta_softplus)
            ctx.delta_softplus, ctx.has_z = delta_softplus, z is not None
            ctx.save_for_backward(u, delta, A, B, C, D, z, delta_bias, x, out)
            return rest[0] if z is not None else out

        @staticmethod
        def backward(ctx, dout):
            u, delta, A, B, C, D, z, delta_bias, x, out = ctx.saved_tensors
            dout = dout if dout.stride(-1) == 1 else dout.contiguous()
            du, ddelta, dA, dB, dC, dD, ddelta_bias, *rest = ss.bwd(u, delta, A, B, C, D, z, delta_bias, dout, x, out, None,
                                                                     ctx.delta_softplus, False)
            return (du, ddelta, dA, dB, dC, dD if D is not None else None, rest[0] if ctx.has_z else None,
                    ddelta_bias if delta_bias is not None else None, None)

    class RefConv(torch.autograd.Function):
        @staticmethod
        def forward(ctx, x, weight, bias, silu):
            x = x if x.stride(2) == 1 or x.stride(1) == 1 else x.contiguous()
            ctx.save_for_backward(x, weight, bias)
            ctx.silu = silu
            return cc.causal_conv1d_fwd(x, weight, bias, silu)

        @staticmethod
        def backward(ctx, dout):
            x, weight, bias = ctx.saved_tensors
            dout = dout if dout.stride(2) == 1 or dout.stride(1) == 1 else dout.contiguous()
            dx, dw, db = cc.causal_conv1d_bwd(x, weight, bias, dout, None, ctx.silu)
            return dx, dw, db if bias is not None else None, None

    orc.selective_scan = lambda u, delta, A, B, C, D=None, z=None, delta_bias=None, delta_softplus=False: RefScan.apply(
        u, delta, A, B, C, D, z, delta_bias, delta_softplus)
    orc.causal_conv1d = lambda x, weight, bias=None, activation=None: RefConv.apply(x, weight, bias, activation in ("silu", "swish"))


def make_ref_step(batch=2, patch=128, dev="cuda"):
    """(step_fn, params): one training step of the reference op sequence on the reference CUDA kernels (oracle/_ref), same
    optimizer / clip / bf16 autocast as bench.py's native arm.  Used by bench.py's ``vs_ref_cuda`` leg and by main() below."""
    from oracle import oracle as orc
    from segmamba_b200.segmamba import SegMamba
    bind_reference_kernels(orc)
    torch.backends.cudnn.benchmark = True
    depths, feat, hidden = [2, 2, 2, 2], [48, 96, 192, 384], 768
    torch.manual_seed(0)
    model = SegMamba(in_chans=4, out_chans=4, depths=depths, feat_size=feat, hidden_size=hidden)   # parameters only: same init
    params = {k: torch.nn.Parameter(v.detach().clone().to(dev).contiguous()) for k, v in model.state_dict().items()}
    del model
    opt = torch.optim.SGD(list(params.values()), lr=1e-2, weight_decay=3e-5, momentum=0.99, nesterov=True)
    nsl = tuple(patch // 2 // (2 ** i) for i in range(4))
    g = torch.Generator().manual_seed(42)
    x = torch.rand(batch, 4, patch, patch, patch, generator=g).to(dev)
    y = torch.randint(0, 4, (batch, patch, patch, patch), generator=g).to(dev)

    def ref_step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            logits = orc.segmamba_forward(params, x, depths=tuple(depths), nslices=nsl)
            loss = torch.nn.functional.cross_entropy(logits.float(), y)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(list(params.values()), 12.0)
        opt.step()
        return loss
    return ref_step, params


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=2)
    ap.add_argument("--patch", type=int, default=128)
    ap.add_argument("--native", action="store_true", help="also time the native module on the same inputs")
    ap.add_argument("--dry-run-cpu", action="store_true", help="plumbing check without a GPU: tiny model, CPU oracle kernels")
    ap.add_argument("--out", default=os.path.join(ROOT, "bench_out", "ref_equivalent_step.json"))
    args = ap.parse_args()
    from oracle import oracle as orc
    from segmamba_b200.segmamba import SegMamba
    torch.manual_seed(0)
    if args.dry_run_cpu:
        dev, depths, feat, hidden, args.patch, args.batch, args.steps, args.warmup = "cpu", [1, 1, 1, 1], [48, 32, 32, 64], 64, 32, 1, 1, 0
        orc.set_precision("f32")
    else:
        assert torch.cuda.is_available(), "needs a CUDA device (or --dry-run-cpu)"
        dev, depths, feat, hidden = "cuda", [2, 2, 2, 2], [48, 96, 192, 384], 768
        bind_reference_kernels(orc)
        torch.backends.cudnn.benchmark = True
    model = SegMamba(in_chans=4, out_chans=4, depths=depths, feat_size=feat, hidden_size=hidden)   # parameters only: same init
    params = {k: torch.nn.Parameter(v.detach().clone().to(dev)) for k, v in model.state_dict().items()}
    opt = torch.optim.SGD(list(params.values()), lr=1e-2, weight_decay=3e-5, momentum=0.99, nesterov=True)
    P = args.patch
    nsl = tuple(P // 2 // (2 ** i) for i in range(4))                   # slices = depth extent of each stage (segmamba.py:154)
    x = torch.rand(args.batch, 4, P, P, P, device=dev)
    y = torch.randint(0, 4, (args.batch, P, P, P), device=dev)

    def ref_step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast(dev, dtype=torch.bfloat16, enabled=dev == "cuda"):
            logits = orc.segmamba_forward(params, x, depths=tuple(depths), nslices=nsl)
            loss = torch.nn.functional.cross_entropy(logits.float(), y)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(list(params.values()), 12.0)
        opt.step()
        return loss

    def timed(fn):
        for _ in range(args.warmup):
            fn()
        if dev == "cuda":
            torch.cuda.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(args.steps):
                loss = fn()
            e.record()
            torch.cuda.synchronize()
            return s.elapsed_time(e) / args.steps, float(loss.detach())
        t0 = time.perf_counter()
        for _ in range(args.steps):
            loss = fn()
        return (time.perf_counter() - t0) * 1e3 / args.steps, float(loss.detach())

    res = {"batch": args.batch, "patch": P, "steps": args.steps, "device": dev}
    res["ref_equivalent_ms_per_step"], res["ref_equivalent_loss"] = timed(ref_step)
    res["ref_equivalent_patches_per_s"] = args.batch / (res["ref_equivalent_ms_per_step"] / 1e3)
    if dev == "cuda":
        res["ref_equivalent_peak_mem_gb"] = torch.cuda.max_memory_allocated() / 2 ** 30
    if args.native and dev == "cuda":
        torch.cuda.reset_peak_memory_stats()
        model = model.to(dev).train()
        nopt = torch.optim.SGD(model.parameters(), lr=1e-2, weight_decay=3e-5, momentum=0.99, nesterov=True)

        def native_step():
            nopt.zero_grad(set_to_none=True)
            with torch.autocast("cuda", dtype=torch.bfloat16):
                loss = torch.nn.functional.cross_entropy(model(x).float(), y)
            loss.backward()
            torch.nn.utils.clip_grad_norm_(model.parameters(), 12.0)
            nopt.step()
            return loss
        res["native_ms_per_step"], res["native_loss"] = timed(native_step)
        res["native_peak_mem_gb"] = torch.cuda.max_memory_allocated() / 2 ** 30
        res["speedup_vs_ref_equivalent"] = res["ref_equivalent_ms_per_step"] / res["native_ms_per_step"]
    print(json.dumps(res, indent=1))
    if not args.dry_run_cpu:
        os.makedirs(os.path.dirname(args.out), exist_ok=True)
        json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
