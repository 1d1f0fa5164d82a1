#!/usr/bin/env python
"""bench.py -- headline benchmark of the SegMamba hot path on H100.

    python bench.py --gpus N --steps K --warmup W            # native arm (one rank per GPU under torchrun for N > 1)
    python bench.py --impl reference --gpus N --steps K --warmup W   # CPU arm: the oracle port on the host cores

Metric (BASELINE.json): patches/sec, one patch = one 4x128^3 volume, forward + backward.
Workload (config.workload): BASELINE.json configs[2] -- default SegMamba (depths [2,2,2,2], dims [48,96,192,384]) training
step on synthetic 4x128^3 patches, batch 2 per GPU, bf16 autocast, CrossEntropy, SGD(nesterov) + grad-clip, DDP over NCCL
for N > 1 (weak scaling).  Prints ONE JSON line on rank 0.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import statistics
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

METRIC = "patches_per_sec_fwd_bwd_128cube_4ch"
UNIT = "patches/s"
PATCH = 128


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="native", choices=["native", "reference"])
    ap.add_argument("--batch", type=int, default=2, help="patches per GPU per step (3_train.py:23)")
    ap.add_argument("--patch", type=int, default=PATCH)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--channels-last", action="store_true", help="channels_last_3d activations for the conv stack")
    ap.add_argument("--cuda-graph", action="store_true", help="capture the whole step (fwd+bwd+clip+SGD) in one CUDA graph")
    ap.add_argument("--bf16-params", action="store_true",
                    help="bf16 matmul / convolution parameters with fp32 masters in the optimizer (segmamba_b200/master_weights.py): "
                         "same arithmetic as autocast, two multi-tensor copies per step instead of ~400 cast kernels")
    ap.add_argument("--amp", default="bf16", choices=["bf16", "fp16"],
                    help="autocast dtype of the step: bf16 (BASELINE.json) or fp16 + GradScaler, which is what the reference's trainer runs "
                         "(light_training/trainer.py:67,450,461-466)")
    ap.add_argument("--cpu-sample", type=int, default=64, help="edge of the cubic crop the CPU arm runs per step")
    ap.add_argument("--cpu-threads", type=int, default=0, help="host threads of the CPU arm (0: min(cores this process may use, 32))")
    ap.add_argument("--workload", default="train_step", choices=["train_step", "sliding_window"],
                    help="train_step: BASELINE.json configs[2] (the headline metric).  sliding_window: configs[4] -- one 240x240x155 "
                         "4-modality volume, roi 128^3, overlap 0.5, gaussian blend, x8 mirror TTA, windows sharded over the ranks")
    ap.add_argument("--no-tta", action="store_true", help="sliding_window: skip the 8 mirrored passes")
    ap.add_argument("--no-ref-cuda", action="store_true",
                    help="skip the vs_ref_cuda leg (reference op sequence on the reference's CUDA kernels from oracle/_ref)")
    ap.add_argument("--ref-cuda-steps", type=int, default=5)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps write what the last timed step computed (loss, logits, updated parameters) as DIR/<name>.npy (float32; an output of more "
                         "than 2^20 elements as a fixed seeded sample).  Inputs and weights are seeded, so two builds can be compared "
                         "output for output")
    return ap.parse_args()


# ----------------------------------------------------------------------------------------------
# clocks / throttle reasons sampled DURING the timed region
# ----------------------------------------------------------------------------------------------
class ClockSampler:
    REASONS = {0x4: "sw_power_cap", 0x8: "hw_slowdown", 0x20: "sw_thermal_slowdown", 0x40: "hw_thermal_slowdown",
               0x80: "hw_power_brake_slowdown"}

    def __init__(self, index: int):
        self.index, self.samples, self.reasons, self.max_mhz = index, [], set(), None
        self._stop = threading.Event()
        self._t = None
        try:
            import pynvml
            pynvml.nvmlInit()
            self.nv = pynvml
            self.h = pynvml.nvmlDeviceGetHandleByIndex(index)
            self.max_mhz = float(pynvml.nvmlDeviceGetMaxClockInfo(self.h, pynvml.NVML_CLOCK_SM))
        except Exception:
            self.nv = None

    def _run(self):
        while not self._stop.is_set():
            try:
                self.samples.append(float(self.nv.nvmlDeviceGetClockInfo(self.h, self.nv.NVML_CLOCK_SM)))
                mask = int(self.nv.nvmlDeviceGetCurrentClocksEventReasons(self.h))
                for bit, name in self.REASONS.items():
                    if mask & bit:
                        self.reasons.add(name)
            except Exception:
                pass
            self._stop.wait(0.1)

    def start(self):
        if self.nv is not None:
            self._t = threading.Thread(target=self._run, daemon=True)
            self._t.start()

    def stop(self):
        self._stop.set()
        if self._t is not None:
            self._t.join()
        med = statistics.median(self.samples) if self.samples else None
        return {"sm_mhz": med, "sm_max_mhz": self.max_mhz, "reasons": sorted(self.reasons), "samples": len(self.samples)}


# ----------------------------------------------------------------------------------------------
# CPU arm: the oracle port (oracle/) on the host cores.  One step = forward + backward of one cubic crop.
# ----------------------------------------------------------------------------------------------
def cpu_threads(requested: int = 0) -> int:
    """threads of the CPU arm: the cores this process may run on (not os.cpu_count(): cgroup / affinity limits), capped at 32 --
    the C oracle parallelises over channels and torch's CPU conv3d stops scaling long before 128 threads."""
    try:
        avail = len(os.sched_getaffinity(0))
    except AttributeError:
        avail = os.cpu_count() or 1
    return max(1, min(requested or 32, avail))


def cpu_step_factory(sample: int, threads: int):
    import torch
    from oracle import oracle as orc
    from segmamba_b200.segmamba import SegMamba
    orc.build()
    orc.set_precision("f32")
    torch.set_num_threads(threads)
    torch.manual_seed(0)
    model = SegMamba(in_chans=4, out_chans=4, depths=[2, 2, 2, 2], feat_size=[48, 96, 192, 384])   # weights only
    sd = {k: v.detach().clone().requires_grad_(v.dtype.is_floating_point) for k, v in model.state_dict().items()}
    x = torch.rand(1, 4, sample, sample, sample)
    y = torch.randint(0, 4, (1, sample, sample, sample))

    def step():
        for v in sd.values():
            v.grad = None
        logits = orc.segmamba_forward(sd, x)
        loss = torch.nn.functional.cross_entropy(logits, y)
        loss.backward()
        return float(loss)

    frac = (sample / PATCH) ** 3
    desc = (f"oracle port (C scan/conv1d with OpenMP + torch CPU convs), fp32, one {sample}^3 crop forward+backward per step = "
            f"{frac:.4g} of a 128^3 patch; value = {frac:.4g} / seconds; {threads} threads (torch and OpenMP each, passive wait)")
    return step, frac, threads, desc


def run_cpu(steps: int, warmup: int, sample: int, threads: int):
    """in-process CPU arm; call through run_cpu_child() so that the thread environment is the same wherever bench.py runs."""
    step, frac, cores, desc = cpu_step_factory(sample, threads)
    for _ in range(warmup):
        step()
    t0 = time.perf_counter()
    for _ in range(steps):
        step()
    dt = (time.perf_counter() - t0) / max(steps, 1)
    return {"value": frac / dt, "unit": UNIT, "cores": cores, "kind": "port", "sample": desc, "seconds_per_step": dt,
            "same_config": sample == PATCH}


def run_cpu_child(steps: int, warmup: int, sample: int, threads: int, timeout_s: float = 900.0):
    """The CPU arm in a child process with an explicit thread environment.  Round 1 ran it in-process: 128 torch threads on
    top of a second OpenMP runtime's 128 spinning threads took 47 s/step, the same code under torchrun's OMP_NUM_THREADS=1
    took 1.9 s/step.  The child gets OMP_NUM_THREADS = MKL_NUM_THREADS = n, OMP_WAIT_POLICY=passive (idle pools sleep instead
    of spinning against each other) and none of the launcher's rank variables."""
    import subprocess
    n = cpu_threads(threads)
    env = {k: v for k, v in os.environ.items()
           if k not in ("RANK", "LOCAL_RANK", "WORLD_SIZE", "MASTER_ADDR", "MASTER_PORT", "OMP_PROC_BIND", "GOMP_CPU_AFFINITY",
                        "KMP_AFFINITY", "TORCHELASTIC_RUN_ID", "GROUP_RANK", "ROLE_RANK", "LOCAL_WORLD_SIZE", "ROLE_WORLD_SIZE")}
    env.update(OMP_NUM_THREADS=str(n), MKL_NUM_THREADS=str(n), OMP_WAIT_POLICY="passive", GOMP_SPINCOUNT="0",
               SMB_CPU_CHILD="1", CUDA_VISIBLE_DEVICES="")
    cmd = [sys.executable, os.path.abspath(__file__), "--impl", "reference", "--steps", str(steps), "--warmup", str(warmup),
           "--cpu-sample", str(sample), "--cpu-threads", str(n)]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=timeout_s)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    if r.returncode != 0 or not lines:
        raise RuntimeError(f"CPU arm child failed (rc {r.returncode}): {r.stderr[-2000:]}")
    return json.loads(lines[-1])


def main_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    if os.environ.get("SMB_CPU_CHILD") != "1":
        print(json.dumps(run_cpu_child(args.steps, args.warmup, args.cpu_sample, args.cpu_threads)))
        return
    res = run_cpu(args.steps, args.warmup, args.cpu_sample, cpu_threads(args.cpu_threads))
    line = {
        "impl": "reference", "metric": METRIC, "value": res["value"], "unit": UNIT, "n_gpus": args.gpus, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": res["seconds_per_step"] * 1e3, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": workload_name(args), "global_batch": 1, "same_config": res["same_config"],
                   "note": "CPU arm: the reference has no CPU path for the model (Mamba.forward v3 is CUDA-only); this is the "
                           "oracle port of it on the host cores, one crop per step scaled by volume.  The like-for-like "
                           "baseline (reference CUDA kernels, same patch / batch / dtype) is the native arm's vs_ref_cuda key."},
        "cpu_baseline": {k: res[k] for k in ("value", "unit", "cores", "kind", "sample")},
        "e2e": {"value": res["value"], "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    print(json.dumps(line))


def workload_name(args):
    amp = "bf16 autocast" if getattr(args, "amp", "bf16") == "bf16" else "fp16 autocast + GradScaler (the reference trainer's setting)"
    return (f"SegMamba default (depths [2,2,2,2], dims [48,96,192,384]) training step on synthetic 4x{args.patch}^3 patches, "
            f"batch {args.batch}/GPU, {amp}, CE loss, SGD nesterov + clip (BASELINE.json configs[2])")


# ----------------------------------------------------------------------------------------------
# native arm
# ----------------------------------------------------------------------------------------------
def scan_fwd_bytes(meta):
    """algorithmic HBM bytes of one fused-path scan forward call: reads u, delta, z, B, C once, writes out_z once and the
    256-position states kept for backward (SURVEY.md section 8d; DESIGN.md 'Roofline')."""
    batch, dim, L, N, s, has_z, has_out = meta
    nck = (L + 255) // 256
    streams = 2 + (2 if has_z else 1) + (1 if (has_out and has_z) else 0)
    return s * batch * L * (streams * dim + 2 * N) + 4 * batch * (nck + 1) * N * dim + 4 * (dim * N + 2 * dim)


def scan_bwd_bytes(meta):
    """reads u, delta, z, dout, B, C, saved states; writes du, ddelta, dz and fp32 dB, dC."""
    batch, dim, L, N, s, has_z, has_hs = meta[:7]
    nck = (L + 255) // 256
    streams = 3 + 2 + (2 if has_z else 0)
    return s * batch * L * (streams * dim + 2 * N) + 2 * 4 * batch * N * L + 4 * batch * (nck + 1) * N * dim


DUMP_CAP = 1 << 20      # elements kept per dumped output


def dump_outputs(directory, arrays):
    """--dump-outputs: one float32 .npy per named tensor; a tensor above DUMP_CAP elements is sampled at positions drawn once from a
    fixed seed, so the same positions are kept in every run."""
    import numpy as np
    import torch
    os.makedirs(directory, exist_ok=True)
    for name, t in arrays.items():
        flat = t.detach().reshape(-1)
        if flat.numel() > DUMP_CAP:
            idx = torch.randint(0, flat.numel(), (DUMP_CAP,), generator=torch.Generator().manual_seed(1234)).sort().values
            flat = flat[idx.to(flat.device)]
        np.save(os.path.join(directory, name + ".npy"), flat.float().cpu().numpy())


_T0 = time.time()


_LAST_PROGRESS = [time.time(), "start"]


def _log(rank, msg):
    """progress on stderr (rank 0 only): stdout carries nothing but the final JSON line.  Every call also feeds the stall
    watchdog of multi-rank runs."""
    _LAST_PROGRESS[0], _LAST_PROGRESS[1] = time.time(), msg
    if rank == 0:
        print(f"[bench +{time.time() - _T0:6.1f}s] {msg}", file=sys.stderr, flush=True)


def _start_stall_watchdog(rank, limit_s=420.0):
    """multi-rank runs only: a collective that never completes would otherwise hold the box until the caller's own timeout.
    If no progress marker is reached for `limit_s`, dump every thread's stack on stderr and exit non-zero."""
    import faulthandler
    import threading

    def watch():
        while True:
            time.sleep(5.0)
            idle = time.time() - _LAST_PROGRESS[0]
            if idle > limit_s:
                print(f"[bench rank {rank}] no progress for {idle:.0f}s after '{_LAST_PROGRESS[1]}': giving up", file=sys.stderr, flush=True)
                faulthandler.dump_traceback(file=sys.stderr)
                os._exit(3)

    threading.Thread(target=watch, daemon=True, name="bench-stall-watchdog").start()


def run_ref_cuda_leg(args, native_ms_per_step, log):
    """The denominator of north_star's ">= 5x the reference CUDA path": the reference's op sequence (NCDHW, flips / stack /
    rearrange copies, ATen InstanceNorm3d / LayerNorm, cuDNN / cuBLAS as the reference calls them) on the reference's OWN CUDA
    kernels compiled for sm_90a (oracle/_ref/*.so, oracle/build_ref.py), same patch / batch / bf16 autocast / optimizer, timed
    on the same GPU right after the native arm's timed region.  Baseline only: nothing here is on the product path."""
    import gc
    import importlib.util
    import torch
    try:
        spec = importlib.util.spec_from_file_location("ref_equivalent_step", os.path.join(ROOT, "tools", "ref_equivalent_step.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        if not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "selective_scan_cuda.so")):
            return {"unavailable": "oracle/_ref/*.so not built (python oracle/build_ref.py where the reference sources are present)"}
        gc.collect()
        torch.cuda.empty_cache()
        log(0, "vs_ref_cuda leg: reference op sequence on the reference CUDA kernels")
        ref_step, params = mod.make_ref_step(args.batch, args.patch, "cuda")
        torch.backends.cudnn.benchmark = False                     # make_ref_step switches autotuning on; both arms run without it
        for _ in range(2):
            ref_step()
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(args.ref_cuda_steps):
            loss = ref_step()
        e.record()
        torch.cuda.synchronize()
        ref_ms = s.elapsed_time(e) / args.ref_cuda_steps
        out = {"ref_ms_per_step": ref_ms, "ref_patches_per_s": args.batch / (ref_ms / 1e3), "native_ms_per_step": native_ms_per_step,
               "ratio": ref_ms / native_ms_per_step, "steps": args.ref_cuda_steps, "ref_loss": float(loss.detach()),
               "kind": "reference CUDA ext (selective_scan_cuda + causal_conv1d_cuda, sm_90a build) + reference op sequence, "
                       "bf16 autocast, batch %d, %d^3 patch, same GPU" % (args.batch, args.patch)}
        del ref_step, params
        gc.collect()
        torch.cuda.empty_cache()
        return out
    except Exception as ex:
        return {"error": repr(ex)[-400:]}


def main_native(args):
    import torch
    import torch.distributed as dist
    from segmamba_b200 import _lib
    from segmamba_b200.segmamba import SegMamba

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    assert torch.cuda.is_available(), "bench.py (native arm) needs a CUDA device"
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        import datetime
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        if os.environ.get("NCCL_DEBUG", "").upper() in ("VERSION", "WARN"):
            del os.environ["NCCL_DEBUG"]               # both levels print a version banner on stdout; keep it to the JSON line
        # In-switch reduction (NVLS) is a bonus for a 270 MB gradient all-reduce, not a requirement (SURVEY.md section 5); its
        # multicast set-up needs fabric-manager support that not every container exposes, so it is opt-in here.
        os.environ.setdefault("NCCL_NVLS_ENABLE", "0")
        os.environ.setdefault("NCCL_MNNVL_ENABLE", "0")   # one box: never wait for a multi-node NVLink fabric (IMEX) that is not there
        if args.cuda_graph:
            # whole-step capture with DDP inside (PyTorch CUDA-graph notes): the process group's watchdog must not poll
            # events of a capturing stream, DDP is constructed on a side stream and runs >= 11 eager iterations before capture
            os.environ["TORCH_NCCL_ASYNC_ERROR_HANDLING"] = "0"
            os.environ["NCCL_ASYNC_ERROR_HANDLING"] = "0"
        _start_stall_watchdog(rank, 420.0 + 0.5 * (args.steps + args.warmup))   # if a collective stalls, say where and stop (stderr; stdout stays the JSON line)
        _log(rank, "init_process_group(nccl)")
        dist.init_process_group(backend="nccl", device_id=dev, timeout=datetime.timedelta(minutes=10))
        dist.barrier()
        _log(rank, "process group ready")
    _lib.lib()   # fail loudly now if the native library is missing

    torch.manual_seed(0)
    # The library convolutions run the plan cuDNN's heuristics pick, not an autotuned one: autotuning times the plans at start-up,
    # picks differently from process to process, and with the plan the rounding of every convolution changes -- two runs of the
    # same build then differ by ~1e-2 in the logits, and by the speed of whichever plans won.  The setting is process-wide, so the
    # vs_ref_cuda leg (same process, afterwards) gets the same treatment.
    torch.backends.cudnn.benchmark = False
    model = SegMamba(in_chans=4, out_chans=4, depths=[2, 2, 2, 2], feat_size=[48, 96, 192, 384]).to(dev)
    if args.channels_last:
        model = model.to(memory_format=torch.channels_last_3d)
    model.train()
    mw = None
    if args.bf16_params:
        from segmamba_b200.master_weights import MasterWeights
        mw = MasterWeights(model)                                  # before DDP: the gradient all-reduce then moves bf16
    net = model
    if world > 1:
        _log(rank, "wrapping the model in DistributedDataParallel")
        if args.cuda_graph:
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                net = torch.nn.parallel.DistributedDataParallel(model, device_ids=[local_rank], gradient_as_bucket_view=True)
            torch.cuda.current_stream().wait_stream(side)
        else:
            net = torch.nn.parallel.DistributedDataParallel(model, device_ids=[local_rank], gradient_as_bucket_view=True)
    opt_params = mw.optimizer_parameters() if mw is not None else list(model.parameters())
    opt = torch.optim.SGD(opt_params, lr=1e-2, weight_decay=3e-5, momentum=0.99, nesterov=True)             # 3_train.py:51-52
    # Every timed step is the FIRST step from the seeded initial weights: the weights and the optimizer's momentum are inputs of
    # a step as much as the patch is, and the backward accumulates with fp32 atomics, so weights carried from step to step
    # differ from run to run in the last bits -- which bf16 activations amplify to ~1e-2 of the logits within one step.
    # Restoring costs two multi-tensor kernels per step (measured inside the timed region like everything else).
    state = list({id(p): p for p in list(model.parameters()) + list(opt_params)}.values())
    state0 = [p.detach().clone() for p in state]

    @torch.no_grad()
    def restore_state():
        torch._foreach_copy_(state, state0)
        bufs = [b for st in opt.state.values() for b in st.values() if torch.is_tensor(b)]
        if bufs:
            torch._foreach_zero_(bufs)                             # a zero momentum buffer gives the first step's update
    B, P = args.batch, args.patch
    g = torch.Generator().manual_seed(42 + rank)                                                           # trainer.py:331
    x_host = torch.rand(B, 4, P, P, P, generator=g).pin_memory()
    y_host = torch.randint(0, 4, (B, P, P, P), generator=g).pin_memory()
    x_dev = x_host.to(dev)
    y_dev = y_host.to(dev)
    loss_host = torch.zeros(1).pin_memory()
    mf = torch.channels_last_3d if args.channels_last else torch.contiguous_format

    amp_dtype = torch.float16 if args.amp == "fp16" else torch.bfloat16
    scaler = torch.amp.GradScaler() if args.amp == "fp16" else None                                        # trainer.py:67

    last = {}                                                      # what the most recent step computed (--dump-outputs)

    def step(x, y):
        opt.zero_grad(set_to_none=True)
        if mw is not None:
            mw.zero_grad()
        with torch.autocast("cuda", dtype=amp_dtype):
            logits = net(x.contiguous(memory_format=mf))
            loss = torch.nn.functional.cross_entropy(logits.float(), y)
        last["logits"] = logits
        if scaler is not None:                                                                             # trainer.py:461-466
            scaler.scale(loss).backward()
            if mw is not None:
                mw.grads_to_master()
            scaler.unscale_(opt)
            torch.nn.utils.clip_grad_norm_(opt_params, 12.0)
            scaler.step(opt)
            scaler.update()
            if mw is not None:
                mw.master_to_model()
            return loss
        loss.backward()
        if mw is not None:
            mw.grads_to_master()
        torch.nn.utils.clip_grad_norm_(opt_params, 12.0)                                                   # trainer.py:464
        opt.step()
        if mw is not None:
            mw.master_to_model()
        return loss

    graphed = None
    if args.cuda_graph:
        from segmamba_b200.graph_step import GraphedTrainStep
        l0 = _lib.launch_count()
        gw = 3 if world == 1 else 11                               # DDP needs 11 eager iterations before a capture
        _log(rank, f"capturing the step in a CUDA graph ({gw} eager warm-up iterations first)")
        graphed = GraphedTrainStep(net, opt, torch.nn.functional.cross_entropy, x_dev.contiguous(memory_format=mf), y_dev,
                                   autocast_dtype=torch.bfloat16, clip_grad_norm=12.0, warmup_iters=gw, master_weights=mw)
        graph_launches = (_lib.launch_count() - l0) // (gw + 1)   # gw warm-up steps + the captured one
        eager_step = step

        def step(x, y):                                            # noqa: F811  (replay instead of eager launch)
            return graphed(x, y)

    def e2e_step():
        restore_state()
        xd = x_host.to(dev, non_blocking=True)
        yd = y_host.to(dev, non_blocking=True)
        loss = step(xd, yd)
        loss_host.copy_(loss.detach().reshape(1), non_blocking=True)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(fn, n):
        barrier()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(n):
            fn()
        e.record()
        barrier()
        ms = torch.tensor([s.elapsed_time(e)], device=dev)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms.item())

    W = max(args.warmup, 3)
    _log(rank, f"model built; {W} warm-up steps")
    layout_seen = {}

    def _layout_hook(mod, inp, out):
        layout_seen[type(mod).__name__] = bool(out.dim() == 5 and out.is_contiguous(memory_format=torch.channels_last_3d)
                                                and not out.is_contiguous())
    hooks = [model.encoder1.register_forward_hook(_layout_hook), model.vit.gscs[0].register_forward_hook(_layout_hook),
             model.decoder2.register_forward_hook(_layout_hook)] if graphed is None else []
    for _ in range(W):
        step(x_dev, y_dev)
    barrier()
    for h in hooks:
        h.remove()
    _log(rank, "warm-up done; timing")
    # host-side enqueue time of one step (no synchronisation inside): tells how close the step is to launch-bound
    t0 = time.perf_counter()
    step(x_dev, y_dev)
    host_ms = (time.perf_counter() - t0) * 1e3
    barrier()

    sampler = ClockSampler(local_rank)
    launches0 = _lib.launch_count()
    sampler.start()

    def timed_step():
        restore_state()
        last["loss"] = step(x_dev, y_dev)

    if graphed is None:
        with _lib.profile() as prof:
            total_ms = timed(timed_step, args.steps)
            durs = prof.durations()
    else:
        total_ms = timed(timed_step, args.steps)
    clocks = sampler.stop()
    launches = _lib.launch_count() - launches0
    if args.dump_outputs and rank == 0:
        # what a caller of the last timed step holds afterwards: its loss, its logits (an eager step; a replayed graph hands
        # back the loss only) and the parameters after its update, through which its gradients show
        with torch.no_grad():
            out = {"loss": last["loss"].reshape(1), "params": torch.cat([p.reshape(-1).float() for p in opt_params])}
            if "logits" in last and graphed is None:
                out["logits"] = last["logits"]
            dump_outputs(args.dump_outputs, out)
    if graphed is not None:
        launches = graph_launches * args.steps      # native kernel nodes replayed from the graph
        with _lib.profile() as prof:                # per-op timings need eager launches: taken right after the timed region
            for _ in range(2):
                eager_step(x_dev, y_dev)
            durs = prof.durations()
    ms_per_step = total_ms / args.steps
    value = world * B / (ms_per_step / 1e3)

    _log(rank, f"timed region done: {ms_per_step:.2f} ms/step")
    e2e = None
    if not args.no_e2e:
        _log(rank, "end-to-end leg")
        e2e_step()
        e2e_ms = timed(e2e_step, args.steps) / args.steps
        e2e = {"value": world * B / (e2e_ms / 1e3), "unit": UNIT,
               "h2d_bytes_per_step": int(x_host.numel() * 4 + y_host.numel() * 8), "d2h_bytes_per_step": 4,
               "ms_per_step": e2e_ms}

    # ---- roofline of the dominant native launch: the stage-0 forward scan (largest L) ----
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    hbm_peak = float(peaks.get("hbm_gbs", 3350.0))
    peak_src = "measured (MEASURED_PEAKS.json hbm_gbs)" if "hbm_gbs" in peaks else "data sheet, H100 SXM HBM3: 3350 GB/s (not a measured peak)"

    def roof(op, bytes_fn):
        metas = [m for (o, m) in durs if o == op]
        if not metas:
            return None
        meta = max(metas, key=lambda m: m[2])            # largest L = stage 0
        d = durs[(op, meta)]
        ms = sum(d) / len(d)
        by = bytes_fn(meta)
        ach = by / (ms * 1e-3) / 1e9
        return {"bound": "hbm", "achieved": ach, "peak": hbm_peak, "unit": "GB/s", "frac": ach / hbm_peak, "traffic": None,
                "traffic_source": None,
                "kernel": f"smb_{op} (all passes) at batch={meta[0]} dim={meta[1]} L={meta[2]} N={meta[3]} elt={meta[4]}B",
                "algorithmic_bytes": by, "avg_ms": ms, "launches_timed": len(d), "peak_source": peak_src}

    roof_fwd = roof("scan_fwd", scan_fwd_bytes)
    roof_bwd = roof("scan_bwd", scan_bwd_bytes)
    # The forward scan is co-bound by the MUFU pipe (DESIGN.md 3.1): one ex2 per (b, d, t, n) update in each of its two passes.
    # Extra key, not part of the contract: ex2 throughput against 132 SMs x 16 lanes/clk at the SM clock sampled under load.
    roof_mufu = None
    try:
        if roof_fwd and clocks and clocks.get("sm_mhz"):
            b_, d_, l_, n_ = [int(v) for v in re.findall(r"batch=(\d+) dim=(\d+) L=(\d+) N=(\d+)", roof_fwd["kernel"])[0]]
            ex2 = 2.0 * b_ * d_ * l_ * n_
            ach = ex2 / (roof_fwd["avg_ms"] * 1e-3) / 1e12
            peak = 132 * 16 * float(clocks["sm_mhz"]) * 1e6 / 1e12
            roof_mufu = {"bound": "mufu", "achieved": ach, "peak": peak, "unit": "Tex2/s", "frac": ach / peak,
                         "ex2_per_call": ex2, "kernel": roof_fwd["kernel"]}
    except Exception:
        roof_mufu = None
    # HBM-streaming native ops (instance norm, conv1d, permutation, layer norm, channel concatenation): achieved GB/s of each op's
    # largest call against the same measured peak -- extra evidence next to `roofline`, same CUDA-event timings
    def hbm_ops():
        models = {
            # bytes per call from the op's meta tuple (reads + writes of whole activation tensors; per-channel vectors ignored)
            "instnorm_fwd": lambda m: m[0] * m[1] * m[2] * m[3] * (3 + {0: 0, 1: 1, 2: 2}[m[4]] + (1 if m[4] == 2 else 0)),
            "instnorm_bwd": lambda m: m[0] * m[1] * m[2] * m[3] * {0: 5, 1: 6, 2: 8}[m[4]],
            "conv1d_fwd": lambda m: 2 * m[0] * m[1] * m[2] * m[3],
            "conv1d_bwd": lambda m: 3 * m[0] * m[1] * m[2] * m[3],
            "seq_permute": lambda m: 2 * m[0] * m[1] * m[2],
            "layernorm_fwd": lambda m: 2 * m[0] * m[1] * m[2],
            "layernorm_bwd": lambda m: 3 * m[0] * m[1] * m[2],
            "copy2d": lambda m: 2 * m[0] * m[1],
        }
        out = {}
        for op, fn in models.items():
            cands = [(fn(m), m) for (o, m) in durs if o == op]
            if not cands:
                continue
            by, meta = max(cands)
            d = durs[(op, meta)]
            ms = sum(d) / len(d)
            out[op] = {"meta": list(meta), "bytes": int(by), "avg_ms": ms, "GBs": by / ms / 1e6, "frac": by / ms / 1e6 / hbm_peak, "calls_timed": len(d)}
        return out

    try:
        hbm_extra = hbm_ops()
    except Exception as ex:                                   # evidence only: never lose the line over it
        hbm_extra = {"error": repr(ex)[-200:]}
    native_ms = {}
    prof_steps = args.steps if graphed is None else 2
    for (op, meta), d in durs.items():
        native_ms[op] = native_ms.get(op, 0.0) + sum(d) / prof_steps
    # `roofline` = the native op with the largest share of the step among those with a byte model (the scans); the other one
    # stays as an extra key
    cands = [(native_ms.get("scan_bwd", 0.0), roof_bwd), (native_ms.get("scan_fwd", 0.0), roof_fwd)]
    roofline = max([c for c in cands if c[1] is not None], key=lambda c: c[0], default=(0.0, None))[1]

    vs_ref_cuda = None
    if rank == 0 and world == 1 and not args.no_ref_cuda and graphed is None:
        vs_ref_cuda = run_ref_cuda_leg(args, ms_per_step, _log)
    if rank == 0:
        line = {
            "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": W,
            "ms_per_step": ms_per_step, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": args.amp,
            "data": "synthetic",
            "config": {"workload": workload_name(args), "global_batch": world * B, "parallelism": f"dp{world}",
                       "l2": "inputs larger than L2: one step touches > 10 GB of activations (50 MB L2)",
                       "channels_last_3d": (all(layout_seen.values()) if layout_seen else None), "cuda_graph": bool(args.cuda_graph), "bf16_params": bool(args.bf16_params)},
            "clocks": clocks, "e2e": e2e, "gpu_launches": int(launches),
            "roofline": roofline,
            "roofline_scan_fwd": roof_fwd,
            "roofline_scan_bwd": roof_bwd,
            "vs_ref_cuda": vs_ref_cuda,
            "roofline_mufu": roof_mufu,
            "hbm_bound_native_ops": hbm_extra,
            "native_ms_per_step": native_ms,
            "host_enqueue_ms_per_step": host_ms,
        }
        if world == 1 and not args.no_cpu_baseline:
            try:
                res = run_cpu_child(1, 1, args.cpu_sample, args.cpu_threads)
                line["cpu_baseline"] = res["cpu_baseline"]
            except Exception as ex:                        # the GPU numbers must not be lost to a CPU-leg problem
                line["cpu_baseline"] = {"error": str(ex)[-300:]}
        print(json.dumps(line))
    if world > 1:
        _log(rank, "done")
        dist.destroy_process_group()


# ----------------------------------------------------------------------------------------------
# sliding-window inference (BASELINE.json configs[4]; 4_predict.py:55-59 + prediction.py:110-159)
# ----------------------------------------------------------------------------------------------
def main_sliding_window(args):
    """One step = one whole 4x155x240x240 volume: 18 windows of 128^3 (stride 64) x 8 mirrored passes = 144 patch forwards,
    gaussian-blended on the device.  Windows are sharded `work[rank::world]` with no data-path collective; the only exchange
    is the final reduce of the weighted accumulator to rank 0.  value = volumes/s over all ranks (strong scaling: the work per
    volume is fixed), `patches_per_s` = window forwards per second.  With N > 1 rank 0 also runs the whole volume alone after
    the timed region and reports the deviation of the sharded result from it."""
    import torch
    import torch.distributed as dist
    from segmamba_b200 import _lib
    from segmamba_b200.segmamba import SegMamba
    from segmamba_b200.sliding_window import sliding_window_inference, window_starts

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    assert torch.cuda.is_available()
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        import datetime
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        if os.environ.get("NCCL_DEBUG", "").upper() in ("VERSION", "WARN"):
            del os.environ["NCCL_DEBUG"]               # both levels print a version banner on stdout; keep it to the JSON line
        os.environ.setdefault("NCCL_NVLS_ENABLE", "0")
        os.environ.setdefault("NCCL_MNNVL_ENABLE", "0")
        _start_stall_watchdog(rank, 600.0)
        dist.init_process_group(backend="nccl", device_id=dev, timeout=datetime.timedelta(minutes=10))
        dist.barrier()
    _lib.lib()
    torch.manual_seed(0)
    torch.backends.cudnn.benchmark = False                         # heuristic plans: the same arithmetic in every run (see main_native)
    model = SegMamba(in_chans=4, out_chans=4, depths=[2, 2, 2, 2], feat_size=[48, 96, 192, 384]).to(dev).eval()
    if world > 1:                                     # same weights everywhere (each rank seeded identically anyway)
        for p_ in model.parameters():
            dist.broadcast(p_.data, 0)
    g = torch.Generator().manual_seed(7)
    vol_host = torch.rand(1, 4, 155, 240, 240, generator=g).pin_memory()            # 4_predict.py: BraTS volume, 4 modalities
    roi = (args.patch,) * 3
    axes = None if args.no_tta else (0, 1, 2)
    n_win = len(window_starts((155, 240, 240), roi, 0.5)) * (1 if args.no_tta else 8)
    out_host = torch.empty(1, 4, 155, 240, 240).pin_memory() if rank == 0 else None

    def predict(x, group):
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            return sliding_window_inference(x, roi, args.batch, lambda t: model(t).float(), overlap=0.5, mode="gaussian",
                                            mirror_axes=axes, group=group, assemble_on=0)

    def step():
        x = vol_host.to(dev, non_blocking=True)                                     # H2D inside the timed region
        out = predict(x, True if world > 1 else None)
        if rank == 0:
            out_host.copy_(out, non_blocking=True)                                  # D2H of the blended logits
        return out

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    W = max(args.warmup, 1)
    _log(rank, f"sliding window: {n_win} window forwards per volume, {W} warm-up volumes")
    for _ in range(W):
        step()
    barrier()
    sampler = ClockSampler(local_rank)
    l0 = _lib.launch_count()
    sampler.start()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(args.steps):
        out = step()
    e.record()
    barrier()
    clocks = sampler.stop()
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, {"blended_logits": out})
    ms = torch.tensor([s.elapsed_time(e)], device=dev)
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    ms_per_vol = float(ms.item()) / args.steps
    launches = _lib.launch_count() - l0
    dev_vs_single = None
    if world > 1 and rank == 0:
        ref = predict(vol_host.to(dev), None)
        dev_vs_single = float((out - ref).abs().max() / ref.abs().max())
    if rank == 0:
        line = {
            "metric": "volumes_per_sec_sliding_window_240x240x155_4ch", "value": 1e3 / ms_per_vol, "unit": "volumes/s", "n_gpus": world,
            "steps": args.steps, "warmup": W, "ms_per_step": ms_per_vol, "higher_is_better": True, "scaling": "strong",
            "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
            "config": {"workload": f"SegMamba default, sliding-window inference of one 4x155x240x240 volume, roi {args.patch}^3, overlap 0.5, "
                                   f"gaussian, sw_batch_size {args.batch}, {'no TTA' if args.no_tta else 'x8 mirror TTA'} "
                                   "(BASELINE.json configs[4])",
                       "window_forwards_per_volume": n_win, "parallelism": f"windows[rank::{world}]",
                       "l2": "inputs larger than L2 (one window forward touches > 3 GB)"},
            "patches_per_s": n_win * 1e3 / ms_per_vol, "clocks": clocks, "gpu_launches": int(launches),
            "e2e": {"value": 1e3 / ms_per_vol, "unit": "volumes/s", "h2d_bytes_per_step": int(vol_host.numel() * 4),
                    "d2h_bytes_per_step": int(out_host.numel() * 4),
                    "note": "the timed region already includes the H2D copy of the volume and the D2H copy of the blended logits"},
            "sharded_vs_single_rank_max_rel": dev_vs_single,
        }
        print(json.dumps(line))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    a = parse_args()
    if a.impl == "reference":
        main_reference(a)
    elif a.workload == "sliding_window":
        main_sliding_window(a)
    else:
        main_native(a)
