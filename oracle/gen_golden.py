"""Generate golden vectors from the REFERENCE's own Python (needs the reference checkout).

TEST INFRASTRUCTURE.  Imports /root/reference (read-only) and writes small fixtures under
tests/golden/.  Nothing else may import this.

What is executed is the reference's code, unmodified:
  * selective_scan_ref          mamba/mamba_ssm/ops/selective_scan_interface.py:86-152
  * causal_conv1d_ref           causal-conv1d/causal_conv1d/causal_conv1d_interface.py:49-65
  * mamba_inner_ref             selective_scan_interface.py:636-670
  * Mamba (v3) / SegMamba       mamba/mamba_ssm/modules/mamba_simple.py, model_segmamba/segmamba.py
The two CUDA extension modules the reference imports (`selective_scan_cuda`, `causal_conv1d_cuda`)
have no CPU build, so they are replaced by stubs that call the reference's own `*_ref` functions
(forward) and autograd through them (backward).  Inputs come from numpy's legacy RandomState so the
tests can regenerate them bit-exactly without torch RNG stability assumptions.

Usage:  python oracle/gen_golden.py [--only scan,conv,inner,mamba,model,sw]
"""
from __future__ import annotations

import argparse
import importlib.util
import os
import sys
import types

import numpy as np
import torch

REF = "/root/reference"
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


# ----------------------------------------------------------------------------------------------
# loading the reference on CPU
# ----------------------------------------------------------------------------------------------
def load_reference():
    """returns (ssi module, causal_conv1d_interface module).  Installs the CUDA-module stubs."""
    if "ref_ssi" in sys.modules:
        return sys.modules["ref_ssi"], sys.modules["causal_conv1d.causal_conv1d_interface"]
    cc_stub = types.ModuleType("causal_conv1d_cuda")
    ss_stub = types.ModuleType("selective_scan_cuda")
    sys.modules["causal_conv1d_cuda"] = cc_stub
    sys.modules["selective_scan_cuda"] = ss_stub
    sys.path.insert(0, os.path.join(REF, "causal-conv1d"))
    import causal_conv1d.causal_conv1d_interface as cci   # reference module

    # stubs for mamba_ssm package pieces that pull in an incompatible `transformers`
    gen = types.ModuleType("mamba_ssm.utils.generation")
    gen.GenerationMixin = type("GenerationMixin", (), {})
    hf = types.ModuleType("mamba_ssm.utils.hf")
    hf.load_config_hf = hf.load_state_dict_hf = lambda *a, **k: None
    sys.path.insert(0, os.path.join(REF, "mamba"))
    sys.path.insert(0, REF)
    pkg = types.ModuleType("mamba_ssm")
    pkg.__path__ = [os.path.join(REF, "mamba", "mamba_ssm")]
    sys.modules["mamba_ssm"] = pkg
    sys.modules["mamba_ssm.utils.generation"] = gen
    sys.modules["mamba_ssm.utils.hf"] = hf
    import mamba_ssm.ops.selective_scan_interface as ssi   # reference module
    sys.modules["ref_ssi"] = ssi

    # ---- stub implementations: the reference's own *_ref functions -------------------------
    def cc_fwd(x, weight, bias, silu):
        return cci.causal_conv1d_ref(x, weight, bias, "silu" if silu else None)

    def cc_bwd(x, weight, bias, dout, dx_, silu):
        with torch.enable_grad():
            xr = x.detach().clone().requires_grad_()
            wr = weight.detach().clone().requires_grad_()
            br = bias.detach().clone().requires_grad_() if bias is not None else None
            out = cci.causal_conv1d_ref(xr, wr, br, "silu" if silu else None)
            grads = torch.autograd.grad(out, [xr, wr] + ([br] if br is not None else []), dout)
        dx = grads[0]
        if dx_ is not None:
            dx_.copy_(dx)
            dx = dx_
        return dx, grads[1], grads[2] if br is not None else None

    def ss_fwd(u, delta, A, B, C, D, z, delta_bias, delta_softplus):
        out = ssi.selective_scan_ref(u, delta, A, B, C, D, None, delta_bias, delta_softplus)
        n_chunks = (u.shape[-1] + 2047) // 2048
        x = torch.zeros(u.shape[0], u.shape[1], n_chunks, 2 * A.shape[1])
        if z is None:
            return out, x
        out_z = ssi.selective_scan_ref(u, delta, A, B, C, D, z, delta_bias, delta_softplus)
        return out, x, out_z

    def ss_bwd(u, delta, A, B, C, D, z, delta_bias, dout, x, out, dz_, delta_softplus, recompute_out_z):
        with torch.enable_grad():
            ins = [t.detach().clone().requires_grad_() for t in (u, delta, A, B, C)]
            Dr = D.detach().clone().requires_grad_() if D is not None else None
            zr = z.detach().clone().requires_grad_() if z is not None else None
            br = delta_bias.detach().clone().requires_grad_() if delta_bias is not None else None
            o = ssi.selective_scan_ref(ins[0], ins[1], ins[2], ins[3], ins[4], Dr, zr, br, delta_softplus)
            wanted = ins + [t for t in (Dr, zr, br) if t is not None]
            grads = list(torch.autograd.grad(o, wanted, dout))
        du, ddelta, dA, dB, dC = grads[:5]
        rest = grads[5:]
        dD = rest.pop(0) if Dr is not None else None
        dz = rest.pop(0) if zr is not None else None
        dbias = rest.pop(0) if br is not None else None
        res = [du, ddelta, dA, dB, dC, dD, dbias]
        if z is not None:
            if dz_ is not None:
                dz_.copy_(dz)
                dz = dz_
            res.append(dz)
        if recompute_out_z:
            res.append(o.detach())
        return res

    cc_stub.causal_conv1d_fwd, cc_stub.causal_conv1d_bwd = cc_fwd, cc_bwd
    ss_stub.fwd, ss_stub.bwd = ss_fwd, ss_bwd
    return ssi, cci


def load_reference_model():
    load_reference()
    import mamba_ssm.modules.mamba_simple as ms
    sys.modules["mamba_ssm"].Mamba = ms.Mamba
    spec = importlib.util.spec_from_file_location("ref_segmamba", os.path.join(REF, "model_segmamba", "segmamba.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return ms, mod


# deterministic inputs and the case tables live in tests/golden_inputs.py (shared with the tests)
sys.path.insert(0, os.path.dirname(OUT))
from golden_inputs import (CONFIG1, CONV_CASES, INNER_CASES, MAMBA_CASES, MODEL_CASE, SCAN_CASES, conv_inputs,  # noqa: E402
                           inner_inputs, model_input, randomize_state_dict, scan_inputs)

def gen_scan():
    ssi, _ = load_reference()
    for case in SCAN_CASES + [CONFIG1]:
        name, seed, batch, dim, L, N, G, tl, has_D, has_z, has_b, sp = case
        d = scan_inputs(seed, batch, dim, L, N, G, tl)
        leaves = {k: d[k].clone().requires_grad_() for k in ("u", "delta", "A", "B", "C", "D", "z", "delta_bias")}
        out, last = ssi.selective_scan_ref(
            leaves["u"], leaves["delta"], leaves["A"], leaves["B"], leaves["C"],
            leaves["D"] if has_D else None, leaves["z"] if has_z else None,
            leaves["delta_bias"] if has_b else None, sp, return_last_state=True)
        res = {"out": out.detach().numpy(), "last_state": last.detach().numpy()}
        if name != CONFIG1[0]:
            keys = ["u", "delta", "A", "B", "C"] + (["D"] if has_D else []) + (["z"] if has_z else []) + (["delta_bias"] if has_b else [])
            grads = torch.autograd.grad(out, [leaves[k] for k in keys], d["dout"])
            for k, g in zip(keys, grads):
                res["d" + k] = g.numpy()
        res["input_checksum"] = np.array([float(d["u"].double().sum()), float(d["B"].double().sum())])
        np.savez_compressed(os.path.join(OUT, f"scan_{name}.npz"), **res)
        print("scan", name, out.shape, float(out.abs().max()))


def gen_conv():
    _, cci = load_reference()
    for name, seed, batch, dim, L, width, has_b, silu in CONV_CASES:
        d = conv_inputs(seed, batch, dim, L, width)
        x = d["x"].clone().requires_grad_()
        w = d["weight"].clone().requires_grad_()
        b = d["bias"].clone().requires_grad_() if has_b else None
        out = cci.causal_conv1d_ref(x, w, b, "silu" if silu else None)
        grads = torch.autograd.grad(out, [x, w] + ([b] if has_b else []), d["dout"])
        res = {"out": out.detach().numpy(), "dx": grads[0].numpy(), "dweight": grads[1].numpy()}
        if has_b:
            res["dbias"] = grads[2].numpy()
        np.savez_compressed(os.path.join(OUT, f"conv_{name}.npz"), **res)
        print("conv", name, out.shape)


def gen_inner():
    ssi, _ = load_reference()
    for name, seed, batch, d_model, L in INNER_CASES:
        d = inner_inputs(seed, batch, d_model, L)
        keys = ["xz", "conv1d_weight", "conv1d_bias", "x_proj_weight", "delta_proj_weight", "A", "D", "delta_bias"]
        lv = {k: d[k].clone().requires_grad_() for k in keys}
        # the reference's fused path: MambaInnerFnNoOutProj (forward + its hand-written backward)
        out = ssi.mamba_inner_fn_no_out_proj(lv["xz"], lv["conv1d_weight"], lv["conv1d_bias"], lv["x_proj_weight"],
                                             lv["delta_proj_weight"], lv["A"], None, None, lv["D"],
                                             delta_bias=lv["delta_bias"], delta_softplus=True)
        grads = torch.autograd.grad(out, [lv[k] for k in keys], d["dout"])
        # cross-check with the reference's own mamba_inner_ref (identity out_proj)
        d_inner = 2 * d_model
        ref = ssi.mamba_inner_ref(d["xz"], d["conv1d_weight"], d["conv1d_bias"], d["x_proj_weight"], d["delta_proj_weight"],
                                  torch.eye(d_inner), None, d["A"], None, None, d["D"], delta_bias=d["delta_bias"],
                                  delta_softplus=True)
        assert torch.allclose(ref.transpose(1, 2), out, rtol=1e-4, atol=1e-5), "reference fused path != mamba_inner_ref"
        res = {"out": out.detach().numpy()}
        for k, g in zip(keys, grads):
            res["d" + k] = g.numpy()
        np.savez_compressed(os.path.join(OUT, f"inner_{name}.npz"), **res)
        print("inner", name, out.shape)


def gen_mamba():
    ms, _ = load_reference_model()
    for name, seed, batch, d_model, L, ns in MAMBA_CASES:
        torch.manual_seed(0)
        m = ms.Mamba(d_model=d_model, d_state=16, d_conv=4, expand=2, bimamba_type="v3", nslices=ns)
        sd = randomize_state_dict(m.state_dict(), seed)
        m.load_state_dict(sd)
        r = np.random.RandomState(seed + 1000)
        x = torch.from_numpy(r.standard_normal((batch, L, d_model)).astype(np.float32)).requires_grad_()
        dout = torch.from_numpy(r.standard_normal((batch, L, d_model)).astype(np.float32))
        out = m(x)
        names = [n for n, _ in m.named_parameters()]
        grads = torch.autograd.grad(out, [x] + [p for _, p in m.named_parameters()], dout)
        res = {"out": out.detach().numpy(), "dx": grads[0].numpy()}
        for n, g in zip(names, grads[1:]):
            res["grad." + n] = g.numpy()
        for k, v in sd.items():
            res["param." + k] = v.numpy()
        np.savez_compressed(os.path.join(OUT, f"mamba_{name}.npz"), **res)
        print("mamba", name, out.shape, float(out.abs().max()))


def gen_model():
    _, seg = load_reference_model()
    c = MODEL_CASE
    torch.manual_seed(0)
    m = seg.SegMamba(in_chans=c["in_chans"], out_chans=c["out_chans"], depths=c["depths"], feat_size=c["feat_size"],
                     hidden_size=c["hidden_size"])
    sd = randomize_state_dict(m.state_dict(), c["seed"])
    m.load_state_dict(sd)
    m.train()
    x = model_input(c["seed"] + 1, (c["batch"], c["in_chans"], c["spatial"], c["spatial"], c["spatial"]))
    out = m(x)
    r = np.random.RandomState(c["seed"] + 2)
    dout = torch.from_numpy(r.standard_normal(tuple(out.shape)).astype(np.float32)) / out.numel() ** 0.5
    names = [n for n, _ in m.named_parameters()]
    grads = torch.autograd.grad(out, [p for _, p in m.named_parameters()], dout)
    res = {"out": out.detach().numpy()}
    # keep the fixture small: grads of a representative subset + the norm of every grad
    keep = [n for n in names if ("stages.0.0.mamba" in n or "stages.3.0.mamba" in n or n.startswith("out.") or
                                 n.startswith("vit.downsample_layers.0") or n.startswith("decoder1.layer.conv1") or
                                 n.startswith("vit.gscs.1.proj4"))]
    for n, g in zip(names, grads):
        if n in keep:
            res["grad." + n] = g.numpy()
    res["grad_norms"] = np.array([float(g.double().norm()) for g in grads])
    res["param_names"] = np.array(names)
    res["state_dict_keys"] = np.array(list(sd.keys()))
    res["state_dict_shapes"] = np.array([",".join(map(str, v.shape)) for v in sd.values()])
    np.savez_compressed(os.path.join(OUT, f"model_{c['name']}.npz"), **res)
    # the full default model's state_dict surface (names + shapes only; SURVEY Appendix A)
    torch.manual_seed(0)
    full = seg.SegMamba(in_chans=4, out_chans=4, depths=[2, 2, 2, 2], feat_size=[48, 96, 192, 384])
    fsd = full.state_dict()
    np.savez_compressed(os.path.join(OUT, "state_dict_surface_default.npz"),
                        keys=np.array(list(fsd.keys())),
                        shapes=np.array([",".join(map(str, v.shape)) for v in fsd.values()]),
                        n_params=np.array([sum(v.numel() for v in fsd.values())]))
    print("model", out.shape, float(out.abs().max()), "default tensors", len(fsd))


def gen_sw():
    """MONAI sliding-window pieces: window starts, gaussian map, and a blended result with a toy predictor."""
    load_reference()
    from monai.inferers import SlidingWindowInferer
    from monai.data.utils import compute_importance_map, dense_patch_slices
    from monai.inferers.utils import _get_scan_interval
    res = {}
    for tag, image, roi in (("brats", (155, 240, 240), (128, 128, 128)), ("small", (40, 50, 33), (32, 32, 32))):
        interval = _get_scan_interval(image, roi, 3, (0.5, 0.5, 0.5))
        slices = dense_patch_slices(image, roi, interval)
        res[f"starts_{tag}"] = np.array([[s.start for s in sl] for sl in slices])
    res["gauss32"] = compute_importance_map((32, 32, 32), mode="gaussian", sigma_scale=0.125).numpy()
    res["gauss128_diag"] = compute_importance_map((128, 128, 128), mode="gaussian", sigma_scale=0.125).numpy()[
        np.arange(128), np.arange(128), np.arange(128)]
    x = model_input(50, (1, 2, 40, 50, 33))
    w = torch.from_numpy(np.random.RandomState(51).standard_normal((3, 2, 3, 3, 3)).astype(np.float32))
    pred = lambda t: torch.nn.functional.conv3d(t, w, padding=1)
    inf = SlidingWindowInferer(roi_size=(32, 32, 32), sw_batch_size=2, overlap=0.5, mode="gaussian")
    res["blend_small"] = inf(x, pred).numpy()
    np.savez_compressed(os.path.join(OUT, "sliding_window.npz"), **res)
    print("sw", res["starts_brats"].shape, res["blend_small"].shape)


def load_reference_poly_lr():
    """the reference's PolyLRScheduler class (light_training/utils/lr_scheduler.py:22-38).  It passes a third positional
    argument (`verbose`) to `_LRScheduler.__init__`, which torch >= 2.7 no longer accepts, so the base class is wrapped to
    swallow it; everything else (the initial `step()` issued by the base constructor included) is the reference's code."""
    import importlib.util
    import torch.optim.lr_scheduler as tls
    base = tls._LRScheduler

    class _Compat(base):
        def __init__(self, optimizer, last_epoch=-1, verbose=False):
            super().__init__(optimizer, last_epoch)

    tls._LRScheduler = _Compat
    try:
        spec = importlib.util.spec_from_file_location("ref_lr_scheduler", os.path.join(REF, "light_training", "utils", "lr_scheduler.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        tls._LRScheduler = base
    return mod.PolyLRScheduler


def train_toy_model():
    """stand-in network for the host-side training-loop fixtures (fixed seed, CPU, fp32)."""
    torch.manual_seed(7)
    return torch.nn.Sequential(torch.nn.Conv3d(2, 6, 3, padding=1), torch.nn.ReLU(), torch.nn.Conv3d(6, 3, 1))


def gen_train():
    """PolyLRScheduler trajectory and six iterations of the reference's inner training loop (trainer.py:444-477: grads to None,
    forward, CE loss, backward, clip_grad_norm_ 12, SGD-nesterov step, scheduler step) on a toy network, CPU fp32."""
    Poly = load_reference_poly_lr()
    res = {}
    p = [torch.nn.Parameter(torch.zeros(1))]
    opt = torch.optim.SGD(p, lr=1e-2)
    sch = Poly(opt, initial_lr=1e-2, max_steps=10)
    lrs = [opt.param_groups[0]["lr"]]
    for _ in range(9):
        opt.step()
        sch.step()
        lrs.append(opt.param_groups[0]["lr"])
    res["poly_lrs"] = np.array(lrs, dtype=np.float64)

    model = train_toy_model()
    opt = torch.optim.SGD(model.parameters(), lr=1e-2, weight_decay=3e-5, momentum=0.99, nesterov=True)   # 3_train.py:51-52
    sch = Poly(opt, initial_lr=1e-2, max_steps=20)
    ce = torch.nn.CrossEntropyLoss()
    rs = np.random.RandomState(70)
    xs = torch.from_numpy(rs.standard_normal((6, 2, 2, 8, 8, 8)).astype(np.float32))
    ys = torch.from_numpy(rs.randint(0, 3, (6, 2, 8, 8, 8)).astype(np.int64))
    losses = []
    for i in range(6):
        for prm in model.parameters():
            prm.grad = None
        loss = ce(model(xs[i]), ys[i])
        loss.backward()
        torch.nn.utils.clip_grad_norm_(model.parameters(), 12)
        opt.step()
        sch.step()
        losses.append(float(loss))
    res["train_x"], res["train_y"] = xs.numpy(), ys.numpy()
    res["train_losses"] = np.array(losses, dtype=np.float64)
    res["train_final_lr"] = np.array(opt.param_groups[0]["lr"], dtype=np.float64)
    for k, v in model.state_dict().items():
        res["train_param_" + k] = v.numpy()
    np.savez_compressed(os.path.join(OUT, "train_loop.npz"), **res)
    print("train", res["poly_lrs"], losses)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="scan,conv,inner,mamba,model,sw,train")
    args = ap.parse_args()
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(os.cpu_count() or 1)
    for part in args.only.split(","):
        {"scan": gen_scan, "conv": gen_conv, "inner": gen_inner, "mamba": gen_mamba, "model": gen_model, "sw": gen_sw, "train": gen_train}[part]()
