"""Shared non-finite checks of the training-step kernels, for the emulator (tests/test_emu_nonfinite.py) and the GPU
(tests/test_gpu_nonfinite.py).

Two properties that value parity on finite data cannot see:
* poisoned memory: every buffer the wrappers take from torch.empty / torch.empty_like is filled with NaN (0xFF bytes for
  uint8 workspaces, a sentinel for integers); a kernel that reads a workspace or output element before writing it, or
  leaves one unwritten, changes its result;
* locality: one NaN / +Inf injected into an input makes exactly the outputs non-finite that the fp64 reference (or the
  rule of the operation, at sizes the reference cannot run) makes non-finite, and every other output keeps the bits of the
  clean run -- a masked read cancelled by a zero factor (0 * NaN = NaN) or a halo read from a neighbouring row shows up.
"""
import contextlib

import torch
import torch.nn.functional as F

from util import assert_close

NAN = float("nan")
INF = float("inf")
INT_SENTINEL = -0x5A5A5A5A
TORCH_EMPTY, TORCH_EMPTY_LIKE = torch.empty, torch.empty_like


# ------------------------------------------------------------------------------------------------------ poisoned memory
def _poison(t):
    if t.is_floating_point():
        t.fill_(NAN)
    elif t.dtype == torch.uint8:
        t.fill_(0xFF)                                      # four of them read as an fp32 NaN
    elif t.dtype != torch.bool:
        t.fill_(max(INT_SENTINEL, torch.iinfo(t.dtype).min))
    return t


@contextlib.contextmanager
def poisoned():
    """torch.empty / torch.empty_like return poisoned tensors inside the block."""
    empty, empty_like = torch.empty, torch.empty_like
    torch.empty = lambda *a, **k: _poison(empty(*a, **k))
    torch.empty_like = lambda *a, **k: _poison(empty_like(*a, **k))
    try:
        yield
    finally:
        torch.empty, torch.empty_like = empty, empty_like


def check_poison_works(device):
    with poisoned():
        f = torch.empty(3, 5, device=device)
        g = torch.empty_like(torch.zeros(2, 48, 2, 2, 2, device=device, dtype=torch.bfloat16),
                             memory_format=torch.channels_last_3d)
        w = torch.empty(64, dtype=torch.uint8, device=device)
        i = torch.empty(4, dtype=torch.int32, device=device)
    assert bool(f.isnan().all()) and bool(g.isnan().all())
    assert bool(w.view(torch.float32).isnan().all())
    assert bool((i == INT_SENTINEL).all())
    assert torch.empty is TORCH_EMPTY and torch.empty_like is TORCH_EMPTY_LIKE


def bits(t):
    return t.view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def nan_filled(t):
    """t keeps the bit pattern of torch.full(..., nan) everywhere"""
    return bool((bits(t) == bits(torch.full((1,), NAN, dtype=t.dtype, device=t.device))).all())


def compare_runs(a, b, atomic, tag):
    """dicts of outputs of two runs on the same inputs: bit-identical, or (fp32 atomics) finite and within 1e-5"""
    for k in a:
        if a[k] is None:
            continue
        if k in atomic:
            assert bool(torch.isfinite(b[k]).all()), f"{tag}{k}: non-finite"
            assert_close(b[k], a[k], 1e-5, tag + k)
        else:
            assert torch.equal(bits(a[k]), bits(b[k])), f"{tag}{k}: differs between clean and poisoned memory"


# --------------------------------------------------------------------------------------------------------------- locality
def check_locality(clean, hit, expect, atomic, tag, changed=None):
    """(a) the non-finite outputs of `hit` are exactly `expect` (name -> bool mask); (b) elsewhere `hit` has the bits of
    `clean` (fp32 atomics: within 1e-5 of the largest clean value), except where `changed` (name -> bool mask) says the
    exact result itself changes."""
    for k, m in expect.items():
        got, want = ~torch.isfinite(hit[k]).cpu(), m.cpu()
        if not torch.equal(got, want):
            extra, miss = (got & ~want).nonzero()[:4].tolist(), (want & ~got).nonzero()[:4].tolist()
            raise AssertionError(f"{tag}{k}: non-finite where finite expected at {extra}, finite where non-finite expected at {miss} "
                                 f"({int(got.sum())} vs {int(want.sum())} non-finite)")
        keep = ~want
        if changed and k in changed:
            keep &= ~changed[k].cpu()
        a, b = clean[k].cpu()[keep], hit[k].cpu()[keep]
        if k in atomic:
            scale = max(float(clean[k].abs().max()), 1e-30)
            err = float((a.double() - b.double()).abs().max()) / scale if a.numel() else 0.0
            assert err <= 1e-5, f"{tag}{k}: finite outputs moved by {err:.2e}"
        else:
            same = bits(a) == bits(b)
            assert bool(same.all()), f"{tag}{k}: {int((~same).sum())} finite outputs differ from the clean run"


def nonfinite(ref):
    return {k: ~torch.isfinite(v) for k, v in ref.items() if v is not None}


# ----------------------------------------------------------------------------------------------------------- selective scan
SCAN_ATOMIC = {"dA", "dB", "dC", "dD", "ddelta_bias"}


def _hbl(t):
    return t.permute(1, 0, 2).contiguous().permute(1, 0, 2)


def _mixer_bc(B, C):
    """(b, 1, N, L) row-slice views of one (2N, b*L) matrix, as the mixer passes them (selective_scan_interface.py)"""
    b, _, N, L = B.shape
    m = torch.cat([B[:, 0].permute(1, 0, 2).reshape(N, b * L), C[:, 0].permute(1, 0, 2).reshape(N, b * L)])
    v = lambda r: r.view(N, b, L).permute(1, 0, 2).unsqueeze(1)
    return v(m[:N]), v(m[N:])


def scan_inputs(seed, batch, dim, L, N, G, dtype, device):
    from util import rand_scan_inputs
    d = rand_scan_inputs(seed, batch, dim, L, N, G, dtype, device=device)
    for k in ("B", "C"):
        if d[k].dim() == 3:
            d[k] = d[k].unsqueeze(1)
    return d


def scan_run(d, direction, low_memory, hbl):
    """forward + one backward path, in the contiguous or the mixer's layout (u, delta, z, dout channel-major, B / C row
    slices of one matrix, dz written into the second half of a NaN-filled dxz as the mixer does)."""
    from segmamba_b200 import selective_scan_cuda as ssc
    u, delta, z, dout, B, C = d["u"], d["delta"], d["z"], d["dout"], d["B"], d["C"]
    batch, dim, L = u.shape
    if hbl:
        u, delta, z, dout = _hbl(u), _hbl(delta), _hbl(z), _hbl(dout)
        B, C = _mixer_bc(B, C)
        dxz = torch.full((2 * dim, batch, L), NAN, dtype=u.dtype, device=u.device).permute(1, 0, 2)
    else:
        dxz = torch.full((batch, 2 * dim, L), NAN, dtype=u.dtype, device=u.device)
    out, x, out_z, hst, hd = ssc.fwd_ex(u, delta, d["A"], B, C, d["D"], z, d["delta_bias"], True, direction=direction,
                                        want_out=True, want_x=True, want_hstates=True, want_hdense=True)
    g = ssc.bwd_ex(u, delta, d["A"], B, C, d["D"], z, d["delta_bias"], dout, dxz[:, dim:], True, True, direction=direction,
                   hstates=hst, hdense=hd if low_memory else None, low_memory=low_memory)
    return dict(out=out, out_z=out_z, last=x[:, :, -1, 1::2], states=x[..., 1::2], du=g[0], ddelta=g[1], dA=g[2], dB=g[3],
                dC=g[4], dD=g[5], ddelta_bias=g[6], dz=dxz[:, dim:], out_z_rec=g[8], hstates=hst), dxz[:, :dim]


def scan_reference(d, direction):
    """fp64 oracle on the same values, in walk order for the states."""
    from oracle import oracle as orc
    f = (lambda t: t.flip(-1)) if direction else (lambda t: t)
    c = {k: (f(v.float().cpu()) if k in ("u", "delta", "z", "B", "C", "dout") else v.float().cpu()) for k, v in d.items()}
    y, oz, last, xc = orc.selective_scan_fwd_raw(c["u"], c["delta"], c["A"], c["B"], c["C"], c["D"], c["z"], c["delta_bias"], True)
    g = orc.selective_scan_bwd_raw(c["u"], c["delta"], c["A"], c["B"], c["C"], c["D"], c["z"], c["delta_bias"], True, c["dout"])
    r = dict(out=f(y), out_z=f(oz), last=last, states=xc[..., 1::2], du=f(g["du"]), ddelta=f(g["ddelta"]), dA=g["dA"],
             dB=f(g["dB"]), dC=f(g["dC"]), dD=g["dD"], ddelta_bias=g["ddelta_bias"], dz=f(g["dz"]), out_z_rec=f(oz))
    return r


def inject(d, key, idx, value):
    e = dict(d)
    e[key] = d[key].clone()
    e[key][idx] = value
    return e


def scan_locality(d, sites, direction, low_memory, hbl, expect_fn=None, tag=""):
    """sites: [(input, index, value)].  expect_fn(hit_inputs, site) -> masks; default: the fp64 oracle's."""
    clean, _ = scan_run(d, direction, low_memory, hbl)
    for key, idx, val in sites:
        e = inject(d, key, idx, val)
        hit, other = scan_run(e, direction, low_memory, hbl)
        assert nan_filled(other), "scan bwd wrote outside dz"
        expect = expect_fn(e, (key, idx)) if expect_fn else nonfinite(scan_reference(e, direction))
        check_locality(clean, hit, expect, SCAN_ATOMIC, f"{tag}[{key}{idx}={val} dir={direction} low={low_memory} hbl={hbl}] ")


def scan_fwd_rule(d, site, direction):
    """u or delta at (b, c, t0): out / out_z at (b, c, t >= t0) in walk order, last state of (b, c)."""
    (key, (b, c, t0)) = site
    assert key in ("u", "delta")
    batch, dim, L = d["u"].shape
    tt = torch.arange(L)
    walk = (tt <= t0) if direction else (tt >= t0)
    m = torch.zeros(batch, dim, L, dtype=torch.bool)
    m[b, c] = walk
    last = torch.zeros(d["u"].shape[0], dim, d["A"].shape[1], dtype=torch.bool)
    last[b, c] = True
    return dict(out=m, out_z=m, last=last)


def scan_poison(d, direction, low_memory, hbl):
    clean, _ = scan_run(d, direction, low_memory, hbl)
    with poisoned():
        dirty, other = scan_run(d, direction, low_memory, hbl)
    assert nan_filled(other), "scan bwd wrote outside dz"
    for k in ("out", "out_z", "du", "ddelta", "dz", "out_z_rec"):
        assert bool(torch.isfinite(clean[k]).all()), k
    compare_runs(clean, dirty, SCAN_ATOMIC, f"[dir={direction} low={low_memory} hbl={hbl}] ")


# ------------------------------------------------------------------------------------------------------------------- conv1d
CONV_ATOMIC = {"dweight", "dbias"}


def conv_run(x, w, bias, dout, direction, hbl):
    """x as the first half of xz, dx written in place into the first half of a NaN-filled dxz (selective_scan_interface.py)."""
    from segmamba_b200 import causal_conv1d_cuda as cc
    batch, dim, L = x.shape
    if hbl:
        xz = torch.zeros(2 * dim, batch, L, dtype=x.dtype, device=x.device).permute(1, 0, 2)
        dxz = torch.full((2 * dim, batch, L), NAN, dtype=x.dtype, device=x.device).permute(1, 0, 2)
        dout = _hbl(dout)
    else:
        xz = torch.zeros(batch, 2 * dim, L, dtype=x.dtype, device=x.device)
        dxz = torch.full((batch, 2 * dim, L), NAN, dtype=x.dtype, device=x.device)
    xz[:, :dim] = x
    out = cc.causal_conv1d_fwd_ex(xz[:, :dim], w, bias, True, direction=direction)
    _, dw, db = cc.causal_conv1d_bwd_ex(xz[:, :dim], w, bias, dout, dxz[:, :dim], True, direction=direction)
    return dict(out=out, dx=dxz[:, :dim], dweight=dw, dbias=db), dxz[:, dim:]


def conv_reference(x, w, bias, dout, direction):
    from oracle import oracle as orc
    f = (lambda t: t.flip(-1)) if direction else (lambda t: t)
    o = orc.causal_conv1d_fwd_raw(f(x.float().cpu()), w.cpu(), bias.cpu(), True)
    dx, dw, db = orc.causal_conv1d_bwd_raw(f(x.float().cpu()), w.cpu(), bias.cpu(), f(dout.float().cpu()), True)
    return dict(out=f(o), dx=f(dx), dweight=dw, dbias=db)


def conv_locality(x, w, bias, dout, sites, direction, hbl, use_rule=False, tag=""):
    clean, _ = conv_run(x, w, bias, dout, direction, hbl)
    width = w.shape[1]
    for key, (b, c, t0), val in sites:
        xi, gi = x.clone(), dout.clone()
        (xi if key == "x" else gi)[b, c, t0] = val
        hit, other = conv_run(xi, w, bias, gi, direction, hbl)
        assert nan_filled(other), "conv1d bwd wrote outside dx"
        if use_rule:
            expect = conv_rule(x.shape, width, key, (b, c, t0), direction)
        else:
            expect = nonfinite(conv_reference(xi, w, bias, gi, direction))
        check_locality(clean, hit, expect, CONV_ATOMIC, f"{tag}[{key}({b},{c},{t0})={val} dir={direction} hbl={hbl}] ")


def conv_rule(shape, width, key, site, direction):
    batch, dim, L = shape
    b, c, t0 = site
    tt = torch.arange(L)
    lag = (t0 - tt) if direction else (tt - t0)            # walk-order distance from the injected position
    m = torch.zeros(batch, dim, L, dtype=torch.bool)
    zero = torch.zeros(batch, dim, L, dtype=torch.bool)
    dw, db = torch.zeros(dim, width, dtype=torch.bool), torch.zeros(dim, dtype=torch.bool)
    if key == "x":      # out (t0 .. t0 + w - 1); with SiLU those pre-activations make g-hat there, and so dx (t0 - w + 1 ..
        m[b, c] = (lag >= 0) & (lag < width)             # t0 + w - 1), dweight[c, :] and dbias[c], non-finite too
        dx = torch.zeros(batch, dim, L, dtype=torch.bool)
        dx[b, c] = (lag > -width) & (lag < width)
        dw[c], db[c] = True, True
        return dict(out=m, dx=dx, dweight=dw, dbias=db)
    m[b, c] = (lag <= 0) & (lag > -width)                   # dout: dx (t0 - w + 1 .. t0), dbias[c] and the taps of
    walk = (L - 1 - t0) if direction else t0                # dweight[c, :] that read input (not the padding before the walk)
    dw[c] = walk - (width - 1 - torch.arange(width)) >= 0
    db[c] = True
    return dict(out=zero, dx=m, dweight=dw, dbias=db)


def conv_poison(x, w, bias, dout, direction, hbl):
    clean, _ = conv_run(x, w, bias, dout, direction, hbl)
    with poisoned():
        dirty, other = conv_run(x, w, bias, dout, direction, hbl)
    assert nan_filled(other), "conv1d bwd wrote outside dx"
    assert bool(torch.isfinite(clean["dx"]).all())
    compare_runs(clean, dirty, CONV_ATOMIC, f"[dir={direction} hbl={hbl}] ")


# ----------------------------------------------------------------------------------------------------------- seq permute
def permute_poison(x, ns):
    from segmamba_b200 import causal_conv1d_cuda as cc
    clean = (cc.seq_permute(x, ns), cc.seq_permute(x, ns, inverse=True))
    with poisoned():
        dirty = (cc.seq_permute(x, ns), cc.seq_permute(x, ns, inverse=True))
    for a, b in zip(clean, dirty):
        assert torch.equal(bits(a), bits(b))


# -------------------------------------------------------------------------------------------------------- instance norm
def in_run(x, add, dy, act, mode):
    from segmamba_b200.instance_norm import fused_instance_norm
    x = x.detach().clone().contiguous(memory_format=torch.channels_last_3d).requires_grad_()
    a = add.detach().clone().requires_grad_() if add is not None else None
    y = fused_instance_norm(x, act, 0.01, add=a, add_norm=(mode == "addnorm"))
    g = torch.autograd.grad(y, [x] + ([a] if a is not None else []), dy)
    return dict(y=y.detach(), dx=g[0], dadd=g[1] if a is not None else None)


def in_reference(x, add, dy, act, mode):
    """fp64 torch: act(instance_norm(x) [+ add | + instance_norm(add)]) and its autograd."""
    xr = x.detach().double().requires_grad_()
    ar = add.detach().double().requires_grad_() if add is not None else None
    v = F.instance_norm(xr, eps=1e-5)
    if ar is not None:
        v = v + (F.instance_norm(ar, eps=1e-5) if mode == "addnorm" else ar)
    if act == "relu":
        v = torch.relu(v)
    elif act == "leaky_relu":
        v = F.leaky_relu(v, 0.01)
    g = torch.autograd.grad(v, [xr] + ([ar] if ar is not None else []), dy.double())
    return dict(y=v.detach(), dx=g[0], dadd=g[1] if ar is not None else None)


def in_inputs(shape, dtype, mode, device, seed=0):
    gen = torch.Generator(device="cpu").manual_seed(seed)
    x = (torch.randn(shape, generator=gen) * 2.0 + 0.7).to(dtype).to(device)
    add = (torch.randn(shape, generator=gen) * 0.5 - 0.3).to(dtype).to(device) if mode != "plain" else None
    dy = torch.randn(shape, generator=gen).to(dtype).to(device)
    return x, add, dy


def in_rule(shape, key, site, mode):
    """x at (b, c, v): y and dx over all of (b, c, :); add at (b, c, v) in mode 1: y at (b, c, v)."""
    b, c = site[:2]
    whole = torch.zeros(shape, dtype=torch.bool)
    whole[b, c] = True
    one = torch.zeros(shape, dtype=torch.bool)
    one[site] = True
    none = torch.zeros(shape, dtype=torch.bool)
    if key == "x":                                          # the gradient of the second operand stays finite
        r = dict(y=whole, dx=whole)
        if mode != "plain":
            r["dadd"] = none
        return r
    assert key == "add" and mode == "add"
    return dict(y=one, dx=none, dadd=none)


def in_locality(x, add, dy, act, mode, sites, use_rule=False, tag=""):
    clean = in_run(x, add, dy, act, mode)
    for key, site, val in sites:
        xs, ads, dys = x.clone(), (add.clone() if add is not None else None), dy.clone()
        {"x": xs, "add": ads, "dy": dys}[key][site] = val
        hit = in_run(xs, ads, dys, act, mode)
        if use_rule:
            expect = in_rule(tuple(x.shape), key, site, mode)
        else:
            expect = nonfinite(in_reference(xs, ads, dys, act, mode))
        changed = None
        if key in ("x", "add") and act is not None and mode != "plain":
            # a NaN pre-activation takes the NaN branch of the activation's backward (dy for ReLU, slope * dy for LeakyReLU):
            # the finite gradients of (b, c) that sum over it change value, in exact arithmetic too
            ch = torch.zeros(tuple(x.shape), dtype=torch.bool)
            ch[site[:2]] = True
            changed = {"dx": ch, "dadd": ch}
        check_locality(clean, hit, expect, set(), f"{tag}[{key}{site}={val} act={act} mode={mode}] ", changed)


def in_poison(x, add, dy, act, mode):
    clean = in_run(x, add, dy, act, mode)
    with poisoned():
        dirty = in_run(x, add, dy, act, mode)
    for k, v in clean.items():
        assert v is None or bool(torch.isfinite(v).all()), k
    compare_runs(clean, dirty, set(), f"[act={act} mode={mode}] ")


def relu_nan_semantics(device, dtype=torch.float32):
    """ReLU(IN(x)) with one NaN voxel: the reference's whole channel is NaN (torch.relu(nan) = nan) and, in mode 1, the
    gradient of the added operand passes through (threshold_backward keeps dy where the pre-activation is NaN); a NaN dy
    where the pre-activation is <= 0 is dropped, as threshold_backward selects rather than multiplies."""
    shape = (2, 16, 4, 4, 4)
    x, add, dy = in_inputs(shape, dtype, "add", device, seed=5)
    x[1, 3, 2, 1, 0] = NAN
    for mode, a in (("plain", None), ("add", add)):
        got, ref = in_run(x, a, dy, "relu", mode), in_reference(x, a, dy, "relu", mode)
        assert bool(got["y"][1, 3].isnan().all()), "ReLU maps NaN to 0"
        for k, v in ref.items():
            if v is not None:
                assert torch.equal(~torch.isfinite(got[k].cpu()), ~torch.isfinite(v.cpu())), k
        if a is not None:
            assert torch.equal(got["dadd"][1, 3], dy[1, 3]), "ReLU backward drops the gradient at NaN"
    x, add, dy = in_inputs(shape, dtype, "add", device, seed=6)
    pre = F.instance_norm(x.double(), eps=1e-5) + add.double()
    site = tuple(int(i) for i in (pre <= 0).nonzero()[0])
    dy[site] = NAN
    got, ref = in_run(x, add, dy, "relu", "add"), in_reference(x, add, dy, "relu", "add")
    for k, v in ref.items():
        assert torch.equal(~torch.isfinite(got[k].cpu()), ~torch.isfinite(v.cpu())), k
    assert bool(torch.isfinite(got["dx"]).all()) and float(got["dadd"][site]) == 0.0


# ----------------------------------------------------------------------------------------------------------- layer norm
LN_ATOMIC = {"dgamma", "dbeta"}


def ln_run(x, w, b, dy):
    from segmamba_b200.layer_norm import fused_layer_norm
    xr, wr, br = x.detach().clone().requires_grad_(), w.detach().clone().requires_grad_(), b.detach().clone().requires_grad_()
    y = fused_layer_norm(xr, wr, br, 1e-5)
    gx, gw, gb = torch.autograd.grad(y, [xr, wr, br], dy)
    return dict(y=y.detach(), dx=gx, dgamma=gw, dbeta=gb)


def ln_reference(x, w, b, dy):
    xr, wr, br = (t.detach().double().requires_grad_() for t in (x, w, b))
    y = F.layer_norm(xr, (x.shape[-1],), wr, br, 1e-5)
    gx, gw, gb = torch.autograd.grad(y, [xr, wr, br], dy.double())
    return dict(y=y.detach(), dx=gx, dgamma=gw, dbeta=gb)


def ln_inputs(rows, C, dtype, device, seed=0):
    gen = torch.Generator(device="cpu").manual_seed(seed)
    x = (torch.randn(rows, C, generator=gen) * 1.7 + 0.4).to(dtype).to(device)
    w = (torch.rand(C, generator=gen) + 0.5).to(device)
    b = (torch.randn(C, generator=gen) * 0.3).to(device)
    dy = torch.randn(rows, C, generator=gen).to(dtype).to(device)
    return x, w, b, dy


def ln_rule(rows, C, key, site):
    r, c = site
    m = torch.zeros(rows, C, dtype=torch.bool)
    m[r] = True
    none = torch.zeros(rows, C, dtype=torch.bool)
    if key == "x":                                          # y[row, :], dx[row, :], dgamma[:] (dbeta = sum dy stays finite)
        return dict(y=m, dx=m, dgamma=torch.ones(C, dtype=torch.bool), dbeta=torch.zeros(C, dtype=torch.bool))
    one = torch.zeros(C, dtype=torch.bool)
    one[c] = True
    return dict(y=none, dx=m, dgamma=one, dbeta=one)


def ln_locality(x, w, b, dy, sites, use_rule=False, tag=""):
    clean = ln_run(x, w, b, dy)
    for key, site, val in sites:
        xs, dys = x.clone(), dy.clone()
        (xs if key == "x" else dys)[site] = val
        hit = ln_run(xs, w, b, dys)
        expect = ln_rule(*x.shape, key, site) if use_rule else nonfinite(ln_reference(xs, w, b, dys))
        check_locality(clean, hit, expect, LN_ATOMIC, f"{tag}[{key}{site}={val}] ")


def ln_poison(x, w, b, dy):
    clean = ln_run(x, w, b, dy)
    with poisoned():
        dirty = ln_run(x, w, b, dy)
    compare_runs(clean, dirty, LN_ATOMIC, "")


def scan_bwd_rule(d, site, direction):
    """dout at (b, c, t0): du, ddelta at walk positions up to t0; dz at t0; dA[c, :], dD[c], ddelta_bias[c]; dB of the group at
    walk positions up to t0, dC of the group at t0; forward outputs untouched."""
    (key, (b, c, t0)) = site
    assert key == "dout"
    batch, dim, L = d["u"].shape
    G, N = d["B"].shape[1], d["A"].shape[1]
    g = c // (dim // G)
    tt = torch.arange(L)
    upto = (tt >= t0) if direction else (tt <= t0)
    seq = torch.zeros(batch, dim, L, dtype=torch.bool)
    seq[b, c] = upto
    at = torch.zeros(batch, dim, L, dtype=torch.bool)
    at[b, c, t0] = True
    dB = torch.zeros(batch, G, N, L, dtype=torch.bool)
    dB[b, g] = upto
    dC = torch.zeros(batch, G, N, L, dtype=torch.bool)
    dC[b, g, :, t0] = True
    dA = torch.zeros(dim, N, dtype=torch.bool)
    dA[c] = True
    per = torch.zeros(dim, dtype=torch.bool)
    per[c] = True
    none = torch.zeros(batch, dim, L, dtype=torch.bool)
    return dict(out=none, out_z=none, out_z_rec=none, du=seq, ddelta=seq, dz=at, dA=dA, dB=dB, dC=dC, dD=per, ddelta_bias=per)


# ------------------------------------------------------------------------------------------------------------------- GEMM
def gemm_operand(rows, cols, major, dtype, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    t = torch.randn(rows, cols, generator=g) / cols ** 0.25
    if major == "k":
        return t.to(dtype).cuda()
    return t.t().contiguous().to(dtype).cuda().t()                                # MN-major view


def gemm_run(a, b, bias, epi, out_dtype, split_k, out=None):
    from segmamba_b200 import gemm as G
    return dict(D=G.gemm(a, b, bias, epi, out_dtype=out_dtype, split_k=split_k, out=out))


def gemm_reference(a, b, bias, epi):
    from segmamba_b200 import gemm as G
    r = a.double() @ b.double().t()
    if epi in (G.EPI_BIAS_N, G.EPI_BIAS_N_GELU):
        r = r + bias.double()[None]
    elif epi == G.EPI_BIAS_M:
        r = r + bias.double()[:, None]
    if epi == G.EPI_BIAS_N_GELU:
        r = F.gelu(r)
    return dict(D=r)


def gemm_rule(M, N, key, idx, epi):
    from segmamba_b200 import gemm as G
    m = torch.zeros(M, N, dtype=torch.bool)
    if key == "a" or (key == "bias" and epi == G.EPI_BIAS_M):
        m[idx[0]] = True
    else:
        m[:, idx[0]] = True
    return dict(D=m)


def gemm_locality(a, b, bias, epi, out_dtype, split_k, sites, use_rule=False, tag=""):
    """sites: [("a" | "b" | "bias", index, value)]; index into the logical (M, K) / (N, K) operand"""
    atomic = {"D"} if split_k > 1 else set()
    clean = gemm_run(a, b, bias, epi, out_dtype, split_k)
    for key, idx, val in sites:
        ops = {"a": a.clone(), "b": b.clone(), "bias": bias.clone() if bias is not None else None}
        # clone() keeps the operand's strides (dense tensors), so MN-major views stay MN-major
        ops[key][idx] = val
        hit = gemm_run(ops["a"], ops["b"], ops["bias"], epi, out_dtype, split_k)
        expect = (gemm_rule(a.shape[0], b.shape[0], key, idx, epi) if use_rule
                  else nonfinite(gemm_reference(ops["a"], ops["b"], ops["bias"], epi)))
        check_locality(clean, hit, expect, atomic, f"{tag}[{key}{idx}={val} epi={epi} split={split_k}] ")


def gemm_poison(a, b, bias, epi, out_dtype, split_k):
    atomic = {"D"} if split_k > 1 else set()
    clean = gemm_run(a, b, bias, epi, out_dtype, split_k)
    with poisoned():
        dirty = gemm_run(a, b, bias, epi, out_dtype, split_k)
    assert bool(torch.isfinite(clean["D"]).all())
    compare_runs(clean, dirty, atomic, f"[epi={epi} split={split_k}] ")
    if split_k == 1:                         # out= without accumulate: the strided gap of the caller's buffer stays NaN
        M, N = clean["D"].shape
        big = torch.full((M, N + 24), NAN, dtype=clean["D"].dtype, device="cuda")
        got = gemm_run(a, b, bias, epi, out_dtype, 1, out=big[:, 8:N + 8])["D"]
        assert got.data_ptr() == big[:, 8:].data_ptr()
        assert torch.equal(bits(got), bits(clean["D"]))
        assert nan_filled(big[:, :8]) and nan_filled(big[:, N + 8:])


# ----------------------------------------------------------------------------------------------------------------- conv3d
CONV3D_ATOMIC = {"dW"}


def conv3d_inputs(b, ci, co, d, h, w, dtype, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn(b, d, h, w, ci, generator=g).to(dtype).cuda()
    wt = (torch.randn(co, 3, 3, 3, ci, generator=g) / (27 * ci) ** 0.5).to(dtype).cuda()
    dy = torch.randn(b, d, h, w, co, generator=g).to(dtype).cuda()
    return x, wt, dy


def conv3d_run(x5, w5, dy5):
    from segmamba_b200 import conv3d as C3
    return dict(y=C3.conv3d_fwd(x5, w5), dx=C3.conv3d_dgrad(dy5, w5), dW=C3.conv3d_wgrad(x5, dy5))


def _conv3d64(x, w):
    """fp64 3x3x3 convolution, stride 1, explicit zero padding, as a sum over the 27 taps; x (N, D, H, W, Ci), w (Co, 3, 3, 3, Ci)"""
    n, D, H, W, _ = x.shape
    xp = F.pad(x, (0, 0, 1, 1, 1, 1, 1, 1))
    y = torch.zeros(n, D, H, W, w.shape[0], dtype=torch.float64, device=x.device)
    for kd in range(3):
        for kh in range(3):
            for kw in range(3):
                y += xp[:, kd:kd + D, kh:kh + H, kw:kw + W] @ w[:, kd, kh, kw].t()
    return y


def conv3d_reference(x5, w5, dy5):
    from segmamba_b200 import conv3d as C3
    x, w, dy = x5.double(), w5.double(), dy5.double()
    n, D, H, W, ci = x.shape
    # dW[tap] = sum_v dY(v - tap + 1) x(v) over zero-padded dY: the kernel's form (_WGRAD_BORDER); in exact arithmetic it
    # equals the sum over zero-padded x
    dyp = F.pad(dy, (0, 0, 1, 1, 1, 1, 1, 1))
    dW = torch.zeros(w.shape, dtype=torch.float64, device=x.device)
    xf = x.reshape(-1, ci)
    for kd in range(3):
        for kh in range(3):
            for kw in range(3):
                dW[:, kd, kh, kw] = dyp[:, 2 - kd:2 - kd + D, 2 - kh:2 - kh + H, 2 - kw:2 - kw + W].reshape(-1, w.shape[0]).t() @ xf
    return dict(y=_conv3d64(x, w), dx=_conv3d64(dy, C3.dgrad_weight(w)), dW=dW)


# _WGRAD_BORDER: the weight gradient contracts dY, zero-filled outside the volume and shifted per tap, against unshifted x.
# In exact arithmetic that equals the reference's sum over zero-padded x, but the non-finite sets differ at the border: a
# non-finite x reaches every tap of its channel (0 * NaN where the shifted dY is padding), and a non-finite dY reaches only
# the taps whose x voxel lies in the volume.
def conv3d_rule(shape_x, co, key, site):
    """x at voxel v of sample n: y over the 3x3x3 neighbourhood of v in sample n (all C_out), dW[:, :, ci]; dy at (n, v, co):
    dx over the neighbourhood (all C_in), dW[co] for the taps whose x voxel lies in the volume (_WGRAD_BORDER)."""
    n, D, H, W, ci = shape_x
    s, z, yy, xx, c = site
    nb = torch.zeros(n, D, H, W, dtype=torch.bool)
    nb[s, max(z - 1, 0):z + 2, max(yy - 1, 0):yy + 2, max(xx - 1, 0):xx + 2] = True
    dW = torch.zeros(co, 3, 3, 3, ci, dtype=torch.bool)
    none_y, none_x = torch.zeros(n, D, H, W, co, dtype=torch.bool), torch.zeros(n, D, H, W, ci, dtype=torch.bool)
    if key == "x":
        dW[..., c] = True                # every tap: see _WGRAD_BORDER
        return dict(y=nb[..., None].expand(-1, -1, -1, -1, co).clone(), dx=none_x, dW=dW)
    for kd in range(3):
        for kh in range(3):
            for kw in range(3):          # x voxel v + (tap - 1) must lie in the volume (_WGRAD_BORDER)
                if 0 <= z + kd - 1 < D and 0 <= yy + kh - 1 < H and 0 <= xx + kw - 1 < W:
                    dW[c, kd, kh, kw] = True
    return dict(y=none_y, dx=nb[..., None].expand(-1, -1, -1, -1, ci).clone(), dW=dW)


def conv3d_locality(x5, w5, dy5, sites, use_rule=False, tag=""):
    clean = conv3d_run(x5, w5, dy5)
    for key, site, val in sites:
        xs, dys = x5.clone(), dy5.clone()
        (xs if key == "x" else dys)[site] = val
        hit = conv3d_run(xs, w5, dys)
        expect = (conv3d_rule(tuple(x5.shape), w5.shape[0], key, site) if use_rule
                  else nonfinite(conv3d_reference(xs, w5, dys)))
        check_locality(clean, hit, expect, CONV3D_ATOMIC, f"{tag}[{key}{site}={val}] ")


def conv3d_poison(x5, w5, dy5):
    clean = conv3d_run(x5, w5, dy5)
    with poisoned():
        dirty = conv3d_run(x5, w5, dy5)
    for v in clean.values():
        assert bool(torch.isfinite(v).all())
    compare_runs(clean, dirty, CONV3D_ATOMIC, "")


# --------------------------------------------------------------------------------------------------------- fp16 headroom
def headroom_scale(ref_max):
    """power of two that brings the largest reference output into [2^13, 2^14], a quarter of fp16's range at most"""
    import math
    return 2.0 ** math.floor(math.log2(2.0 ** 14 / ref_max))


def check_headroom(got, ref, lead, tol, tag):
    """every output finite, and within `tol` of the fp64 reference (max-norm relative); `lead` names the 16-bit outputs whose
    largest reference value was scaled to the headroom"""
    top = max(float(ref[k].abs().max()) for k in lead)
    assert 2.0 ** 13 <= top <= 2.0 ** 14 * 1.001, f"{tag}: reference maximum {top:.4g} is not at the headroom being tested"
    for k, v in ref.items():
        assert bool(torch.isfinite(got[k]).all()), f"{tag}{k}: non-finite at fp16 headroom"
        assert_close(got[k], v, tol, tag + k)
