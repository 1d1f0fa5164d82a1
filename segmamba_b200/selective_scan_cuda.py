"""Drop-in for the reference's pybind module ``selective_scan_cuda`` (mamba/csrc/selective_scan/selective_scan.cpp:494-497).

``fwd`` / ``bwd`` keep the reference signatures, argument meaning, output allocation rules and error behaviour
(RuntimeError on dtype / shape / stride / device violations), and forward to the C ABI ``smb_scan_fwd`` /
``smb_scan_bwd`` of libsegmamba_b200.so.  ``fwd_ex`` / ``bwd_ex`` expose what the native library adds on top:
the walk direction (flip folded into the kernel) and the saved 256-position states that let the backward
skip its forward recompute.

Register under the reference's import name with ``segmamba_b200.install_dropin()``.
"""
from __future__ import annotations

import ctypes

import torch

from . import _lib

CHUNK = 2048      # the reference's chunk-state granularity (selective_scan.cpp:307)
CKPT = 256        # native checkpoint interval (csrc/common.cuh: kCkpt)


def _check(cond, msg):
    if not cond:
        raise RuntimeError(msg)


def _validate(u, delta, A, B, C, D_, z_, delta_bias_):
    """mirrors the TORCH_CHECKs of selective_scan.cpp:233-301 for the supported (real A, variable B/C) case."""
    _lib.require_cuda(u, delta, A, B, C, D_, z_, delta_bias_)
    it = u.dtype
    _check(it in (torch.float32, torch.float16, torch.bfloat16), "selective_scan: input must be float32/float16/bfloat16")
    _check(A.dtype == torch.float32, "selective_scan: only real fp32 A is supported by segmamba_b200 (complex A is out of scope)")
    _check(B.dim() >= 3 and C.dim() >= 3, "selective_scan: only input-dependent (variable) B and C are supported by segmamba_b200")
    _check(delta.dtype == it and B.dtype == it and C.dtype == it, "selective_scan: delta, B, C must have the dtype of u")
    _check(u.dim() == 3, "selective_scan: u must be (batch, dim, seqlen)")
    batch, dim, L = u.shape
    N = A.shape[1]
    _check(tuple(delta.shape) == (batch, dim, L), "selective_scan: delta has wrong shape")
    _check(tuple(A.shape) == (dim, N), "selective_scan: A has wrong shape")
    _check(u.stride(-1) == 1 and delta.stride(-1) == 1, "selective_scan: u and delta must have stride(-1) == 1")
    if B.dim() == 3:
        B = B.unsqueeze(1)
    if C.dim() == 3:
        C = C.unsqueeze(1)
    G = B.shape[1]
    _check(tuple(B.shape) == (batch, G, N, L) and tuple(C.shape) == (batch, G, N, L), "selective_scan: B / C have wrong shape")
    _check(B.stride(-1) == 1 and C.stride(-1) == 1, "selective_scan: B and C must have stride(-1) == 1")
    _check(N <= 256, "selective_scan only supports state dimension <= 256")
    for name, t in (("D", D_), ("delta_bias", delta_bias_)):
        if t is not None:
            _check(t.dtype == torch.float32 and tuple(t.shape) == (dim,) and t.stride(-1) == 1,
                   f"selective_scan: {name} must be contiguous fp32 of shape (dim,)")
    if z_ is not None:
        _check(z_.dtype == it and tuple(z_.shape) == (batch, dim, L) and z_.stride(-1) == 1,
               "selective_scan: z must match u in dtype/shape with stride(-1) == 1")
    return batch, dim, L, N, G, B, C


def _ws(nbytes, device):
    return torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=device)


# Dense checkpoints (the state entering every 8th scan position, 8 bytes per position and channel): with them the backward's
# main pass starts every 8-position run from a saved state and a saved local adjoint instead of linking the runs with two
# 5-step warp scans per state.  DENSE_STATES=False keeps the 256-position checkpoints only (A/B; both paths are parity-tested).
DENSE_STATES = True


def fwd_ex(u, delta, A, B, C, D_=None, z_=None, delta_bias_=None, delta_softplus=False, *, direction=0,
           want_out=True, want_x=True, want_hstates=False, want_hdense=False):
    """returns (out | None, x | None, out_z | None, hstates | None) and, with want_hdense, a fifth entry: the dense
    checkpoints (or None when DENSE_STATES is off)."""
    batch, dim, L, N, G, B, C = _validate(u, delta, A, B, C, D_, z_, delta_bias_)
    A = A.contiguous()
    dev = u.device
    has_z = z_ is not None
    with torch.cuda.device(dev):
        out = torch.empty_like(delta) if (want_out or not has_z) else None        # selective_scan.cpp:311
        out_z = torch.empty_like(z_) if has_z else None                            # :303
        x = torch.empty(batch, dim, (L + CHUNK - 1) // CHUNK, 2 * N, dtype=torch.float32, device=dev) if want_x else None
        nck = (L + CKPT - 1) // CKPT
        hst = torch.empty(batch, nck + 1, N, dim, dtype=torch.float32, device=dev) if want_hstates else None
        l = _lib.lib()
        hdense = None
        if want_hdense and DENSE_STATES:
            hdense = torch.empty(l.smb_scan_dense_floats(batch, dim, L, N, G), dtype=torch.float32, device=dev)
        wsb = l.smb_scan_fwd_workspace_bytes(batch, dim, L, N)
        ws = _ws(wsb, dev)
        a = _lib.ScanFwdArgs()
        a.batch, a.dim, a.seqlen, a.dstate, a.n_groups = batch, dim, L, N, G
        a.dtype = _lib.dtype_code(u.dtype)
        a.delta_softplus = int(bool(delta_softplus))
        a.direction = int(direction)
        a.u, a.delta, a.z = _lib.ptr(u), _lib.ptr(delta), _lib.ptr(z_)
        a.A, a.D, a.delta_bias = _lib.ptr(A), _lib.ptr(D_), _lib.ptr(delta_bias_)
        a.B, a.C = _lib.ptr(B), _lib.ptr(C)
        a.out, a.out_z, a.x, a.hstates = _lib.ptr(out), _lib.ptr(out_z), _lib.ptr(x), _lib.ptr(hst)
        a.u_bs, a.u_ds = u.stride(0), u.stride(1)
        a.delta_bs, a.delta_ds = delta.stride(0), delta.stride(1)
        if has_z:
            a.z_bs, a.z_ds = z_.stride(0), z_.stride(1)
            a.out_z_bs, a.out_z_ds = out_z.stride(0), out_z.stride(1)
        if out is not None:
            a.out_bs, a.out_ds = out.stride(0), out.stride(1)
        a.B_bs, a.B_gs, a.B_ns, a.B_ls = B.stride(0), B.stride(1), B.stride(2), B.stride(3)
        a.C_bs, a.C_gs, a.C_ns, a.C_ls = C.stride(0), C.stride(1), C.stride(2), C.stride(3)
        a.workspace, a.workspace_bytes = ws.data_ptr(), wsb
        a.hdense = _lib.ptr(hdense)
        sp = _lib.stream_ptr(dev)
        _lib.call("scan_fwd", (batch, dim, L, N, u.element_size(), has_z, out is not None), lambda: l.smb_scan_fwd(ctypes.byref(a), sp), dev)
    if want_hdense:
        return out, x, out_z, hst, hdense
    return out, x, out_z, hst


def fwd(u, delta, A, B, C, D_, z_, delta_bias_, delta_softplus):
    """selective_scan_cuda.fwd -> [out, x] or [out, x, out_z]   (selective_scan.cpp:226-336)."""
    out, x, out_z, _ = fwd_ex(u, delta, A, B, C, D_, z_, delta_bias_, delta_softplus)
    return [out, x, out_z] if z_ is not None else [out, x]


LOW_MEMORY_BWD = True      # True: chunk-parallel recompute backward (small workspace; the default);
                           # False: state-stash forward-recompute + lane-per-channel reverse sweep (workspace = B*L*N*D elements)


def bwd_ex(u, delta, A, B, C, D_, z_, delta_bias_, dout, dz_=None, delta_softplus=False, recompute_out_z=False, *,
           direction=0, hstates=None, hdense=None, low_memory=None):
    """returns (du, ddelta, dA, dB(fp32), dC(fp32), dD, ddelta_bias, dz | None, out_z | None)."""
    batch, dim, L, N, G, B, C = _validate(u, delta, A, B, C, D_, z_, delta_bias_)
    _lib.require_cuda(dout)
    _check(dout.dtype == u.dtype and tuple(dout.shape) == (batch, dim, L) and dout.stride(-1) == 1,
           "selective_scan_bwd: dout must match u in dtype/shape with stride(-1) == 1")
    A = A.contiguous()
    dev = u.device
    has_z = z_ is not None
    with torch.cuda.device(dev):
        du = torch.empty_like(u)                                                   # selective_scan.cpp:458-466
        ddelta = torch.empty_like(delta)
        dA = torch.zeros_like(A)
        dB = torch.zeros(B.shape, dtype=torch.float32, device=dev)
        dC = torch.zeros(C.shape, dtype=torch.float32, device=dev)
        dD = torch.zeros_like(D_) if D_ is not None else None
        dbias = torch.zeros_like(delta_bias_) if delta_bias_ is not None else None
        dz = out_z = None
        if has_z:
            if dz_ is not None:
                _check(dz_.dtype == u.dtype and tuple(dz_.shape) == (batch, dim, L) and dz_.stride(-1) == 1,
                       "selective_scan_bwd: dz must match z")
                dz = dz_
            else:
                dz = torch.empty_like(z_)
            if recompute_out_z:
                out_z = torch.empty_like(z_)
        l = _lib.lib()
        low = int(LOW_MEMORY_BWD if low_memory is None else bool(low_memory))
        wsb = l.smb_scan_bwd_workspace_bytes(batch, dim, L, N, _lib.dtype_code(u.dtype), low)
        ws = _ws(wsb, dev)
        a = _lib.ScanBwdArgs()
        a.low_memory = low
        a.batch, a.dim, a.seqlen, a.dstate, a.n_groups = batch, dim, L, N, G
        a.dtype = _lib.dtype_code(u.dtype)
        a.delta_softplus = int(bool(delta_softplus))
        a.direction = int(direction)
        a.u, a.delta, a.z = _lib.ptr(u), _lib.ptr(delta), _lib.ptr(z_)
        a.A, a.D, a.delta_bias = _lib.ptr(A), _lib.ptr(D_), _lib.ptr(delta_bias_)
        a.B, a.C, a.dout = _lib.ptr(B), _lib.ptr(C), _lib.ptr(dout)
        a.hstates = _lib.ptr(hstates)
        mdense = None
        if hdense is not None and low:
            mdense = torch.empty_like(hdense)
            a.hdense, a.mdense = _lib.ptr(hdense), _lib.ptr(mdense)
        a.du, a.ddelta, a.dz, a.out_z = _lib.ptr(du), _lib.ptr(ddelta), _lib.ptr(dz), _lib.ptr(out_z)
        a.dA, a.dB, a.dC, a.dD, a.ddelta_bias = _lib.ptr(dA), _lib.ptr(dB), _lib.ptr(dC), _lib.ptr(dD), _lib.ptr(dbias)
        a.u_bs, a.u_ds = u.stride(0), u.stride(1)
        a.delta_bs, a.delta_ds = delta.stride(0), delta.stride(1)
        a.dout_bs, a.dout_ds = dout.stride(0), dout.stride(1)
        a.du_bs, a.du_ds = du.stride(0), du.stride(1)
        a.ddelta_bs, a.ddelta_ds = ddelta.stride(0), ddelta.stride(1)
        if has_z:
            a.z_bs, a.z_ds = z_.stride(0), z_.stride(1)
            a.dz_bs, a.dz_ds = dz.stride(0), dz.stride(1)
            if out_z is not None:
                a.out_z_bs, a.out_z_ds = out_z.stride(0), out_z.stride(1)
        a.B_bs, a.B_gs, a.B_ns, a.B_ls = B.stride(0), B.stride(1), B.stride(2), B.stride(3)
        a.C_bs, a.C_gs, a.C_ns, a.C_ls = C.stride(0), C.stride(1), C.stride(2), C.stride(3)
        a.workspace, a.workspace_bytes = ws.data_ptr(), wsb
        sp = _lib.stream_ptr(dev)
        _lib.call("scan_bwd", (batch, dim, L, N, u.element_size(), has_z, hstates is not None, low + (1 if mdense is not None else 0)), lambda: l.smb_scan_bwd(ctypes.byref(a), sp), dev)
    return du, ddelta, dA, dB, dC, dD, dbias, dz, out_z


def bwd(u, delta, A, B, C, D_, z_, delta_bias_, dout, x_, out_, dz_, delta_softplus, recompute_out_z):
    """selective_scan_cuda.bwd -> [du, ddelta, dA, dB, dC, dD, ddelta_bias, (dz), (out_z)]  (selective_scan.cpp:338-492).

    ``x_`` and ``out_`` are accepted for signature compatibility; the native backward recomputes the chunk
    states it needs (at 256-position granularity) and y, so neither is read."""
    if z_ is not None:
        _check(out_ is not None, "selective_scan_bwd: out is required when z is given")    # selective_scan.cpp:427
    n_chunks = (u.shape[-1] + CHUNK - 1) // CHUNK
    if n_chunks > 1:
        _check(x_ is not None, "selective_scan_bwd: x is required when seqlen > 2048")      # selective_scan.cpp:449
    squeeze_B, squeeze_C = B.dim() == 3, C.dim() == 3
    du, ddelta, dA, dB, dC, dD, dbias, dz, out_z = bwd_ex(u, delta, A, B, C, D_, z_, delta_bias_, dout, dz_,
                                                          delta_softplus, recompute_out_z)
    dB = dB.to(B.dtype)                                                                    # selective_scan.cpp:488
    dC = dC.to(C.dtype)
    if squeeze_B:
        dB = dB.squeeze(1)
    if squeeze_C:
        dC = dC.squeeze(1)
    res = [du, ddelta, dA, dB, dC, dD, dbias]
    if z_ is not None:
        res.append(dz)
    if recompute_out_z:
        res.append(out_z)
    return res
