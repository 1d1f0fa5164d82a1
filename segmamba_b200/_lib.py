"""ctypes binding of libsegmamba_b200.so (the C ABI declared in include/segmamba_b200.h).

The product path has NO fallback: if the shared library is missing or a call fails, a RuntimeError is
raised (the reference surfaces TORCH_CHECK / CUDA failures the same way, selective_scan.cpp:14-51).
PyTorch is used here only as the owner of device memory and of the current CUDA stream.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
import threading

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SMB_LIB") or os.path.join(_HERE, "libsegmamba_b200.so")   # SMB_LIB: tuning variants
CSRC = os.path.join(_HERE, "csrc")

SMB_F32, SMB_F16, SMB_BF16 = 0, 1, 2
DIR_FORWARD, DIR_REVERSE = 0, 1

_i32, _i64, _vp, _sz = ctypes.c_int32, ctypes.c_int64, ctypes.c_void_p, ctypes.c_size_t


class ScanFwdArgs(ctypes.Structure):
    _fields_ = (
        [(n, _i32) for n in ("batch", "dim", "seqlen", "dstate", "n_groups", "dtype", "delta_softplus", "direction")]
        + [(n, _vp) for n in ("u", "delta", "z", "A", "D", "delta_bias", "B", "C", "out", "out_z", "x", "hstates")]
        + [(n, _i64) for n in ("u_bs", "u_ds", "delta_bs", "delta_ds", "z_bs", "z_ds", "out_bs", "out_ds", "out_z_bs",
                               "out_z_ds", "B_bs", "B_gs", "B_ns", "B_ls", "C_bs", "C_gs", "C_ns", "C_ls")]
        + [("workspace", _vp), ("workspace_bytes", _sz), ("hdense", _vp)]
    )


class ScanBwdArgs(ctypes.Structure):
    _fields_ = (
        [(n, _i32) for n in ("batch", "dim", "seqlen", "dstate", "n_groups", "dtype", "delta_softplus", "direction",
                             "low_memory")]
        + [(n, _vp) for n in ("u", "delta", "z", "A", "D", "delta_bias", "B", "C", "dout", "hstates", "du", "ddelta",
                              "dz", "out_z", "dA", "dB", "dC", "dD", "ddelta_bias")]
        + [(n, _i64) for n in ("u_bs", "u_ds", "delta_bs", "delta_ds", "z_bs", "z_ds", "dout_bs", "dout_ds",
                               "du_bs", "du_ds", "ddelta_bs", "ddelta_ds", "dz_bs", "dz_ds", "out_z_bs", "out_z_ds",
                               "B_bs", "B_gs", "B_ns", "B_ls", "C_bs", "C_gs", "C_ns", "C_ls")]
        + [("workspace", _vp), ("workspace_bytes", _sz), ("hdense", _vp), ("mdense", _vp)]
    )


class Conv1dArgs(ctypes.Structure):
    _fields_ = (
        [(n, _i32) for n in ("batch", "dim", "seqlen", "width", "dtype", "silu", "direction")]
        + [(n, _vp) for n in ("x", "weight", "bias", "out")]
        + [(n, _i64) for n in ("x_bs", "x_ds", "out_bs", "out_ds", "w_ds", "w_ws")]
    )


class Conv1dBwdArgs(ctypes.Structure):
    _fields_ = (
        [(n, _i32) for n in ("batch", "dim", "seqlen", "width", "dtype", "silu", "direction")]
        + [(n, _vp) for n in ("x", "dout", "weight", "bias", "dx", "dweight", "dbias")]
        + [(n, _i64) for n in ("x_bs", "x_ds", "dout_bs", "dout_ds", "dx_bs", "dx_ds", "w_ds", "w_ws")]
    )


class SeqPermuteArgs(ctypes.Structure):
    _fields_ = (
        [(n, _i32) for n in ("rows", "seqlen", "nslices", "dtype", "inverse", "accumulate")]
        + [("src", _vp), ("dst", _vp), ("src_rs", _i64), ("dst_rs", _i64)]
    )


class InstNormArgs(ctypes.Structure):
    _fields_ = (
        [(n, _i32) for n in ("batch", "channels", "dtype", "act", "mode2")]
        + [("slope", ctypes.c_float), ("eps", ctypes.c_float), ("spatial", _i64)]
        + [(n, _vp) for n in ("x", "x2", "y", "stats", "stats2", "workspace")]
        + [("workspace_bytes", _sz)]
    )


class InstNormBwdArgs(ctypes.Structure):
    _fields_ = (
        [(n, _i32) for n in ("batch", "channels", "dtype", "act", "mode2")]
        + [("slope", ctypes.c_float), ("eps", ctypes.c_float), ("spatial", _i64)]
        + [(n, _vp) for n in ("x", "x2", "dy", "stats", "stats2", "dx", "dx2", "workspace")]
        + [("workspace_bytes", _sz)]
    )


class LayerNormArgs(ctypes.Structure):
    _fields_ = ([("rows", _i64), ("channels", _i32), ("dtype", _i32), ("eps", ctypes.c_float)]
                + [(n, _vp) for n in ("x", "gamma", "beta", "y")])


class LayerNormBwdArgs(ctypes.Structure):
    _fields_ = ([("rows", _i64), ("channels", _i32), ("dtype", _i32), ("eps", ctypes.c_float)]
                + [(n, _vp) for n in ("x", "dy", "gamma", "dx", "dgamma", "dbeta")])


class GemmArgs(ctypes.Structure):
    _fields_ = ([(n, _i32) for n in ("M", "N", "K", "dtype", "out_dtype", "a_major", "b_major", "epilogue", "split_k", "accumulate")]
                + [(n, _vp) for n in ("A", "B", "bias", "D")] + [(n, _i64) for n in ("lda", "ldb", "ldd")])


# every symbol include/segmamba_b200.h declares (tests/test_abi.py checks the header against this list)
EXPORTS = {
    "smb_version": (ctypes.c_int, []),
    "smb_last_error": (ctypes.c_char_p, []),
    "smb_launch_count": (ctypes.c_uint64, []),
    "smb_scan_fwd_workspace_bytes": (_sz, [_i32, _i32, _i32, _i32]),
    "smb_scan_dense_floats": (_sz, [_i32, _i32, _i32, _i32, _i32]),
    "smb_scan_fwd": (ctypes.c_int, [ctypes.POINTER(ScanFwdArgs), _vp]),
    "smb_scan_bwd_workspace_bytes": (_sz, [_i32, _i32, _i32, _i32, _i32, _i32]),
    "smb_scan_bwd": (ctypes.c_int, [ctypes.POINTER(ScanBwdArgs), _vp]),
    "smb_conv1d_fwd": (ctypes.c_int, [ctypes.POINTER(Conv1dArgs), _vp]),
    "smb_conv1d_bwd": (ctypes.c_int, [ctypes.POINTER(Conv1dBwdArgs), _vp]),
    "smb_seq_permute": (ctypes.c_int, [ctypes.POINTER(SeqPermuteArgs), _vp]),
    "smb_instnorm_workspace_bytes": (_sz, [_i32, _i32, _i64, _i32]),
    "smb_instnorm_fwd": (ctypes.c_int, [ctypes.POINTER(InstNormArgs), _vp]),
    "smb_instnorm_bwd": (ctypes.c_int, [ctypes.POINTER(InstNormBwdArgs), _vp]),
    "smb_layernorm_fwd": (ctypes.c_int, [ctypes.POINTER(LayerNormArgs), _vp]),
    "smb_layernorm_bwd": (ctypes.c_int, [ctypes.POINTER(LayerNormBwdArgs), _vp]),
    "smb_gemm": (ctypes.c_int, [ctypes.POINTER(GemmArgs), _vp]),
    "smb_copy2d": (ctypes.c_int, [_vp, _i64, _vp, _i64, _i64, _i64, _vp]),
}

_lib = None
_lock = threading.Lock()


def build(verbose: bool = False) -> str:
    """Compile the CUDA sources for sm_90a with nvcc (cross-compiles without a GPU). Returns the .so path."""
    cmd = ["make", "-C", CSRC, "-j8", "all"]
    if not verbose:
        cmd.insert(1, "-s")
    subprocess.run(cmd, check=True)
    return LIB_PATH


def lib() -> ctypes.CDLL:
    """Load the shared library; raise loudly if it has not been built (no CPU / eager fallback exists)."""
    global _lib
    if _lib is None:
        with _lock:
            if _lib is None:
                if not os.path.exists(LIB_PATH):
                    raise RuntimeError(
                        f"segmamba_b200: {LIB_PATH} is missing. Build it with `python -c 'import __graft_entry__ as g; "
                        "g.build()'` (or `make -C segmamba_b200/csrc`). There is no fallback path.")
                l = ctypes.CDLL(LIB_PATH)
                for name, (res, args) in EXPORTS.items():
                    fn = getattr(l, name)
                    fn.restype = res
                    fn.argtypes = args
                _lib = l
    return _lib


# ---- optional per-op device timing (bench.py's roofline leg).  Events are recorded on torch's current stream, which is
# the stream the library's kernels are enqueued on (stream_ptr below). ----
_PROF = None


class profile:
    """with _lib.profile() as prof: ...  ->  prof.durations() = {(op, meta): [ms, ...]} after a synchronize."""

    def __enter__(self):
        global _PROF
        self.records = []
        _PROF = self.records
        return self

    def __exit__(self, *exc):
        global _PROF
        _PROF = None
        return False

    def durations(self):
        torch.cuda.synchronize()
        out = {}
        for op, meta, s, e in self.records:
            out.setdefault((op, meta), []).append(s.elapsed_time(e))
        return out


def call(op: str, meta: tuple, fn, device) -> None:
    """run one C-ABI call (returns its int code through check()); time it with CUDA events when profiling is on."""
    if _PROF is None:
        check(fn())
        return
    stream = torch.cuda.current_stream(device)
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record(stream)
    rc = fn()
    e.record(stream)
    _PROF.append((op, meta, s, e))
    check(rc)


def launch_count() -> int:
    return int(lib().smb_launch_count())


def check(rc: int) -> None:
    if rc != 0:
        msg = lib().smb_last_error()
        raise RuntimeError(f"segmamba_b200 (code {rc}): {msg.decode() if msg else 'unknown error'}")


def dtype_code(t: torch.dtype) -> int:
    if t == torch.float32:
        return SMB_F32
    if t == torch.float16:
        return SMB_F16
    if t == torch.bfloat16:
        return SMB_BF16
    raise RuntimeError(f"segmamba_b200: unsupported dtype {t} (float32, float16, bfloat16 only)")


def ptr(t) -> int | None:
    return None if t is None else t.data_ptr()


def stream_ptr(device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def require_cuda(*tensors) -> None:
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError("segmamba_b200: expected CUDA tensors (the hot path has no CPU implementation)")
