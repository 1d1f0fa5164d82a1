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


class Conv3dArgs(ctypes.Structure):
    _fields_ = ([(n, _i32) for n in ("batch", "d", "h", "w", "c_in", "c_out", "dtype")]
                + [(n, _vp) for n in ("x", "weight", "y", "dy", "dweight")])


# training-patch augmentation (include/segmamba_b200.h, "Training-patch sampling and augmentation")
_f64, _f32 = ctypes.c_double, ctypes.c_float


class AugCase(ctypes.Structure):
    _fields_ = ([("data", _vp), ("seg", _vp)] + [(n, _i64) for n in ("data_cs", "data_zs", "data_ys", "seg_zs", "seg_ys")]
                + [(n, _i32) for n in ("D", "H", "W", "lz", "ly", "lx")])


class AugCropArgs(ctypes.Structure):
    _fields_ = ([(n, _i32) for n in ("batch", "channels", "pd", "ph", "pw")]
                + [("cases", ctypes.POINTER(AugCase)), ("data", _vp), ("seg", _vp)])


class AugPrefilterJob(ctypes.Structure):
    _fields_ = [("src", _vp), ("coef", _vp)] + [(n, _i32) for n in ("n0", "n1", "n2", "boundary")]


class AugResampleJob(ctypes.Structure):
    _fields_ = ([("src", _vp), ("dst", _vp), ("clip", _vp)]
                + [(n, _i32) for n in ("n0", "n1", "n2", "m0", "m1", "m2", "order", "map")]
                + [(f"a{r}{c}", _f64) for r in range(3) for c in range(4)])


class AugBlurJob(ctypes.Structure):
    _fields_ = [("x", _vp), ("tmp", _vp), ("sigma", _f32)] + [(n, _i32) for n in ("n0", "n1", "n2")]


class AugStatsJob(ctypes.Structure):
    _fields_ = [("x", _vp), ("stats", _vp), ("scratch", _vp), ("n", _i64)]


class AugPointJob(ctypes.Structure):
    _fields_ = ([("x", _vp), ("stats", _vp), ("retain_ref", _vp), ("n", _i64), ("seed", _i64)]
                + [(n, _i32) for n in ("step", "sample", "channel", "ops")]
                + [(n, _f32) for n in ("noise_std", "brightness", "contrast", "gamma")])


class AugEmitSample(ctypes.Structure):
    _fields_ = [("data", _vp), ("seg", _vp), ("flip", _i32)]


class AugEmitArgs(ctypes.Structure):
    _fields_ = ([(n, _i32) for n in ("batch", "channels", "pd", "ph", "pw", "out_dtype", "channels_last")]
                + [("samples", ctypes.POINTER(AugEmitSample)), ("image", _vp), ("label", _vp)])


AUG_MIRROR, AUG_EDGE = 0, 1
AUG_AFFINE, AUG_ZOOM = 0, 1
(OP_RETAIN, OP_UNINVERT, OP_NOISE, OP_BRIGHT, OP_CONTRAST, OP_INVERT, OP_GAMMA) = (1, 2, 4, 8, 16, 32, 64)
AUG_STATS_SCRATCH = 512


# segmentation metrics (include/segmamba_b200.h, "Segmentation metrics on the GPU")
class MetricBitsArgs(ctypes.Structure):
    _fields_ = ([("src", _vp), ("bits", _vp)] + [(n, _i64) for n in ("voxels", "sample_stride", "class_stride", "voxel_stride")]
                + [(n, _i32) for n in ("batch", "kind", "dtype", "classes")] + [("lut", ctypes.c_uint8 * 256)])


class MetricCountArgs(ctypes.Structure):
    _fields_ = ([(n, _vp) for n in ("pred", "target", "pred_border", "target_border", "counts")]
                + [(n, _i32) for n in ("batch", "regions", "d", "h", "w")])


class MetricEdtArgs(ctypes.Structure):
    _fields_ = ([(n, _vp) for n in ("pred_border", "target_border", "feat", "pool", "counts")] + [("pool_cap", _i64)]
                + [(n, _i32) for n in ("batch", "regions", "d", "h", "w")] + [(n, _f64) for n in ("s0", "s1", "s2")])


class MetricSelectArgs(ctypes.Structure):
    _fields_ = ([(n, _vp) for n in ("pool", "counts", "out")] + [("pool_cap", _i64)]
                + [(n, _i32) for n in ("batch", "regions")] + [("frac", _f64)])


class MetricClassCountArgs(ctypes.Structure):
    _fields_ = ([(n, _vp) for n in ("pred", "target", "pred_border", "target_border", "record")]
                + [(n, _i32) for n in ("batch", "classes", "d", "h", "w")])


class MetricEdtJob(ctypes.Structure):
    _fields_ = ([(n, _vp) for n in ("src", "tgt", "feat", "pool", "fill", "lines")]
                + [(n, _i32) for n in ("bd", "bh", "bw", "src_mask", "src_val", "tgt_mask", "tgt_val")])


class MetricClassEdtArgs(ctypes.Structure):
    _fields_ = ([("jobs", _vp)] + [(n, _i64) for n in ("row_stride", "slice_stride")]
                + [(n, _i32) for n in ("njobs", "max_d", "max_h", "max_w")] + [(n, _f64) for n in ("s0", "s1", "s2")])


class MetricPool(ctypes.Structure):
    _fields_ = [("dist", _vp), ("lines", _vp), ("n0", _i64), ("n1", _i64), ("lines0", _i32), ("lines1", _i32)]


class MetricClassReduceArgs(ctypes.Structure):
    _fields_ = [("pools", _vp), ("out", _vp), ("npools", _i32), ("frac", _f64)]


METRIC_MAX_REGIONS, METRIC_MAX_AXIS, METRIC_NCOUNTS = 8, 768, 8
METRIC_I8, METRIC_U8, METRIC_I32, METRIC_I64, METRIC_LOGITS, METRIC_I16 = 0, 1, 2, 3, 4, 5
METRIC_MAX_CLASSES, METRIC_CLASS_NREC = 255, 11


# case prediction (include/segmamba_b200.h, "Case prediction on the GPU")
class PredRestoreArgs(ctypes.Structure):
    _fields_ = ([("src", _vp), ("out", _vp), ("class_stride", _i64), ("voxel_stride", _i64)]
                + [(n, _i32) for n in ("dtype", "classes", "regions", "d", "h", "w", "cd", "ch", "cw", "z0", "y0", "x0",
                                       "D0", "H0", "W0")] + [("lut", ctypes.c_uint8 * 256)])


class PredCcArgs(ctypes.Structure):
    _fields_ = ([(n, _vp) for n in ("mask", "out", "counts", "workspace")] + [("workspace_bytes", _sz)]
                + [(n, _i32) for n in ("batch", "d", "h", "w", "op")])


PRED_LABEL, PRED_FILL_HOLES, PRED_LARGEST = 0, 1, 2


# case preprocessing (include/segmamba_b200.h, "Case preprocessing on the GPU")
class PrepRecord(ctypes.Structure):
    _fields_ = [(n, _i64) for n in ("lo_flip0", "lo_flip1", "lo_flip2", "hi0", "hi1", "hi2", "foreground", "nan_voxels",
                                    "bad_labels")]


class PrepMaskArgs(ctypes.Structure):
    _fields_ = [(n, _vp) for n in ("data", "seg", "mask", "seg8", "record")] + [(n, _i32) for n in ("channels", "d", "h", "w")]


class PrepCropArgs(ctypes.Structure):
    _fields_ = ([(n, _vp) for n in ("data", "mask", "seg8", "out", "seg_out")]
                + [(n, _i32) for n in ("channels", "d", "h", "w", "z0", "y0", "x0", "cd", "ch", "cw", "nonzero_label")])


class PrepNormJob(ctypes.Structure):
    _fields_ = [(n, _vp) for n in ("src", "dst", "stats", "moments")] + [("n", _i64)]


class PrepCtNormJob(ctypes.Structure):
    _fields_ = [("src", _vp), ("dst", _vp), ("n", _i64)] + [(n, ctypes.c_float) for n in ("lo", "hi", "mean", "div")]


class PrepLabelResizeArgs(ctypes.Structure):
    _fields_ = [("src", _vp), ("dst", _vp)] + [(n, _i32) for n in ("n0", "n1", "n2", "m0", "m1", "m2")]


class PrepCompactJob(ctypes.Structure):
    _fields_ = [(n, _vp) for n in ("seg", "chunk", "count", "index")] + [("n", _i64), ("set", ctypes.c_uint32 * 8)]


class PrepGatherArgs(ctypes.Structure):
    _fields_ = ([(n, _vp) for n in ("index", "select", "rows", "data", "values")]
                + [(n, _i64) for n in ("n", "channel_stride", "select_channel_stride")]
                + [(n, _i32) for n in ("channels", "d", "h", "w")])


PREP_CHUNK, PREP_MAX_JOBS = 1024, 8


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
    "smb_conv3d": (ctypes.c_int, [ctypes.POINTER(Conv3dArgs), _vp]),
    "smb_conv3d_wgrad": (ctypes.c_int, [ctypes.POINTER(Conv3dArgs), _vp]),
    "smb_copy2d": (ctypes.c_int, [_vp, _i64, _vp, _i64, _i64, _i64, _vp]),
    "smb_aug_crop": (ctypes.c_int, [ctypes.POINTER(AugCropArgs), _vp]),
    "smb_aug_prefilter": (ctypes.c_int, [ctypes.POINTER(AugPrefilterJob), _i32, _vp]),
    "smb_aug_resample": (ctypes.c_int, [ctypes.POINTER(AugResampleJob), _i32, _vp]),
    "smb_aug_blur": (ctypes.c_int, [ctypes.POINTER(AugBlurJob), _i32, _vp]),
    "smb_aug_stats": (ctypes.c_int, [ctypes.POINTER(AugStatsJob), _i32, _vp]),
    "smb_aug_pointwise": (ctypes.c_int, [ctypes.POINTER(AugPointJob), _i32, _vp]),
    "smb_aug_emit": (ctypes.c_int, [ctypes.POINTER(AugEmitArgs), _vp]),
    "smb_metric_region_bits": (ctypes.c_int, [ctypes.POINTER(MetricBitsArgs), _vp]),
    "smb_metric_count": (ctypes.c_int, [ctypes.POINTER(MetricCountArgs), _vp]),
    "smb_metric_edt": (ctypes.c_int, [ctypes.POINTER(MetricEdtArgs), _vp]),
    "smb_metric_select": (ctypes.c_int, [ctypes.POINTER(MetricSelectArgs), _vp]),
    "smb_metric_class_count": (ctypes.c_int, [ctypes.POINTER(MetricClassCountArgs), _vp]),
    "smb_metric_class_edt": (ctypes.c_int, [ctypes.POINTER(MetricClassEdtArgs), _vp]),
    "smb_metric_class_reduce": (ctypes.c_int, [ctypes.POINTER(MetricClassReduceArgs), _vp]),
    "smb_pred_restore": (ctypes.c_int, [ctypes.POINTER(PredRestoreArgs), _vp]),
    "smb_pred_cc_workspace_bytes": (_sz, [_i32, _i32, _i32, _i32]),
    "smb_pred_cc": (ctypes.c_int, [ctypes.POINTER(PredCcArgs), _vp]),
    "smb_prep_mask": (ctypes.c_int, [ctypes.POINTER(PrepMaskArgs), _vp]),
    "smb_prep_crop": (ctypes.c_int, [ctypes.POINTER(PrepCropArgs), _vp]),
    "smb_prep_normalize": (ctypes.c_int, [ctypes.POINTER(PrepNormJob), _i32, _vp]),
    "smb_prep_ct_normalize": (ctypes.c_int, [ctypes.POINTER(PrepCtNormJob), _i32, _vp]),
    "smb_prep_label_resize": (ctypes.c_int, [ctypes.POINTER(PrepLabelResizeArgs), _vp]),
    "smb_prep_count": (ctypes.c_int, [ctypes.POINTER(PrepCompactJob), _i32, _vp]),
    "smb_prep_compact": (ctypes.c_int, [ctypes.POINTER(PrepCompactJob), _i32, _vp]),
    "smb_prep_gather": (ctypes.c_int, [ctypes.POINTER(PrepGatherArgs), _vp]),
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
