"""Training augmentation of SegMamba patches on the GPU: the transforms of the reference's ``get_train_transforms``
(light_training/augment/train_augment.py:23-62, batchgenerators) as native sm_90a stages (csrc/augment.cu).

``TrainAugment(patch_size, pipeline=True, seed=0)(data, seg) -> (image, label)``.  The pipelines ``True``, ``"nomirror"``,
``"onlymirror"``, ``"onlyspatial"`` and ``False`` select the transforms of trainer.py:135-149.  Per sample, in this order:

  spatial   p 0.2 rotation (three angles U(-pi/6, pi/6)), p 0.2 scale (half/half U(0.7, 1) or U(1, 1.4)); data cubic B-spline,
            labels per label linear >= 0.5, both 0 outside the patch
  noise     p 0.1, one std U(0, 0.1) for all channels (Philox stream on the device)
  blur      p 0.2, each channel with p 0.5, sigma U(0.5, 1)
  bright    p 0.15, factor U(0.75, 1.25) per channel
  contrast  p 0.15, factor per channel (half/half over 0.75..1.25), clipped to the channel's range
  low-res   p 0.25, each channel with p 0.5: nearest down to round(shape * U(0.5, 1)), cubic back up, clipped
  gamma     inverted with p 0.1, then not inverted with p 0.3; gamma per channel (half/half over 0.7..1.5), retaining mean and std
  mirror    each axis with p 0.5; labels -1 become 0

Every random number is drawn on the host by ``AugmentSampler`` (a seeded ``numpy.random.Generator``); the device stages are
deterministic functions of those draws, so one seed gives bitwise-identical batches.  Transforms that are not drawn cost no pass.
"""
from __future__ import annotations

import ctypes
import math

import numpy as np
import torch

from . import _lib

PIPELINES = {
    True: ("spatial", "intensity", "mirror"),
    "nomirror": ("spatial", "intensity"),
    "onlymirror": ("intensity", "mirror"),
    "onlyspatial": ("spatial", "mirror"),
    False: (),
}

# per-sample probabilities of get_train_transforms; "*_channel" are the per-channel probabilities inside a drawn sample
PROBABILITIES = {"rot": 0.2, "scale": 0.2, "noise": 0.1, "blur": 0.2, "blur_channel": 0.5, "bright": 0.15, "contrast": 0.15,
                 "lowres": 0.25, "lowres_channel": 0.5, "gamma_inv": 0.1, "gamma": 0.3, "mirror": 0.5}


def pipeline_groups(pipeline) -> tuple:
    key = pipeline if isinstance(pipeline, str) else bool(pipeline)
    if key not in PIPELINES:
        raise ValueError(f"unknown augmentation pipeline {pipeline!r} (True, 'nomirror', 'onlymirror', 'onlyspatial', False)")
    return PIPELINES[key]


class AugmentSampler:
    """Draws the parameters of one sample at a time, following the draw structure of the batchgenerators transforms.

    A sample's record is a dict; a transform that was not drawn is None (for per-channel transforms, a list with None for the
    channels that were not drawn).  ``force=True`` sets every probability to 1 (every transform on every channel)."""

    def __init__(self, channels: int, pipeline=True, seed: int = 0, force: bool = False, probabilities: dict | None = None):
        self.channels = channels
        self.groups = pipeline_groups(pipeline)
        self.p = dict(PROBABILITIES)
        if probabilities:
            self.p.update(probabilities)
        if force:
            self.p = {k: 1.0 for k in self.p}
        self.rng = np.random.default_rng(seed)

    def _half(self, lo: float, hi: float) -> float:
        r = self.rng
        return float(r.uniform(lo, 1.0)) if r.random() < 0.5 and lo < 1 else float(r.uniform(max(lo, 1.0), hi))

    def _per_channel(self, p_channel: float, draw):
        return [draw() if self.rng.random() < p_channel else None for _ in range(self.channels)]

    def sample(self) -> dict:
        r, p, C = self.rng, self.p, self.channels
        rec = {k: None for k in ("rot", "scale", "noise", "blur", "bright", "contrast", "lowres", "gamma_inv", "gamma")}
        rec["mirror"] = (False, False, False)
        if "spatial" in self.groups:
            if r.random() < p["rot"]:
                rec["rot"] = tuple(float(r.uniform(-math.pi / 6, math.pi / 6)) for _ in range(3))
            if r.random() < p["scale"]:
                rec["scale"] = self._half(0.7, 1.4)
        if "intensity" in self.groups:
            if r.random() < p["noise"]:
                rec["noise"] = float(r.uniform(0.0, 0.1))
            if r.random() < p["blur"]:
                rec["blur"] = self._per_channel(p["blur_channel"], lambda: float(r.uniform(0.5, 1.0)))
            if r.random() < p["bright"]:
                rec["bright"] = [float(r.uniform(0.75, 1.25)) for _ in range(C)]
            if r.random() < p["contrast"]:
                rec["contrast"] = [self._half(0.75, 1.25) for _ in range(C)]
            if r.random() < p["lowres"]:
                rec["lowres"] = self._per_channel(p["lowres_channel"], lambda: float(r.uniform(0.5, 1.0)))
            if r.random() < p["gamma_inv"]:
                rec["gamma_inv"] = [self._half(0.7, 1.5) for _ in range(C)]
            if r.random() < p["gamma"]:
                rec["gamma"] = [self._half(0.7, 1.5) for _ in range(C)]
        if "mirror" in self.groups:
            rec["mirror"] = tuple(bool(r.random() < p["mirror"]) for _ in range(3))
        return rec


def rotation_matrix(a0: float, a1: float, a2: float) -> np.ndarray:
    """R = Rx(a0) Ry(a1) Rz(a2) of batchgenerators' rotate_coords_3d."""
    c, s = math.cos, math.sin
    rx = np.array([[1, 0, 0], [0, c(a0), -s(a0)], [0, s(a0), c(a0)]])
    ry = np.array([[c(a1), 0, s(a1)], [0, 1, 0], [-s(a1), 0, c(a1)]])
    rz = np.array([[c(a2), -s(a2), 0], [s(a2), c(a2), 0], [0, 0, 1]])
    return rx @ ry @ rz


def spatial_affine(rec: dict, patch) -> np.ndarray | None:
    """3x4 map o -> s R^T (o - c) + c, c = (P - 1) / 2; None when neither rotation nor scale was drawn."""
    if rec["rot"] is None and rec["scale"] is None:
        return None
    R = rotation_matrix(*rec["rot"]) if rec["rot"] is not None else np.eye(3)
    A = (rec["scale"] if rec["scale"] is not None else 1.0) * R.T
    c = (np.asarray(patch, dtype=np.float64) - 1) / 2
    return np.concatenate([A, (c - A @ c)[:, None]], axis=1)


def zoom_target(shape, z: float) -> tuple:
    return tuple(int(v) for v in np.round(np.asarray(shape) * z).astype(int))


# ---- thin launchers (one C-ABI call over a job list on the current stream) --------------------------------------------------
def _run(name: str, jtype, jobs: list, device) -> None:
    if not jobs:
        return
    arr = (jtype * len(jobs))(*jobs)
    fn = getattr(_lib.lib(), name)
    sp = _lib.stream_ptr(device)
    _lib.call(name, (len(jobs),), lambda: fn(arr, len(jobs), sp), device)


def _p(t: torch.Tensor | None, offset: int = 0):
    return None if t is None else t.data_ptr() + offset * t.element_size()


def prefilter_job(src, coef, shape, boundary):
    return _lib.AugPrefilterJob(_p(src), _p(coef), *shape, boundary)


def resample_job(src, dst, n, m, order, affine=None, zoom=None, clip=None):
    j = _lib.AugResampleJob(src=_p(src), dst=_p(dst), clip=_p(clip), n0=n[0], n1=n[1], n2=n[2], m0=m[0], m1=m[1], m2=m[2], order=order)
    if zoom is not None:
        j.map = _lib.AUG_ZOOM
        j.a00, j.a11, j.a22 = (n[d] / m[d] for d in range(3))
    else:
        j.map = _lib.AUG_AFFINE
        a = np.eye(3, 4) if affine is None else np.asarray(affine, dtype=np.float64)
        for r in range(3):
            for c in range(4):
                setattr(j, f"a{r}{c}", float(a[r, c]))
    return j


def stats_job(x, stats, scratch, n):
    return _lib.AugStatsJob(_p(x), _p(stats), _p(scratch), n)


def point_job(x, n, ops, stats=None, retain_ref=None, seed=0, step=0, sample=0, channel=0, noise_std=0.0, brightness=1.0,
              contrast=1.0, gamma=1.0):
    return _lib.AugPointJob(x=_p(x), stats=_p(stats), retain_ref=_p(retain_ref), n=n, seed=seed, step=step, sample=sample,
                            channel=channel, ops=ops, noise_std=noise_std, brightness=brightness, contrast=contrast, gamma=gamma)


def prefilter(jobs, device):
    _run("smb_aug_prefilter", _lib.AugPrefilterJob, jobs, device)


def resample(jobs, device):
    _run("smb_aug_resample", _lib.AugResampleJob, jobs, device)


def blur(jobs, device):
    _run("smb_aug_blur", _lib.AugBlurJob, jobs, device)


def stats(jobs, device):
    _run("smb_aug_stats", _lib.AugStatsJob, jobs, device)


def pointwise(jobs, device):
    _run("smb_aug_pointwise", _lib.AugPointJob, jobs, device)


def crop(cases: list, data: torch.Tensor, seg: torch.Tensor, patch) -> None:
    """cases: smb_aug_case records (one per sample); data (B, C, *patch) fp32, seg (B, *patch) int8, both on the device."""
    B, C = data.shape[:2]
    arr = (_lib.AugCase * B)(*cases)
    a = _lib.AugCropArgs(B, C, *patch, ctypes.cast(arr, ctypes.POINTER(_lib.AugCase)), _p(data), _p(seg))
    dev = data.device
    sp = _lib.stream_ptr(dev)
    _lib.call("smb_aug_crop", (B,), lambda: _lib.lib().smb_aug_crop(ctypes.byref(a), sp), dev)


def emit(samples: list, image: torch.Tensor, label: torch.Tensor, patch, channels: int, channels_last: bool) -> None:
    B = len(samples)
    arr = (_lib.AugEmitSample * B)(*samples)
    a = _lib.AugEmitArgs(B, channels, *patch, _lib.dtype_code(image.dtype), int(channels_last),
                         ctypes.cast(arr, ctypes.POINTER(_lib.AugEmitSample)), _p(image), _p(label))
    dev = image.device
    sp = _lib.stream_ptr(dev)
    _lib.call("smb_aug_emit", (B,), lambda: _lib.lib().smb_aug_emit(ctypes.byref(a), sp), dev)


class TrainAugment:
    """``(data (B, C, *patch) fp32 cuda, seg (B, [1,] *patch)) -> (image (B, C, *patch), label (B, *patch) int64)``.

    pipeline      True / "nomirror" / "onlymirror" / "onlyspatial" / False (trainer.py:135-149)
    seed          seeds the host sampler and keys the device noise stream
    force         every transform on every sample and channel (p = 1), for tests and measurements
    out_dtype     torch.float32 (default), torch.bfloat16 or torch.float16 image
    channels_last image in torch.channels_last_3d memory format

    Kernels run on the current CUDA stream; the call does not synchronise with the host.  Work buffers are kept per shape.
    """

    def __init__(self, patch_size, pipeline=True, seed: int = 0, force: bool = False, probabilities: dict | None = None,
                 out_dtype: torch.dtype = torch.float32, channels_last: bool = False):
        self.patch = tuple(int(v) for v in patch_size)
        if len(self.patch) != 3 or min(self.patch) < 8 or max(self.patch) > 256:
            raise ValueError(f"patch_size must be three axes of 8..256 voxels, got {patch_size}")
        self.pipeline, self.seed, self.force, self.probabilities = pipeline, int(seed), force, probabilities
        pipeline_groups(pipeline)
        self.out_dtype, self.channels_last = out_dtype, channels_last
        self.sampler = None
        self.step = 0
        self._buf = None

    # -- buffers ---------------------------------------------------------------------------------------------------------
    def buffers(self, B: int, C: int, device) -> dict:
        key = (B, C, str(device))
        if self._buf is None or self._buf["key"] != key:
            P = self.patch
            vol = P[0] * P[1] * P[2]
            evol = (P[0] + 4) * (P[1] + 4) * (P[2] + 4)
            self._buf = {"key": key,
                         "x": torch.empty((B, C) + P, dtype=torch.float32, device=device),
                         "s0": torch.empty((B,) + P, dtype=torch.int8, device=device),
                         "s1": torch.empty((B,) + P, dtype=torch.int8, device=device),
                         "ext": torch.empty((B * C, evol), dtype=torch.float32, device=device),
                         "aux": torch.empty((B * C, 2 * vol), dtype=torch.float32, device=device),
                         "st": torch.empty((B * C, 6, 4), dtype=torch.float64, device=device),
                         "scr": torch.empty((B * C, _lib.AUG_STATS_SCRATCH), dtype=torch.float64, device=device)}
        if self.sampler is None or self.sampler.channels != C:
            self.sampler = AugmentSampler(C, self.pipeline, self.seed, self.force, self.probabilities)
        return self._buf

    def draw(self, B: int, C: int) -> list:
        if self.sampler is None or self.sampler.channels != C:
            self.sampler = AugmentSampler(C, self.pipeline, self.seed, self.force, self.probabilities)
        return [self.sampler.sample() for _ in range(B)]

    def __call__(self, data: torch.Tensor, seg: torch.Tensor, params: list | None = None):
        _lib.require_cuda(data, seg)
        if data.dim() != 5 or tuple(data.shape[2:]) != self.patch:
            raise ValueError(f"data must be (B, C, {self.patch}), got {tuple(data.shape)}")
        if seg.dim() == 5:
            seg = seg[:, 0]
        B, C = data.shape[:2]
        buf = self.buffers(B, C, data.device)
        buf["x"].copy_(data)
        buf["s0"].copy_(seg)
        return self.run(params if params is not None else self.draw(B, C))

    # -- the chain on the work buffers (x, s0 filled by the caller) -----------------------------------------------------
    def run(self, params: list, step: int | None = None):
        buf = self._buf
        x, s0, s1, ext, aux, st, scr = (buf[k] for k in ("x", "s0", "s1", "ext", "aux", "st", "scr"))
        B, C = x.shape[:2]
        dev = x.device
        P = self.patch
        vol = P[0] * P[1] * P[2]
        step = self.step if step is None else step
        self.step = step + 1
        X = lambda b, c: x[b, c]
        pair = lambda b, c: b * C + c
        S = lambda b, c, k: st[pair(b, c), k]
        SCR = lambda b, c: scr[pair(b, c)]
        seg_now = [s0] * B

        # spatial
        pre, res = [], []
        for b, rec in enumerate(params):
            A = spatial_affine(rec, P)
            if A is None:
                continue
            for c in range(C):
                pre.append(prefilter_job(X(b, c), ext[pair(b, c)], P, _lib.AUG_MIRROR))
                res.append(resample_job(ext[pair(b, c)], X(b, c), P, P, 3, affine=A))
            res.append(resample_job(s0[b], s1[b], P, P, 1, affine=A))
            seg_now[b] = s1
        prefilter(pre, dev)
        resample(res, dev)

        def has(rec, key, c=None):
            v = rec[key]
            return v is not None and (c is None or not isinstance(v, list) or v[c] is not None)

        pairs = [(b, c, rec) for b, rec in enumerate(params) for c in range(C)]
        # noise on its own pass when a blur or a contrast follows it
        noise_alone = lambda b, c, rec: has(rec, "noise") and (has(rec, "blur", c) or has(rec, "contrast"))
        nz = lambda b, c, rec, ops: dict(seed=self.seed, step=step, sample=b, channel=c, noise_std=rec["noise"]) if ops & _lib.OP_NOISE else {}
        pointwise([point_job(X(b, c), vol, _lib.OP_NOISE, **nz(b, c, rec, _lib.OP_NOISE))
                   for b, c, rec in pairs if noise_alone(b, c, rec)], dev)
        blur([_lib.AugBlurJob(_p(X(b, c)), _p(aux[pair(b, c)]), rec["blur"][c], *P) for b, c, rec in pairs if has(rec, "blur", c)], dev)
        stats([stats_job(X(b, c), S(b, c, 0), SCR(b, c), vol) for b, c, rec in pairs if has(rec, "contrast")], dev)
        jobs = []
        for b, c, rec in pairs:
            ops = (_lib.OP_NOISE if has(rec, "noise") and not noise_alone(b, c, rec) else 0) | \
                  (_lib.OP_BRIGHT if has(rec, "bright") else 0) | (_lib.OP_CONTRAST if has(rec, "contrast") else 0)
            if ops:
                jobs.append(point_job(X(b, c), vol, ops, stats=S(b, c, 0) if ops & _lib.OP_CONTRAST else None,
                                      brightness=rec["bright"][c] if has(rec, "bright") else 1.0,
                                      contrast=rec["contrast"][c] if has(rec, "contrast") else 1.0, **nz(b, c, rec, ops)))
        pointwise(jobs, dev)

        # low resolution: nearest down into aux, its range, edge-variant prefilter into ext, cubic up clipped to that range
        lr = [(b, c, zoom_target(P, rec["lowres"][c])) for b, c, rec in pairs if has(rec, "lowres", c)]
        resample([resample_job(X(b, c), aux[pair(b, c)], P, t, 0, zoom=True) for b, c, t in lr], dev)
        stats([stats_job(aux[pair(b, c)], S(b, c, 1), SCR(b, c), t[0] * t[1] * t[2]) for b, c, t in lr], dev)
        prefilter([prefilter_job(aux[pair(b, c)], ext[pair(b, c)], t, _lib.AUG_EDGE) for b, c, t in lr], dev)
        resample([resample_job(ext[pair(b, c)], X(b, c), t, P, 3, zoom=True, clip=S(b, c, 1)) for b, c, t in lr], dev)

        # gamma, inverted: power pass, then retain (+ undo the inversion)
        g1 = [(b, c, rec) for b, c, rec in pairs if has(rec, "gamma_inv")]
        stats([stats_job(X(b, c), S(b, c, 2), SCR(b, c), vol) for b, c, _ in g1], dev)
        pointwise([point_job(X(b, c), vol, _lib.OP_INVERT | _lib.OP_GAMMA, stats=S(b, c, 2), gamma=rec["gamma_inv"][c])
                   for b, c, rec in g1], dev)
        stats([stats_job(X(b, c), S(b, c, 3), SCR(b, c), vol) for b, c, _ in g1], dev)
        pointwise([point_job(X(b, c), vol, _lib.OP_RETAIN | _lib.OP_UNINVERT, stats=S(b, c, 3), retain_ref=S(b, c, 2))
                   for b, c, _ in g1], dev)
        # gamma, not inverted
        g2 = [(b, c, rec) for b, c, rec in pairs if has(rec, "gamma")]
        stats([stats_job(X(b, c), S(b, c, 4), SCR(b, c), vol) for b, c, _ in g2], dev)
        pointwise([point_job(X(b, c), vol, _lib.OP_GAMMA, stats=S(b, c, 4), gamma=rec["gamma"][c]) for b, c, rec in g2], dev)
        stats([stats_job(X(b, c), S(b, c, 5), SCR(b, c), vol) for b, c, _ in g2], dev)
        pointwise([point_job(X(b, c), vol, _lib.OP_RETAIN, stats=S(b, c, 5), retain_ref=S(b, c, 4)) for b, c, _ in g2], dev)

        # mirror, layout, labels
        mf = _lib.AugEmitSample
        samples = [mf(_p(x[b]), _p(seg_now[b][b]), sum(1 << a for a in range(3) if rec["mirror"][a])) for b, rec in enumerate(params)]
        if self.channels_last:
            image = torch.empty((B, C) + P, dtype=self.out_dtype, device=dev, memory_format=torch.channels_last_3d)
        else:
            image = torch.empty((B, C) + P, dtype=self.out_dtype, device=dev)
        label = torch.empty((B,) + P, dtype=torch.int64, device=dev)
        emit(samples, image, label, P, C, self.channels_last)
        return image, label
