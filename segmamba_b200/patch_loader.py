"""GPU-resident training patch loader: the crop of the reference's ``DataLoaderMultiProcess``
(light_training/dataloading/base_data_loader.py:39-213) followed by ``TrainAugment`` (segmamba_b200/augment.py), yielding
``(image, label)`` on the device as the reference trainer's ``get_input`` does (3_train.py:75-80).

A case is a dict with ``data`` (C, D, H, W) float32, ``seg`` (1, D, H, W) integer labels and ``class_locations``
({label: (K, 4) array of (channel, z, y, x) rows}).  ``data`` and ``seg`` may be CUDA tensors, or page-locked host tensors:
then the crop kernel reads the crop box through the host mapping, so only the box crosses the bus, on the loader's stream.

    loader = GpuPatchLoader(load_preprocessed("fullres/train"), (128, 128, 128), batch_size=2, seed=0)
    for step, (image, label) in zip(range(steps), loader):
        loss = train_step(image, label)
"""
from __future__ import annotations

import glob
import os
import pickle

import numpy as np
import torch

from . import _lib
from . import augment as aug


def class_locations_from_seg(seg, max_per_class: int = 10000, seed: int = 0) -> dict:
    """{label: (K, 4) int64 rows (channel, z, y, x)} for every label > 0 of ``seg`` (1, D, H, W), at most ``max_per_class``
    voxels per label drawn without replacement: the ``class_locations`` of the reference's preprocessing .pkl."""
    s = seg.cpu().numpy() if isinstance(seg, torch.Tensor) else np.asarray(seg)
    rng = np.random.default_rng(seed)
    out = {}
    for c in np.unique(s):
        if c <= 0:
            continue
        loc = np.argwhere(s == c)
        if len(loc) > max_per_class:
            loc = loc[np.sort(rng.choice(len(loc), max_per_class, replace=False))]
        out[int(c)] = loc.astype(np.int64)
    return out


def load_preprocessed(directory: str, device=None) -> list:
    """cases of the reference's preprocessed layout (dataset.py:57-77): ``<case>.npy`` data, ``<case>_seg.npy`` labels,
    ``<case>.pkl`` properties holding ``class_locations``.  device None: page-locked host tensors; else moved there."""
    cases = []
    for path in sorted(glob.glob(os.path.join(directory, "*.npy"))):
        if path.endswith("_seg.npy"):
            continue
        stem = path[:-4]
        data = torch.from_numpy(np.ascontiguousarray(np.load(path), dtype=np.float32))
        seg = torch.from_numpy(np.ascontiguousarray(np.load(stem + "_seg.npy")).astype(np.int8))
        with open(stem + ".pkl", "rb") as f:
            props = pickle.load(f)
        if device is None:
            data, seg = data.pin_memory(), seg.pin_memory()
        else:
            data, seg = data.to(device), seg.to(device)
        cases.append({"data": data, "seg": seg, "class_locations": props["class_locations"], "name": os.path.basename(stem)})
    return cases


def get_bbox(rng: np.random.Generator, data_shape, patch_size, force_fg: bool, class_locations: dict | None):
    """lower / upper crop corners, as DataLoaderMultiProcess.get_bbox (base_data_loader.py:161-213) with need_to_pad = 0."""
    dim = len(data_shape)
    need_to_pad = [max(0, patch_size[d] - data_shape[d]) for d in range(dim)]
    lbs = [-(need_to_pad[d] // 2) for d in range(dim)]
    ubs = [data_shape[d] + need_to_pad[d] // 2 + need_to_pad[d] % 2 - patch_size[d] for d in range(dim)]
    bbox_lbs = None
    if force_fg and class_locations is not None:
        eligible = [k for k in class_locations.keys() if len(class_locations[k]) > 0]
        if eligible:
            voxels = class_locations[eligible[int(rng.integers(len(eligible)))]]
            v = voxels[int(rng.integers(len(voxels)))]
            bbox_lbs = [max(lbs[d], int(v[d + 1]) - patch_size[d] // 2) for d in range(dim)]
    if bbox_lbs is None:
        bbox_lbs = [int(rng.integers(lbs[d], ubs[d] + 1)) for d in range(dim)]
    return bbox_lbs, [bbox_lbs[d] + patch_size[d] for d in range(dim)]


class GpuPatchLoader:
    """Infinite iterator of ``(image (B, C, *patch), label (B, *patch) int64)`` on ``device``.

    Cases are drawn with replacement; sample j of a batch is forced to contain foreground iff
    j >= round(B * (1 - oversample_foreground_percent)).  ``augmentation`` is a TrainAugment pipeline.  ``prefetch=True``
    prepares the next batch on a side stream while the caller uses the current one (ordered by events).
    """

    def __init__(self, cases: list, patch_size, batch_size: int = 2, oversample_foreground_percent: float = 0.33,
                 augmentation=True, seed: int = 0, device="cuda", channels_last: bool = False, prefetch: bool = False,
                 out_dtype: torch.dtype = torch.float32, force: bool = False):
        if not cases:
            raise ValueError("GpuPatchLoader needs at least one case")
        self.device = torch.device(device)
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.patch = tuple(int(v) for v in patch_size)
        self.batch_size, self.oversample = int(batch_size), float(oversample_foreground_percent)
        self.cases = [self._prepare(c) for c in cases]
        self.channels = int(self.cases[0]["data"].shape[0])
        if any(int(c["data"].shape[0]) != self.channels for c in self.cases):
            raise ValueError("all cases must have the same number of channels")
        self.rng = np.random.default_rng(seed)
        self.augment = aug.TrainAugment(self.patch, augmentation, seed=seed, force=force, out_dtype=out_dtype,
                                        channels_last=channels_last)
        self.prefetch = prefetch
        self.stream = torch.cuda.Stream(self.device) if prefetch else None
        self._pending = None

    def _prepare(self, case: dict) -> dict:
        data, seg = case["data"], case["seg"]
        if not isinstance(data, torch.Tensor):
            data = torch.from_numpy(np.ascontiguousarray(data, dtype=np.float32))
        if not isinstance(seg, torch.Tensor):
            seg = torch.from_numpy(np.ascontiguousarray(seg))
        if data.dim() != 4 or seg.dim() != 4 or seg.shape[0] != 1 or tuple(seg.shape[1:]) != tuple(data.shape[1:]):
            raise ValueError(f"a case needs data (C, D, H, W) and seg (1, D, H, W), got {tuple(data.shape)} / {tuple(seg.shape)}")
        if data.dtype != torch.float32 or data.stride(-1) != 1:
            data = data.float().contiguous()
        if seg.dtype != torch.int8 or not seg.is_contiguous():
            seg = seg.to(torch.int8).contiguous()
        for t in (data, seg):
            if t.is_cuda:
                if t.device != self.device:
                    raise ValueError(f"case tensors on {t.device}, loader on {self.device}")
            elif not t.is_pinned():
                raise ValueError("host-resident cases must be page-locked (tensor.pin_memory()); the crop reads them from the GPU")
        return {"data": data, "seg": seg, "class_locations": case.get("class_locations")}

    def __iter__(self):
        return self

    def draw(self):
        """host draws of one batch: case indices and crop corners"""
        B = self.batch_size
        keys = self.rng.choice(len(self.cases), B, replace=True)
        boxes = []
        for j, k in enumerate(keys):
            force_fg = not j < round(B * (1 - self.oversample))
            case = self.cases[int(k)]
            lbs, _ = get_bbox(self.rng, tuple(case["data"].shape[1:]), self.patch, force_fg, case["class_locations"])
            boxes.append(lbs)
        return [int(k) for k in keys], boxes

    def _produce(self):
        keys, boxes = self.draw()
        buf = self.augment.buffers(self.batch_size, self.channels, self.device)
        recs = []
        for k, lbs in zip(keys, boxes):
            d, s = self.cases[k]["data"], self.cases[k]["seg"]
            recs.append(_lib.AugCase(data=d.data_ptr(), seg=s.data_ptr(), data_cs=d.stride(0), data_zs=d.stride(1), data_ys=d.stride(2),
                                     seg_zs=s.stride(1), seg_ys=s.stride(2), D=d.shape[1], H=d.shape[2], W=d.shape[3],
                                     lz=lbs[0], ly=lbs[1], lx=lbs[2]))
        aug.crop(recs, buf["x"], buf["s0"], self.patch)
        return self.augment.run(self.augment.draw(self.batch_size, self.channels))

    def __next__(self):
        with torch.cuda.device(self.device):
            if not self.prefetch:
                return self._produce()
            cur = torch.cuda.current_stream(self.device)
            if self._pending is None:
                self._pending = self._launch(cur)
            image, label, ev = self._pending
            cur.wait_event(ev)
            image.record_stream(cur)
            label.record_stream(cur)
            self._pending = self._launch(cur)
            return image, label

    def _launch(self, consumer):
        # the side stream reuses the work buffers: it must not start before the consumer stream has enqueued everything
        # issued so far (the previous batch's emit is on the side stream, so only the consumer's use of the outputs matters)
        self.stream.wait_stream(consumer)
        with torch.cuda.stream(self.stream):
            image, label = self._produce()
            ev = torch.cuda.Event()
            ev.record(self.stream)
        return image, label, ev
