"""The augmentation kernels and the GPU patch loader on the H100, against the CPU oracle (oracle/augment_oracle.py)."""
import numpy as np
import pytest
import torch

from aug_checks import check_blur_stats_pointwise, check_chain, check_prefilter, check_resample, labels, volume
from segmamba_b200.patch_loader import GpuPatchLoader, class_locations_from_seg

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SHAPES = [(128, 128, 128), (13, 17, 19)]


@pytest.mark.parametrize("shape", SHAPES)
def test_prefilter(shape):
    e = check_prefilter(shape, DEV)
    assert e["mirror"] < 1e-4 and e["edge"] < 1e-4, e


@pytest.mark.parametrize("shape", SHAPES)
def test_resample(shape):
    e = check_resample(shape, DEV)
    assert e["order3"] < 1e-4 and e["up"] < 1e-4 and e["down"] == 0 and e["seg_mismatch"] == 0, e
    assert e["lowres"] < 1e-4, e


@pytest.mark.parametrize("shape", SHAPES)
def test_blur_stats_pointwise(shape):
    e = check_blur_stats_pointwise(shape, DEV)
    assert e["blur"] < 1e-5 and e["stats"] < 1e-6 and e["noise"] < 1e-6 and e["contrast"] < 1e-5 and e["gamma"] < 1e-5, e


@pytest.mark.parametrize("shape", SHAPES)
def test_whole_chain_forced(shape):
    r = check_chain(shape, DEV)
    assert r["crop_exact"] and r["chain"] < 1e-3 and r["seg_mismatch"] == 0, {k: v for k, v in r.items() if k not in ("image", "label")}


def _cases(n=3, shape=(40, 48, 44), C=4, device=DEV):
    out = []
    for i in range(n):
        data = torch.from_numpy(np.stack([volume(shape, 20 + 4 * i + c) for c in range(C)]))
        seg = torch.from_numpy(labels(shape, 30 + i)[None])
        locs = class_locations_from_seg(seg, 1000, seed=i)
        if device == "pinned":
            data, seg = data.pin_memory(), seg.pin_memory()
        else:
            data, seg = data.to(device), seg.to(device)
        out.append({"data": data, "seg": seg, "class_locations": locs})
    return out


def _batches(loader, k):
    return [tuple(t.clone() for t in next(loader)) for _ in range(k)]


def test_loader_deterministic_prefetch_and_pinned():
    patch = (32, 32, 32)
    a = _batches(GpuPatchLoader(_cases(), patch, seed=7, force=True), 3)
    b = _batches(GpuPatchLoader(_cases(), patch, seed=7, force=True), 3)
    c = _batches(GpuPatchLoader(_cases(), patch, seed=7, force=True, prefetch=True), 3)
    d = _batches(GpuPatchLoader(_cases(device="pinned"), patch, seed=7, force=True), 3)
    torch.cuda.synchronize()
    for other in (b, c, d):
        for (i0, l0), (i1, l1) in zip(a, other):
            assert torch.equal(i0, i1) and torch.equal(l0, l1)
    img, lab = a[0]
    assert img.shape == (2, 4) + patch and img.dtype == torch.float32 and lab.dtype == torch.int64 and lab.min() >= 0
    assert not torch.equal(a[0][0], a[1][0])


def test_loader_reference_probabilities_and_layout():
    loader = GpuPatchLoader(_cases(), (32, 32, 32), batch_size=3, seed=1, channels_last=True, out_dtype=torch.bfloat16)
    img, lab = next(loader)
    torch.cuda.synchronize()
    assert img.is_contiguous(memory_format=torch.channels_last_3d) and img.dtype == torch.bfloat16 and lab.shape == (3, 32, 32, 32)
    assert torch.isfinite(img.float()).all()
    # the last sample is forced to foreground (round(3 * 0.67) = 2)
    for _ in range(5):
        _, lab = next(loader)
        assert int((lab[2] > 0).sum()) > 0


def test_loader_does_not_synchronize():
    loader = GpuPatchLoader(_cases(), (32, 32, 32), seed=3, force=True)
    next(loader)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(2):
            next(loader)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def test_tiny_segmamba_trains_from_the_loader():
    from segmamba_b200.segmamba import SegMamba
    from segmamba_b200.train_step import TrainStep, reference_optimizer
    torch.manual_seed(0)
    m = SegMamba(in_chans=4, out_chans=4, depths=[1, 1, 1, 1], feat_size=[48, 32, 32, 64], hidden_size=64).to(DEV)
    step = TrainStep(m, reference_optimizer(m), torch.nn.CrossEntropyLoss())
    loader = GpuPatchLoader(_cases(), (32, 32, 32), batch_size=2, seed=0)
    losses = [float(step(*next(loader))) for _ in range(3)]
    assert all(np.isfinite(losses)), losses
