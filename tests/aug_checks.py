"""Stage-by-stage comparisons of the augmentation kernels (segmamba_b200/augment.py, csrc/augment.cu) with the CPU oracle
(oracle/augment_oracle.py).  Shared by the emulator tests (CPU tensors under tests/emu.emulated()) and the GPU tests."""
import numpy as np
import torch

from oracle import augment_oracle as orc
from segmamba_b200 import _lib
from segmamba_b200 import augment as aug


def rel(got, want) -> float:
    got = np.asarray(got, np.float64)
    want = np.asarray(want, np.float64)
    return float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-30))


def _t(a, dev, dtype=torch.float32):
    return torch.tensor(np.ascontiguousarray(a)).to(device=dev, dtype=dtype)      # a copy: kernels work in place


def _sync(dev):
    if torch.device(dev).type == "cuda":
        torch.cuda.synchronize(dev)


def volume(shape, seed):
    rng = np.random.default_rng(seed)
    g = np.meshgrid(*[np.linspace(-1, 1, n) for n in shape], indexing="ij")
    return (np.sin(3 * g[0] + 1) * np.cos(2 * g[1]) + 0.5 * g[2] + 0.3 * rng.standard_normal(shape)).astype(np.float32)


def labels(shape, seed):
    g = np.meshgrid(*[np.arange(n) - n / 2 for n in shape], indexing="ij")
    r = np.sqrt(sum(x * x for x in g)) / (min(shape) / 2)
    s = np.where(r < 0.4, 3, np.where(r < 0.6, 1, np.where(r < 0.8, 2, 0))).astype(np.int8)
    s[np.random.default_rng(seed).random(shape) < 0.02] = -1
    return s


def check_prefilter(shape, dev):
    x = volume(shape, 1)
    out = {}
    for name, b in (("mirror", _lib.AUG_MIRROR), ("edge", _lib.AUG_EDGE)):
        xs = _t(x, dev)
        coef = torch.full([n + 4 for n in shape], float("nan"), device=dev)
        aug.prefilter([aug.prefilter_job(xs, coef, shape, b)], dev)
        _sync(dev)
        out[name] = rel(coef.cpu().numpy(), orc.prefilter(x, name))
    return out


def check_resample(shape, dev):
    """order 3 affine (spatial), order 1 labels, order 0 zoom down, order 3 zoom up with clip"""
    x, s = volume(shape, 2), labels(shape, 3)
    rec = {"rot": (0.3, -0.2, 0.45), "scale": 1.2}
    A = aug.spatial_affine(rec, shape)
    xs = _t(x, dev)
    coef = torch.empty([n + 4 for n in shape], device=dev)
    y = torch.empty(shape, device=dev)
    aug.prefilter([aug.prefilter_job(xs, coef, shape, _lib.AUG_MIRROR)], dev)
    segi = _t(s, dev, torch.int8)
    sego = torch.empty(shape, dtype=torch.int8, device=dev)
    aug.resample([aug.resample_job(coef, y, shape, shape, 3, affine=A), aug.resample_job(segi, sego, shape, shape, 1, affine=A)], dev)
    # low resolution of the same volume
    t = aug.zoom_target(shape, 0.61)
    down = torch.empty(t, device=dev)
    aug.resample([aug.resample_job(xs, down, shape, t, 0, zoom=True)], dev)
    st = torch.empty(4, dtype=torch.float64, device=dev)
    scr = torch.empty(_lib.AUG_STATS_SCRATCH, dtype=torch.float64, device=dev)
    aug.stats([aug.stats_job(down, st, scr, t[0] * t[1] * t[2])], dev)
    coef2 = torch.empty([n + 4 for n in t], device=dev)
    aug.prefilter([aug.prefilter_job(down, coef2, t, _lib.AUG_EDGE)], dev)
    up = torch.empty(shape, device=dev)
    aug.resample([aug.resample_job(coef2, up, t, shape, 3, zoom=True, clip=st)], dev)
    _sync(dev)
    ys, near = orc.resample_seg(s, A)
    bad = (sego.cpu().numpy() != ys) & (near > 1e-5)
    d0 = orc.resize(x, t, 0)
    return {"order3": rel(y.cpu().numpy(), orc.resample_data(x, A)), "seg_mismatch": int(bad.sum()),
            "down": rel(down.cpu().numpy(), d0), "up": rel(up.cpu().numpy(), orc.resize(d0, shape, 3)),
            "lowres": rel(up.cpu().numpy(), orc.lowres(x, 0.61))}


def check_blur_stats_pointwise(shape, dev):
    x = volume(shape, 4)
    n = x.size
    xs = _t(x, dev)
    tmp = torch.empty(2 * n, device=dev)
    aug.blur([_lib.AugBlurJob(xs.data_ptr(), tmp.data_ptr(), 0.83, *shape)], dev)
    st = torch.empty((4, 4), dtype=torch.float64, device=dev)
    scr = torch.empty((4, _lib.AUG_STATS_SCRATCH), dtype=torch.float64, device=dev)
    _sync(dev)
    out = {"blur": rel(xs.cpu().numpy(), orc.blur(x, 0.83))}
    xb = xs.cpu().numpy().astype(np.float64)
    aug.stats([aug.stats_job(xs, st[0], scr[0], n)], dev)
    _sync(dev)
    out["stats"] = rel(st[0].cpu().numpy(), orc.stats(xb))
    # noise alone
    z = _t(x, dev)
    aug.pointwise([aug.point_job(z, n, _lib.OP_NOISE, seed=99, step=5, sample=1, channel=2, noise_std=0.07)], dev)
    _sync(dev)
    out["noise"] = rel(z.cpu().numpy(), x + 0.07 * orc.normals(n, 99, 5, 1, 2).reshape(shape))
    # brightness + contrast from the entry statistics
    z = _t(x, dev)
    aug.pointwise([aug.point_job(z, n, _lib.OP_BRIGHT | _lib.OP_CONTRAST, stats=_stats(z, st[1], scr[1], n, dev), brightness=1.1,
                                 contrast=0.8)], dev)
    _sync(dev)
    out["contrast"] = rel(z.cpu().numpy(), orc.contrast(x.astype(np.float64) * 1.1, 0.8))
    # inverted gamma: power pass, then retain + uninvert
    z = _t(x, dev)
    s0 = _stats(z, st[2], scr[2], n, dev)
    aug.pointwise([aug.point_job(z, n, _lib.OP_INVERT | _lib.OP_GAMMA, stats=s0, gamma=1.37)], dev)
    s1 = _stats(z, st[3], scr[3], n, dev)
    aug.pointwise([aug.point_job(z, n, _lib.OP_RETAIN | _lib.OP_UNINVERT, stats=s1, retain_ref=s0)], dev)
    _sync(dev)
    out["gamma"] = rel(z.cpu().numpy(), orc.gamma(x.astype(np.float64), 1.37, True))
    return out


def _stats(x, st, scr, n, dev):
    aug.stats([aug.stats_job(x, st, scr, n)], dev)
    return st


def check_chain(shape, dev, C=2, B=2, seed=5, case_shape=None):
    """crop (box partly outside the case) + every transform forced, against the oracle sample by sample"""
    case_shape = case_shape or tuple(n + 6 for n in shape)
    data = np.stack([volume(case_shape, 10 + c) for c in range(C)])
    seg = labels(case_shape, 11)
    ta = aug.TrainAugment(shape, True, seed=seed, force=True)
    buf = ta.buffers(B, C, dev)
    dcase = _t(data, dev)
    scase = _t(seg, dev, torch.int8)
    boxes = [(-3, 4, -5), (5, -2, 7)][:B]
    cases = [_lib.AugCase(data=dcase.data_ptr(), seg=scase.data_ptr(), data_cs=dcase.stride(0), data_zs=dcase.stride(1),
                          data_ys=dcase.stride(2), seg_zs=scase.stride(0), seg_ys=scase.stride(1), D=case_shape[0], H=case_shape[1],
                          W=case_shape[2], lz=b[0], ly=b[1], lx=b[2]) for b in boxes]
    aug.crop(cases, buf["x"], buf["s0"], shape)
    _sync(dev)
    crops = [orc.crop(data, seg, b, shape) for b in boxes]
    crop_ok = all(np.array_equal(buf["x"][i].cpu().numpy(), crops[i][0]) and np.array_equal(buf["s0"][i].cpu().numpy(), crops[i][1])
                  for i in range(B))
    params = ta.draw(B, C)
    image, label = ta.run(params, step=3)
    _sync(dev)
    errs, seg_bad = [], 0
    for i in range(B):
        img, lab, near = orc.augment_sample(crops[i][0], crops[i][1], params[i], seed, 3, i, aug.spatial_affine)
        errs.append(rel(image[i].cpu().numpy(), img))
        got = label[i].cpu().numpy()
        seg_bad += int(((got != lab) & (near > 1e-5)).sum()) if near is not None else int((got != lab).sum())
    return {"crop_exact": crop_ok, "chain": max(errs), "seg_mismatch": seg_bad, "image": image, "label": label}
