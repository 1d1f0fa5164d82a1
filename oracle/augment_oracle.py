"""CPU restatement (numpy / scipy, float64) of the training-patch crop and augmentation of segmamba_b200/augment.py, from the
same parameter records and the same Philox noise values.  Test infrastructure only: the product never imports it.

Each stage follows the batchgenerators transform it replaces (see segmamba_b200/augment.py for the list); the resampling stages
call scipy.ndimage exactly as batchgenerators / skimage do.
"""
from __future__ import annotations

import numpy as np
import scipy.ndimage as ndi

M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
_U32 = 0xFFFFFFFF


def philox4x32_10(counter, key) -> np.ndarray:
    """Philox4x32-10 on arrays: counter (4, N) uint32-valued, key (k0, k1) -> (4, N) uint64 holding 32-bit words."""
    c = [np.asarray(v, dtype=np.uint64) & _U32 for v in counter]
    k0, k1 = np.uint64(key[0] & _U32), np.uint64(key[1] & _U32)
    for _ in range(10):
        p0 = np.uint64(M0) * c[0]
        p1 = np.uint64(M1) * c[2]
        hi0, lo0 = p0 >> np.uint64(32), p0 & np.uint64(_U32)
        hi1, lo1 = p1 >> np.uint64(32), p1 & np.uint64(_U32)
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
        k0 = (k0 + np.uint64(W0)) & np.uint64(_U32)
        k1 = (k1 + np.uint64(W1)) & np.uint64(_U32)
    return np.stack(c)


def normals(n: int, seed: int, step: int, sample: int, channel: int) -> np.ndarray:
    """the device's N(0, 1) values for voxels 0 .. n-1: Box-Muller on Philox((voxel / 4, step, sample, channel), seed)."""
    q = np.arange((n + 3) // 4, dtype=np.uint64)
    ones = np.ones_like(q)
    seed &= (1 << 64) - 1
    w = philox4x32_10([q, ones * step, ones * sample, ones * channel], (seed & _U32, seed >> 32)).astype(np.float64)
    u = (w + 0.5) * 2.0 ** -32
    out = np.empty((4, len(q)))
    for h in range(2):
        r = np.sqrt(-2.0 * np.log(u[2 * h]))
        th = 2 * np.pi * u[2 * h + 1]
        out[2 * h], out[2 * h + 1] = r * np.cos(th), r * np.sin(th)
    return out.T.reshape(-1)[:n]


# ---- crop ------------------------------------------------------------------------------------------------------------------
def crop(data: np.ndarray, seg: np.ndarray, lbs, patch):
    """(C, D, H, W), (D, H, W) -> patch at lower corner lbs, zero outside (base_data_loader.py:87-113)."""
    shape = data.shape[1:]
    ubs = [lbs[d] + patch[d] for d in range(3)]
    v_lo = [max(0, lbs[d]) for d in range(3)]
    v_hi = [min(shape[d], ubs[d]) for d in range(3)]
    pad = [(-min(0, lbs[d]), max(ubs[d] - shape[d], 0)) for d in range(3)]
    sl = tuple(slice(a, b) for a, b in zip(v_lo, v_hi))
    d = np.pad(data[(slice(None),) + sl], [(0, 0)] + pad, "constant", constant_values=0)
    s = np.pad(seg[sl], pad, "constant", constant_values=0)
    return d, s


# ---- spline machinery ------------------------------------------------------------------------------------------------------
def prefilter(x: np.ndarray, boundary: str) -> np.ndarray:
    """coefficients on the (n + 4)^3 grid of smb_aug_prefilter; boundary 'mirror' or 'edge'."""
    if boundary == "mirror":
        c = ndi.spline_filter(np.asarray(x, np.float64), order=3, mode="mirror")
        return np.pad(c, 2, mode="reflect")                     # numpy 'reflect' = whole-sample mirror
    padded = np.pad(np.asarray(x, np.float64), 12, mode="edge")
    c = ndi.spline_filter(padded, order=3, mode="nearest")
    return c[10:-10, 10:-10, 10:-10]


def spatial_coords(A: np.ndarray, patch) -> np.ndarray:
    o = np.stack(np.meshgrid(*[np.arange(p, dtype=np.float64) for p in patch], indexing="ij"))
    return np.einsum("de,e...->d...", A[:, :3], o) + A[:, 3].reshape(3, 1, 1, 1)


def resample_data(x: np.ndarray, A: np.ndarray) -> np.ndarray:
    """map_coordinates(order=3, mode='constant', cval=0) of batchgenerators' interpolate_img."""
    return ndi.map_coordinates(np.asarray(x, np.float64), spatial_coords(A, x.shape), order=3, mode="constant", cval=0.0)


def resample_seg(seg: np.ndarray, A: np.ndarray):
    """batchgenerators interpolate_img(is_seg=True): labels in order of first appearance; returns (labels, max indicator
    distance from 0.5 per voxel over all labels, for tie tolerance)."""
    coords = spatial_coords(A, seg.shape)
    flat = seg.ravel()
    _, first = np.unique(flat, return_index=True)
    labels = flat[np.sort(first)]
    out = np.zeros(seg.shape, seg.dtype)
    near = np.full(seg.shape, np.inf)
    for c in labels:
        ind = ndi.map_coordinates((seg == c).astype(np.float64), coords, order=1, mode="constant", cval=-1)
        out[ind >= 0.5] = c
        near = np.minimum(near, np.abs(ind - 0.5))
    return out, near


def resize(x: np.ndarray, shape, order: int) -> np.ndarray:
    """skimage.transform.resize(mode='edge', anti_aliasing=False): zoom(grid_mode, mode 'nearest'), clipped to the input range."""
    x = np.asarray(x, np.float64)
    zoom = np.asarray(shape, np.float64) / np.asarray(x.shape, np.float64)
    y = ndi.zoom(x, zoom, order=order, mode="nearest", grid_mode=True)
    assert y.shape == tuple(shape)
    return np.clip(y, x.min(), x.max())


def lowres(x: np.ndarray, z: float) -> np.ndarray:
    t = tuple(int(v) for v in np.round(np.asarray(x.shape) * z).astype(int))
    return resize(resize(x, t, 0), x.shape, 3)


def blur(x: np.ndarray, sigma: float) -> np.ndarray:
    return ndi.gaussian_filter(np.asarray(x, np.float64), sigma, mode="reflect", truncate=4.0)


def stats(x: np.ndarray) -> np.ndarray:
    x = np.asarray(x, np.float64)
    return np.array([x.sum(), (x * x).sum(), x.min(), x.max()])


def contrast(x, f):
    mn, lo, hi = x.mean(), x.min(), x.max()
    return np.clip((x - mn) * f + mn, lo, hi)


def gamma(x, g, invert):
    if invert:
        x = -x
    mn, sd = x.mean(), x.std()
    lo = x.min()
    rng = x.max() - lo
    x = ((x - lo) / (rng + 1e-7)) ** g * rng + lo
    x = (x - x.mean()) / (x.std() + 1e-8) * sd + mn
    return -x if invert else x


# ---- the whole chain -------------------------------------------------------------------------------------------------------
def augment_sample(data: np.ndarray, seg: np.ndarray, rec: dict, seed: int, step: int, sample: int, spatial_affine):
    """one sample (C, *P), (*P) through every drawn transform; returns (image float64, label int64, seg tie distance or None)."""
    x = np.asarray(data, np.float64).copy()
    s = np.asarray(seg).copy()
    C = x.shape[0]
    near = None
    A = spatial_affine(rec, x.shape[1:])
    if A is not None:
        x = np.stack([resample_data(x[c], A) for c in range(C)])
        s, near = resample_seg(s, A)
    n = x[0].size
    if rec["noise"] is not None:
        for c in range(C):
            x[c] += rec["noise"] * normals(n, seed, step, sample, c).reshape(x[c].shape)
    if rec["blur"] is not None:
        for c in range(C):
            if rec["blur"][c] is not None:
                x[c] = blur(x[c], rec["blur"][c])
    if rec["bright"] is not None:
        for c in range(C):
            x[c] *= rec["bright"][c]
    if rec["contrast"] is not None:
        for c in range(C):
            x[c] = contrast(x[c], rec["contrast"][c])
    if rec["lowres"] is not None:
        for c in range(C):
            if rec["lowres"][c] is not None:
                x[c] = lowres(x[c], rec["lowres"][c])
    if rec["gamma_inv"] is not None:
        for c in range(C):
            x[c] = gamma(x[c], rec["gamma_inv"][c], True)
    if rec["gamma"] is not None:
        for c in range(C):
            x[c] = gamma(x[c], rec["gamma"][c], False)
    for a in range(3):
        if rec["mirror"][a]:
            x = np.flip(x, a + 1)
            s = np.flip(s, a)
            if near is not None:
                near = np.flip(near, a)
    label = np.where(s == -1, 0, s).astype(np.int64)
    return np.ascontiguousarray(x), label, near
