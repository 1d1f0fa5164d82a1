// Case prediction after the sliding window, and exact 6-connected component post-processing.
//
// Restore: one thread per voxel of the uncropped volume does what the reference's Predictor does with three full-size
// intermediates -- F.interpolate(mode="trilinear", align_corners=False) of every class channel to the crop shape in fp32,
// stored as fp16, argmax over the classes, the region conversion and the copy into the zeroed original volume.  Indices and
// weights follow ATen's area_pixel_compute_scale / area_pixel_compute_source_index / guard_index_and_lambda; an axis whose
// size does not change is copied, as ATen does.
//
// Components: a union-find over int32 linear indices in which every parent is smaller than its child, so the root of a
// component is its minimum linear index whatever order the links are made in.  Linking hooks the larger root under the
// smaller with atomicMin and retries when the hooked node had stopped being a root; finds while linking halve the path with
// plain stores of an ancestor (they only shorten paths, and a store racing a hook is made good by the hook's retry).  Stages,
// a fixed number of launches whatever the data:
//   local     one block per 4 x 8 x 32 tile: the union-find over the tile in shared memory; the parent of every voxel is
//             the global index of its tile-local root (-1: background)
//   merge     the voxels on the low faces of each tile link to their neighbours in the next tile down
//   compress  every parent becomes its root (read-only walks, one store per voxel by its owner), plus one of: roots counted
//             per 1024-voxel chunk (labelling), exact component sizes with one atomic per run of equal roots in a warp
//             (largest), or flags on the roots of background components that touch the volume boundary (hole filling)
// Numbering is the rank of the root in raster order (an ordered scan of the chunk counts, then a ballot scan inside each
// chunk), which is scipy.ndimage.label's numbering because the root is the component's first voxel.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cstdint>

#include "predict_internal.h"

namespace smb {
void count_launch();

namespace {

template <typename T> __device__ inline float as_float(T v);
template <> __device__ inline float as_float<float>(float v) { return v; }
template <> __device__ inline float as_float<__half>(__half v) { return __half2float(v); }
template <> __device__ inline float as_float<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

unsigned grid_for(int64_t work, int per_block, int jobs) {
    int64_t b = (work + per_block - 1) / per_block;
    const int64_t cap = (132 * 16 + jobs - 1) / jobs;
    if (b > cap) b = cap;
    return (unsigned)(b < 1 ? 1 : b);
}

// ---- restore ----------------------------------------------------------------------------------------------------------------
struct Axis {
    int i0, i1;
    float l0, l1;
};

// ATen's compute_source_index_and_lambda for one output index of a linear resize (align_corners=False, no scale given)
__device__ inline Axis axis_of(int dst, int in, int out) {
    Axis a;
    if (in == out) {
        a.i0 = a.i1 = dst;
        a.l0 = 1.f;
        a.l1 = 0.f;
        return a;
    }
    const float scale = (float)in / (float)out;
    float src = __fadd_rn(__fmul_rn(scale, __fadd_rn((float)dst, 0.5f)), -0.5f);
    if (src < 0.f) src = 0.f;
    const int i0 = min((int)floorf(src), in - 1);
    a.i0 = i0;
    a.i1 = i0 + (i0 < in - 1 ? 1 : 0);
    a.l1 = fminf(fmaxf(__fadd_rn(src, -(float)i0), 0.f), 1.f);
    a.l0 = __fadd_rn(1.f, -a.l1);
    return a;
}

__device__ inline float lerp2(float x0, float x1, float l0, float l1) { return __fadd_rn(__fmul_rn(x0, l0), __fmul_rn(x1, l1)); }

__device__ inline float to_half(float v) { return __half2float(__float2half_rn(v)); }

template <typename T>
__global__ void __launch_bounds__(256) restore_kernel(smb_pred_restore_args a) {
    const int64_t n0 = (int64_t)a.D0 * a.H0 * a.W0;
    const int64_t cs = a.class_stride, vs = a.voxel_stride;
    const bool ident = a.cd == a.d && a.ch == a.h && a.cw == a.w;
    const T *src = reinterpret_cast<const T *>(a.src);
    uint8_t *out = reinterpret_cast<uint8_t *>(a.out);
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < n0; v += (int64_t)gridDim.x * blockDim.x) {
        const int x = (int)(v % a.W0), y = (int)((v / a.W0) % a.H0), z = (int)(v / ((int64_t)a.W0 * a.H0));
        const int cz = z - a.z0, cy = y - a.y0, cx = x - a.x0;
        int arg = -1;
        if (cz >= 0 && cz < a.cd && cy >= 0 && cy < a.ch && cx >= 0 && cx < a.cw) {
            float best;
            if (ident) {
                const T *p = src + (((int64_t)cz * a.h + cy) * a.w + cx) * vs;
                best = to_half(as_float<T>(p[0]));
                arg = 0;
                for (int c = 1; c < a.classes && best == best; ++c) {   // the first maximum; a NaN is the maximum
                    const float s = to_half(as_float<T>(p[(int64_t)c * cs]));
                    if (s > best || s != s) { best = s; arg = c; }
                }
            } else {
                const Axis az = axis_of(cz, a.d, a.cd), ay = axis_of(cy, a.h, a.ch), ax = axis_of(cx, a.w, a.cw);
                const int64_t r00 = ((int64_t)az.i0 * a.h + ay.i0) * a.w, r01 = ((int64_t)az.i0 * a.h + ay.i1) * a.w;
                const int64_t r10 = ((int64_t)az.i1 * a.h + ay.i0) * a.w, r11 = ((int64_t)az.i1 * a.h + ay.i1) * a.w;
                const int64_t o[8] = {(r00 + ax.i0) * vs, (r00 + ax.i1) * vs, (r01 + ax.i0) * vs, (r01 + ax.i1) * vs,
                                      (r10 + ax.i0) * vs, (r10 + ax.i1) * vs, (r11 + ax.i0) * vs, (r11 + ax.i1) * vs};
                for (int c = 0; c < a.classes; ++c) {
                    const T *p = src + (int64_t)c * cs;
                    // ATen's CPU kernel nests the sums outermost axis first: d( h( w ) )
                    const float s = to_half(lerp2(
                        lerp2(lerp2(as_float<T>(p[o[0]]), as_float<T>(p[o[1]]), ax.l0, ax.l1),
                              lerp2(as_float<T>(p[o[2]]), as_float<T>(p[o[3]]), ax.l0, ax.l1), ay.l0, ay.l1),
                        lerp2(lerp2(as_float<T>(p[o[4]]), as_float<T>(p[o[5]]), ax.l0, ax.l1),
                              lerp2(as_float<T>(p[o[6]]), as_float<T>(p[o[7]]), ax.l0, ax.l1), ay.l0, ay.l1),
                        az.l0, az.l1));
                    if (c == 0 || s > best || (s != s && best == best)) { best = s; arg = c; }
                }
            }
        }
        if (a.regions == 0) {
            out[v] = arg < 0 ? (uint8_t)0 : (uint8_t)arg;
        } else {
            const uint8_t bits = (arg < 0 || arg >= 256) ? (uint8_t)0 : a.lut[arg];
            for (int r = 0; r < a.regions; ++r) out[(int64_t)r * n0 + v] = (bits >> r) & 1;
        }
    }
}

// ---- connected components ---------------------------------------------------------------------------------------------------
constexpr int kTz = 4, kTy = 8, kTx = 32, kTile = kTz * kTy * kTx;
constexpr int kCcThreads = 256, kChunk = 1024;

// parents are read around the L1 cache: other blocks link them while this one walks
__device__ inline int ldv(const int *p) { return *reinterpret_cast<const volatile int *>(p); }
__device__ inline void stv(int *p, int v) { *reinterpret_cast<volatile int *>(p) = v; }

__device__ inline int find_root(int *P, int x) {
    int p = ldv(P + x);
    while (p != x) {
        const int g = ldv(P + p);
        if (g != p) stv(P + x, g);                                      // path halving: g is an ancestor of x
        x = g;
        p = ldv(P + x);
    }
    return x;
}

// read-only find for the compress pass, whose stores must leave every parent at its root: a halving store there could land
// after the owner's store of the root and put a mere ancestor back
__device__ inline int root_of(const int *P, int x) {
    int p = ldv(P + x);
    while (p != x) {
        x = p;
        p = ldv(P + x);
    }
    return x;
}

// hook the larger root under the smaller; when the hooked node is no longer a root, retry from its new parent
__device__ inline void unite(int *P, int a, int b) {
    for (;;) {
        a = find_root(P, a);
        b = find_root(P, b);
        if (a == b) return;
        if (a > b) { const int t = a; a = b; b = t; }
        const int old = atomicMin(P + b, a);
        if (old == b) return;
        b = old;
    }
}

struct Vol {
    int d, h, w;
    int64_t n;
};

__device__ inline Vol vol_of(int d, int h, int w) { return Vol{d, h, w, (int64_t)d * h * w}; }

__device__ inline int tile_global(const Vol &V, int bz, int by, int bx, int i) {
    const int x = bx * kTx + i % kTx, y = by * kTy + (i / kTx) % kTy, z = bz * kTz + i / (kTx * kTy);
    return (x < V.w && y < V.h && z < V.d) ? (int)(((int64_t)z * V.h + y) * V.w + x) : -1;
}

// fg = (mask != 0) != invert; P[v] = global index of the tile-local root of v, -1 for background
__global__ void __launch_bounds__(kCcThreads) cc_local_kernel(const uint8_t *mask, int *P, int d, int h, int w, int invert) {
    __shared__ int L[kTile];
    const Vol V = vol_of(d, h, w);
    const int tx = (w + kTx - 1) / kTx, ty = (h + kTy - 1) / kTy;
    const int bx = (int)(blockIdx.x % tx), by = (int)((blockIdx.x / tx) % ty), bz = (int)(blockIdx.x / (tx * ty));
    const uint8_t *m = mask + (int64_t)blockIdx.y * V.n;
    int *Pb = P + (int64_t)blockIdx.y * V.n;
    for (int i = threadIdx.x; i < kTile; i += kCcThreads) {
        const int g = tile_global(V, bz, by, bx, i);
        L[i] = (g >= 0 && ((m[g] != 0) != (invert != 0))) ? i : -1;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kTile; i += kCcThreads) {
        if (ldv(L + i) < 0) continue;                                   // links never make a voxel background
        const int lx = i % kTx, ly = (i / kTx) % kTy, lz = i / (kTx * kTy);
        if (lx > 0 && ldv(L + i - 1) >= 0) unite(L, i, i - 1);
        if (ly > 0 && ldv(L + i - kTx) >= 0) unite(L, i, i - kTx);
        if (lz > 0 && ldv(L + i - kTx * kTy) >= 0) unite(L, i, i - kTx * kTy);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kTile; i += kCcThreads) {
        const int g = tile_global(V, bz, by, bx, i);
        if (g < 0) continue;
        // local order is raster order within the tile, so the local minimum maps to the global minimum
        Pb[g] = ldv(L + i) < 0 ? -1 : tile_global(V, bz, by, bx, find_root(L, i));
    }
}

// link every foreground voxel on the low face of a tile to its foreground neighbour across that face
__global__ void __launch_bounds__(kCcThreads) cc_merge_kernel(int *P, int d, int h, int w) {
    const Vol V = vol_of(d, h, w);
    int *Pb = P + (int64_t)blockIdx.y * V.n;
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < V.n; v += (int64_t)gridDim.x * blockDim.x) {
        const int x = (int)(v % w), y = (int)((v / w) % h), z = (int)(v / ((int64_t)w * h));
        const bool fx = x > 0 && x % kTx == 0, fy = y > 0 && y % kTy == 0, fz = z > 0 && z % kTz == 0;
        if (!(fx || fy || fz) || ldv(Pb + v) < 0) continue;
        const int u = (int)v;
        if (fx && ldv(Pb + u - 1) >= 0) unite(Pb, u, u - 1);
        if (fy && ldv(Pb + u - w) >= 0) unite(Pb, u, u - w);
        if (fz && ldv(Pb + u - w * h) >= 0) unite(Pb, u, u - w * h);
    }
}

enum { kCountRoots = 0, kSizes = 1, kBorder = 2 };

// P[v] = root of v, chunk by chunk (voxel k * 256 + t of the chunk for thread t), plus the per-op side result
template <int kOp>
__global__ void __launch_bounds__(kCcThreads) cc_compress_kernel(int *P, int *aux, int *chunk_roots, int d, int h, int w) {
    __shared__ int red[kCcThreads / 32];
    const Vol V = vol_of(d, h, w);
    int *Pb = P + (int64_t)blockIdx.y * V.n;
    int *Ab = aux + (int64_t)blockIdx.y * V.n;
    const int lane = threadIdx.x & 31;
    int roots = 0;
    for (int k = 0; k < kChunk / kCcThreads; ++k) {
        const int64_t v = (int64_t)blockIdx.x * kChunk + k * kCcThreads + threadIdx.x;
        int r = -1;
        if (v < V.n && ldv(Pb + v) >= 0) {
            r = root_of(Pb, (int)v);
            stv(Pb + v, r);
            roots += r == (int)v;
        }
        if (kOp == kSizes) {                                           // one atomic per run of equal roots in the warp
            const unsigned grp = __match_any_sync(0xffffffffu, r);
            if (r >= 0 && lane == __ffs(grp) - 1) atomicAdd(Ab + r, __popc(grp));
        } else if (kOp == kBorder && r >= 0) {
            const int x = (int)(v % w), y = (int)((v / w) % h), z = (int)(v / ((int64_t)w * h));
            if (x == 0 || y == 0 || z == 0 || x == w - 1 || y == h - 1 || z == d - 1) stv(Ab + r, 1);
        }
    }
    if (kOp == kCountRoots) {
        for (int o = 16; o; o >>= 1) roots += __shfl_down_sync(0xffffffffu, roots, o);
        if (lane == 0) red[threadIdx.x >> 5] = roots;
        __syncthreads();
        if (threadIdx.x == 0) {
            int s = 0;
            for (int q = 0; q < kCcThreads / 32; ++q) s += red[q];
            chunk_roots[(int64_t)blockIdx.y * gridDim.x + blockIdx.x] = s;
        }
    }
}

// per volume (one block each): exclusive scan of the chunk root counts in place, the total to counts
constexpr int kScanThreads = 1024;

__global__ void __launch_bounds__(kScanThreads) cc_scan_kernel(int *chunk_roots, int64_t *counts, int nchunks) {
    __shared__ int wsum[kScanThreads / 32];
    int *c = chunk_roots + (int64_t)blockIdx.x * nchunks;
    const int per = (nchunks + kScanThreads - 1) / kScanThreads;
    const int lo = min((int)threadIdx.x * per, nchunks), hi = min(lo + per, nchunks);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int s = 0;
    for (int i = lo; i < hi; ++i) s += c[i];
    int incl = s;
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
    }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        const int ws = wsum[lane];
        int wi = ws;
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, wi, o);
            if (lane >= o) wi += y;
        }
        wsum[lane] = wi - ws;
    }
    __syncthreads();
    int run = wsum[warp] + incl - s;
    for (int i = lo; i < hi; ++i) {
        const int t = c[i];
        c[i] = run;
        run += t;
    }
    if (threadIdx.x == kScanThreads - 1) counts[blockIdx.x] = run;
}

// labels of roots (chunk offset + rank inside the chunk + 1) and of background (0)
__global__ void __launch_bounds__(kCcThreads) cc_number_kernel(const int *P, const int *chunk_off, int *out, int d, int h, int w) {
    __shared__ int wsum[kCcThreads / 32];
    const Vol V = vol_of(d, h, w);
    const int *Pb = P + (int64_t)blockIdx.y * V.n;
    int *Ob = out + (int64_t)blockIdx.y * V.n;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int base = chunk_off[(int64_t)blockIdx.y * gridDim.x + blockIdx.x];
    for (int k = 0; k < kChunk / kCcThreads; ++k) {
        const int64_t v = (int64_t)blockIdx.x * kChunk + k * kCcThreads + threadIdx.x;
        const int p = v < V.n ? Pb[v] : -2;
        const bool root = p == (int)v;
        const unsigned m = __ballot_sync(0xffffffffu, root);
        if (lane == 0) wsum[warp] = __popc(m);
        __syncthreads();
        int before = 0, total = 0;
        for (int q = 0; q < kCcThreads / 32; ++q) {
            before += q < warp ? wsum[q] : 0;
            total += wsum[q];
        }
        if (p == -1) Ob[v] = 0;
        else if (root) Ob[v] = base + before + __popc(m & ((1u << lane) - 1u)) + 1;
        base += total;
        __syncthreads();
    }
}

__global__ void __launch_bounds__(kCcThreads) cc_gather_kernel(const int *P, int *out, int d, int h, int w) {
    const Vol V = vol_of(d, h, w);
    const int *Pb = P + (int64_t)blockIdx.y * V.n;
    int *Ob = out + (int64_t)blockIdx.y * V.n;
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < V.n; v += (int64_t)gridDim.x * blockDim.x) {
        const int p = Pb[v];
        if (p >= 0 && p != (int)v) Ob[v] = Ob[p];
    }
}

// best[b] = max over roots of size << 32 | root: the largest component, ties to the highest root (the highest label)
__global__ void __launch_bounds__(kCcThreads) cc_select_kernel(const int *P, const int *sizes, unsigned long long *best, int d, int h, int w) {
    const Vol V = vol_of(d, h, w);
    const int *Pb = P + (int64_t)blockIdx.y * V.n;
    const int *Sb = sizes + (int64_t)blockIdx.y * V.n;
    unsigned long long key = 0;
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < V.n; v += (int64_t)gridDim.x * blockDim.x) {
        if (Pb[v] == (int)v) {
            const unsigned long long k = ((unsigned long long)(unsigned)Sb[v] << 32) | (unsigned)v;
            key = k > key ? k : key;
        }
    }
    for (int o = 16; o; o >>= 1) {
        const unsigned long long y = __shfl_down_sync(0xffffffffu, key, o);
        key = y > key ? y : key;
    }
    if ((threadIdx.x & 31) == 0 && key) atomicMax(best + blockIdx.y, key);
}

__global__ void __launch_bounds__(kCcThreads) cc_keep_kernel(const int *P, const unsigned long long *best, uint8_t *keep, int d, int h, int w) {
    const Vol V = vol_of(d, h, w);
    const int *Pb = P + (int64_t)blockIdx.y * V.n;
    uint8_t *Kb = keep + (int64_t)blockIdx.y * V.n;
    const unsigned long long b = best[blockIdx.y];
    const int root = b ? (int)(unsigned)(b & 0xffffffffull) : -2;
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < V.n; v += (int64_t)gridDim.x * blockDim.x)
        Kb[v] = Pb[v] == root;
}

// P labels the background; a background voxel stays background when its component touches the boundary
__global__ void __launch_bounds__(kCcThreads) cc_fill_kernel(const int *P, const int *flags, uint8_t *out, int d, int h, int w) {
    const Vol V = vol_of(d, h, w);
    const int *Pb = P + (int64_t)blockIdx.y * V.n;
    const int *Fb = flags + (int64_t)blockIdx.y * V.n;
    uint8_t *Ob = out + (int64_t)blockIdx.y * V.n;
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < V.n; v += (int64_t)gridDim.x * blockDim.x) {
        const int p = Pb[v];
        Ob[v] = !(p >= 0 && Fb[p]);
    }
}

struct Work {
    unsigned long long *best;
    int *P, *aux, *chunk;
    uint8_t *keep;
};

size_t align16(size_t b) { return (b + 15) & ~(size_t)15; }

int64_t chunks_of(int d, int h, int w) { return ((int64_t)d * h * w + kChunk - 1) / kChunk; }

Work carve(void *ws, int batch, int d, int h, int w) {
    const size_t n = (size_t)batch * d * h * w;
    char *p = static_cast<char *>(ws);
    Work k;
    k.best = reinterpret_cast<unsigned long long *>(p);
    p += align16(8 * (size_t)batch);
    k.P = reinterpret_cast<int *>(p);
    p += align16(4 * n);
    k.aux = reinterpret_cast<int *>(p);
    p += align16(4 * n);
    k.chunk = reinterpret_cast<int *>(p);
    p += align16(4 * (size_t)batch * chunks_of(d, h, w));
    k.keep = reinterpret_cast<uint8_t *>(p);
    return k;
}

// local + merge + compress<kOp>: P holds the root of every foreground voxel of (mask != 0) != invert
template <int kOp>
cudaError_t components(const uint8_t *mask, int invert, const Work &k, int batch, int d, int h, int w, cudaStream_t st) {
    const int64_t n = (int64_t)d * h * w;
    const unsigned tiles = (unsigned)(((d + kTz - 1) / kTz) * (int64_t)((h + kTy - 1) / kTy) * ((w + kTx - 1) / kTx));
    cc_local_kernel<<<dim3(tiles, batch), kCcThreads, 0, st>>>(mask, k.P, d, h, w, invert);
    count_launch();
    cc_merge_kernel<<<dim3(grid_for(n, kCcThreads, batch), batch), kCcThreads, 0, st>>>(k.P, d, h, w);
    count_launch();
    cc_compress_kernel<kOp><<<dim3((unsigned)chunks_of(d, h, w), batch), kCcThreads, 0, st>>>(k.P, k.aux, k.chunk, d, h, w);
    count_launch();
    return cudaGetLastError();
}

cudaError_t fill_holes(const uint8_t *mask, uint8_t *out, const Work &k, int batch, int d, int h, int w, cudaStream_t st) {
    const int64_t n = (int64_t)d * h * w;
    cudaError_t e = cudaMemsetAsync(k.aux, 0, 4 * (size_t)batch * n, st);
    if (e != cudaSuccess) return e;
    e = components<kBorder>(mask, 1, k, batch, d, h, w, st);
    if (e != cudaSuccess) return e;
    cc_fill_kernel<<<dim3(grid_for(n, kCcThreads, batch), batch), kCcThreads, 0, st>>>(k.P, k.aux, out, d, h, w);
    count_launch();
    return cudaGetLastError();
}

}  // namespace

cudaError_t pred_restore_launch(const smb_pred_restore_args &a, cudaStream_t st) {
    const unsigned grid = grid_for((int64_t)a.D0 * a.H0 * a.W0, 256, 1);
    if (a.dtype == SMB_F32) restore_kernel<float><<<grid, 256, 0, st>>>(a);
    else if (a.dtype == SMB_F16) restore_kernel<__half><<<grid, 256, 0, st>>>(a);
    else restore_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>(a);
    count_launch();
    return cudaGetLastError();
}

size_t pred_cc_workspace_bytes(int batch, int d, int h, int w) {
    const size_t n = (size_t)batch * d * h * w;
    return align16(8 * (size_t)batch) + 2 * align16(4 * n) + align16(4 * (size_t)batch * chunks_of(d, h, w)) + align16(n);
}

cudaError_t pred_cc_launch(const smb_pred_cc_args &a, cudaStream_t st) {
    const int B = a.batch, d = a.d, h = a.h, w = a.w;
    const int64_t n = (int64_t)d * h * w;
    const Work k = carve(a.workspace, B, d, h, w);
    const uint8_t *mask = static_cast<const uint8_t *>(a.mask);
    const dim3 grid(grid_for(n, kCcThreads, B), B);
    cudaError_t e;
    if (a.op == SMB_PRED_LABEL) {
        e = components<kCountRoots>(mask, 0, k, B, d, h, w, st);
        if (e != cudaSuccess) return e;
        const int nchunks = (int)chunks_of(d, h, w);
        cc_scan_kernel<<<B, kScanThreads, 0, st>>>(k.chunk, a.counts, nchunks);
        count_launch();
        int *out = static_cast<int *>(a.out);
        cc_number_kernel<<<dim3((unsigned)nchunks, B), kCcThreads, 0, st>>>(k.P, k.chunk, out, d, h, w);
        count_launch();
        cc_gather_kernel<<<grid, kCcThreads, 0, st>>>(k.P, out, d, h, w);
        count_launch();
        return cudaGetLastError();
    }
    if (a.op == SMB_PRED_FILL_HOLES) return fill_holes(mask, static_cast<uint8_t *>(a.out), k, B, d, h, w, st);
    // SMB_PRED_LARGEST: sizes, the best root, its mask, then its holes filled
    e = cudaMemsetAsync(k.aux, 0, 4 * (size_t)B * n, st);
    if (e != cudaSuccess) return e;
    e = cudaMemsetAsync(k.best, 0, 8 * (size_t)B, st);
    if (e != cudaSuccess) return e;
    e = components<kSizes>(mask, 0, k, B, d, h, w, st);
    if (e != cudaSuccess) return e;
    cc_select_kernel<<<grid, kCcThreads, 0, st>>>(k.P, k.aux, k.best, d, h, w);
    count_launch();
    cc_keep_kernel<<<grid, kCcThreads, 0, st>>>(k.P, k.best, k.keep, d, h, w);
    count_launch();
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    return fill_holes(k.keep, static_cast<uint8_t *>(a.out), k, B, d, h, w, st);
}

}  // namespace smb
