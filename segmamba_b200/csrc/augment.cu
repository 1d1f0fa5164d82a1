// Training-patch crop and augmentation (the CPU data path of the reference trainer, base_data_loader.py:39-213 and
// train_augment.py:23-62, as GPU stages).  The host draws every random parameter and composes the stages
// (segmamba_b200/augment.py); each kernel here is a deterministic function of its job records.
//
// What bounds them: all are HBM-streaming passes over 4-byte voxels except the cubic resample (64 gathered taps per voxel out of
// L1 / L2, the coefficient volume of one channel is 9 MB and stays resident in the 50 MB L2) and the prefilter (a two-pass
// recursive filter per line, one thread per line, lines of up to 256 samples staged in shared memory, longer ones streamed).
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>

#include "aug_internal.h"

namespace smb {
void count_launch();

namespace {

template <class T> struct Jobs {
    T j[kAugMaxJobs];
    int n;
};

constexpr float kPole = -0.26794919243112270f;   // sqrt(3) - 2, the pole of the cubic B-spline prefilter

__host__ __device__ inline int mirror_index(int i, int n) {    // whole-sample symmetric: -1 -> 1, n -> n - 2
    if (n == 1) return 0;
    const int p = 2 * (n - 1);
    i = i < 0 ? -i : i;
    i %= p;
    return i >= n ? p - i : i;
}

__device__ inline int reflect_index(int i, int n) {             // half-sample symmetric: -1 -> 0, n -> n - 1
    const int p = 2 * n;
    i %= p;
    if (i < 0) i += p;
    return i >= n ? p - 1 - i : i;
}

__device__ inline void bspline3(float t, float w[4]) {          // weights of taps floor(x) - 1 .. floor(x) + 2, t = x - floor(x)
    const float s = 1.f - t;
    w[0] = s * s * s * (1.f / 6.f);
    w[1] = (2.f / 3.f) - t * t + 0.5f * t * t * t;
    w[2] = (2.f / 3.f) - s * s + 0.5f * s * s * s;
    w[3] = t * t * t * (1.f / 6.f);
}

// ---- crop ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) crop_kernel(Jobs<smb_aug_case> cases, int C, int pd, int ph, int pw, float *__restrict__ data,
                                                   int8_t *__restrict__ seg, int sample0) {
    const smb_aug_case cs = cases.j[blockIdx.y];
    const int s = sample0 + (int)blockIdx.y;
    const int64_t vol = (int64_t)pd * ph * pw;
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < vol; v += (int64_t)gridDim.x * blockDim.x) {
        const int k = (int)(v % pw), j = (int)((v / pw) % ph), i = (int)(v / ((int64_t)pw * ph));
        const int z = cs.lz + i, y = cs.ly + j, x = cs.lx + k;
        const bool in = z >= 0 && z < cs.D && y >= 0 && y < cs.H && x >= 0 && x < cs.W;
        const int64_t off = (int64_t)z * cs.data_zs + (int64_t)y * cs.data_ys + x;
        for (int c = 0; c < C; ++c) data[((int64_t)s * C + c) * vol + v] = in ? cs.data[off + c * cs.data_cs] : 0.f;
        seg[(int64_t)s * vol + v] = in ? reinterpret_cast<const int8_t *>(cs.seg)[(int64_t)z * cs.seg_zs + (int64_t)y * cs.seg_ys + x]
                                       : (int8_t)0;
    }
}

// ---- cubic B-spline prefilter, one axis per launch ----------------------------------------------------------------------------
// Line t of a block lives in smem column t: s[q * 33 + t].  Axis 0 reads src (compact) and writes coef; axes 1 and 2 work in place
// on coef over the border rows the earlier axes wrote (edge padding and mirroring commute with filtering along another axis).
__device__ inline void filter_line(float *s, int t, int n, bool reflect_init) {
    const float z = kPole;
    for (int q = 0; q < n; ++q) s[q * 33 + t] *= 6.f;               // gain (1 - z)(1 - 1/z)
    float c0;
    if (!reflect_init) {                                              // causal init, whole-sample mirror boundary
        const float zn1 = powf(-z, (float)(n - 1)) * ((n - 1) & 1 ? -1.f : 1.f);
        float zi = z;
        c0 = s[t] + zn1 * s[(n - 1) * 33 + t];
        for (int q = 1; q < n - 1; ++q) {
            c0 += zi * (s[q * 33 + t] + zn1 * s[(n - 1 - q) * 33 + t]);
            zi *= z;
        }
        c0 /= 1.f - zn1 * zn1;
    } else {                                                          // causal init, half-sample boundary (scipy 'nearest')
        const float zn = powf(-z, (float)n) * (n & 1 ? -1.f : 1.f);
        float zi = z;
        float acc = s[t] + zn * s[(n - 1) * 33 + t];
        for (int q = 1; q < n; ++q) {
            acc += zi * (s[q * 33 + t] + zn * s[(n - 1 - q) * 33 + t]);
            zi *= z;
        }
        c0 = acc * z / (1.f - zn * zn) + s[t];
    }
    s[t] = c0;
    for (int q = 1; q < n; ++q) s[q * 33 + t] += z * s[(q - 1) * 33 + t];
    if (!reflect_init)
        s[(n - 1) * 33 + t] = (z * s[(n - 2) * 33 + t] + s[(n - 1) * 33 + t]) * z / (z * z - 1.f);
    else
        s[(n - 1) * 33 + t] *= z / (z - 1.f);
    for (int q = n - 2; q >= 0; --q) s[q * 33 + t] = z * (s[(q + 1) * 33 + t] - s[q * 33 + t]);
}

__global__ void __launch_bounds__(32) prefilter_kernel(Jobs<smb_aug_prefilter_job> jobs, int axis) {
    extern __shared__ float sm[];
    const smb_aug_prefilter_job jb = jobs.j[blockIdx.y];
    const int n[3] = {jb.n0, jb.n1, jb.n2};
    const int E1 = jb.n1 + 4, E2 = jb.n2 + 4;
    const int64_t es[3] = {(int64_t)E1 * E2, E2, 1};
    const int na = n[axis];
    if (na > kAugShortLine) return;                                  // prefilter_long_*_kernel's line
    // lines of this axis: over the border-extended range of the axes already filtered, the valid range of the others
    const int r0 = axis == 0 ? jb.n1 : jb.n0 + 4;                    // outer line index range
    const int r1 = axis == 2 ? E1 : jb.n2;                           // inner line index range (axis 0: n2, axis 1: n2, axis 2: E1)
    const int64_t lines = (int64_t)r0 * r1;
    const int64_t l0 = (int64_t)blockIdx.x * 32;
    if (l0 >= lines) return;
    const int t = threadIdx.x;
    const bool edge = jb.boundary == SMB_AUG_EDGE;
    const int pad = edge ? 12 : 0, L = na + 2 * pad;
    // coef offset of line l at position p (p in [-2, na + 2)); src offset (axis 0 only) of position p in [0, na)
    auto line_base = [&](int64_t l) -> int64_t {
        const int a = (int)(l / r1), b = (int)(l % r1);
        if (axis == 0) return (int64_t)(a + 2) * es[1] + (b + 2);
        if (axis == 1) return (int64_t)a * es[0] + (b + 2);
        return (int64_t)a * es[0] + (int64_t)b * es[1];
    };
    auto src_at = [&](int64_t l, int p) -> float {
        if (axis == 0) {
            const int a = (int)(l / r1), b = (int)(l % r1);
            return jb.src[((int64_t)p * jb.n1 + a) * jb.n2 + b];
        }
        return jb.coef[line_base(l) + (int64_t)(p + 2) * es[axis]];
    };
    const int nl = (int)((lines - l0) < 32 ? (lines - l0) : 32);
    if (axis == 2) {                                                  // contiguous lines: lanes along the line
        for (int u = 0; u < nl; ++u)
            for (int p = t; p < na; p += 32) sm[(p + pad) * 33 + u] = src_at(l0 + u, p);
    } else {                                                          // strided lines: lanes across lines
        if (t < nl)
            for (int p = 0; p < na; ++p) sm[(p + pad) * 33 + t] = src_at(l0 + t, p);
    }
    __syncwarp();
    if (t < nl) {
        if (edge)
            for (int q = 0; q < pad; ++q) {
                sm[q * 33 + t] = sm[pad * 33 + t];
                sm[(pad + na + q) * 33 + t] = sm[(pad + na - 1) * 33 + t];
            }
        filter_line(sm, t, L, edge);
    }
    __syncwarp();
    if (axis == 2) {
        for (int u = 0; u < nl; ++u) {
            const int64_t base = line_base(l0 + u);
            for (int p = t - 2; p < na + 2; p += 32) {
                const int q = edge ? p + pad : mirror_index(p, na);
                jb.coef[base + (p + 2)] = sm[q * 33 + u];
            }
        }
    } else if (t < nl) {
        const int64_t base = line_base(l0 + t);
        for (int p = -2; p < na + 2; ++p) {
            const int q = edge ? p + pad : mirror_index(p, na);
            jb.coef[base + (int64_t)(p + 2) * es[axis]] = sm[q * 33 + t];
        }
    }
}

// ---- cubic B-spline prefilter of lines longer than kAugShortLine, edge boundary -------------------------------------------------
// filter_line's steps on the padded line q = p + 12 in [0, n + 24) without staging it: the 12 pad samples per side are the first
// and last sample, so they are never stored.  The causal pass streams p = -2 .. n + 1 forward, writing c+ over the coefficient
// grid, and keeps the 10 pad values past it in registers; the anticausal pass streams the grid range backward.  The recursion
// state lives in a register, so shared memory does not grow with n.  The causal initial value is filter_line's 'nearest' sum:
// for n + 24 > 280 samples z^(n+24) is 0 in fp32, so the terms of the far end vanish and the sum stops once z^q underflows.
constexpr int kEdgePad = 12, kLongThreads = 128, kLongBatch = 8;

struct LongLine {                                                    // line l of the axis: (outer a, inner b) and its grid offset
    int a, b;
    int64_t base;
};

__device__ inline LongLine long_line(const smb_aug_prefilter_job &jb, int axis, int64_t l) {
    const int E1 = jb.n1 + 4, E2 = jb.n2 + 4;
    const int r1 = axis == 2 ? E1 : jb.n2;
    LongLine ln;
    ln.a = (int)(l / r1);
    ln.b = (int)(l % r1);
    ln.base = axis == 0 ? (int64_t)(ln.a + 2) * E2 + (ln.b + 2)
                        : (axis == 1 ? (int64_t)ln.a * E1 * E2 + (ln.b + 2) : (int64_t)ln.a * E1 * E2 + (int64_t)ln.b * E2);
    return ln;
}

__device__ inline int64_t long_lines(const smb_aug_prefilter_job &jb, int axis) {
    return axis == 0 ? (int64_t)jb.n1 * jb.n2 : (axis == 1 ? (int64_t)(jb.n0 + 4) * jb.n2 : (int64_t)(jb.n0 + 4) * (jb.n1 + 4));
}

// c+ at q = 9 (p = -3) from the gained edge value g0 and the first samples of the line, ld(p) for p in [0, n)
template <class Ld> __device__ inline float long_causal_start(float g0, int n, Ld &&ld) {
    const float z = kPole;
    float acc = g0, zi = z;
    for (int q = 1; q < kEdgePad; ++q) {
        acc += zi * g0;
        zi *= z;
    }
    for (int p = 0; p < n && zi != 0.f; ++p) {
        acc += zi * (6.f * ld(p));
        zi *= z;
    }
    float c = acc * z + g0;                                           // q = 0
    for (int q = 1; q < kEdgePad - 2; ++q) c = g0 + z * c;
    return c;
}

// axes 0 and 1: one line per thread, adjacent lanes on adjacent lines (coalesced); kLongBatch loads ahead of the recursion
__global__ void __launch_bounds__(kLongThreads) prefilter_long_strided_kernel(Jobs<smb_aug_prefilter_job> jobs, int axis) {
    const smb_aug_prefilter_job jb = jobs.j[blockIdx.y];
    const int n = axis == 0 ? jb.n0 : jb.n1;
    if (n <= kAugShortLine) return;                                   // prefilter_kernel's line
    const int64_t l = (int64_t)blockIdx.x * kLongThreads + threadIdx.x;
    if (l >= long_lines(jb, axis)) return;
    const LongLine ln = long_line(jb, axis, l);
    const int64_t step = axis == 0 ? (int64_t)(jb.n1 + 4) * (jb.n2 + 4) : jb.n2 + 4;
    float *cf = jb.coef + ln.base + 2 * step;                         // cf[p * step]: grid position p of the line
    auto ld = [&](int p) -> float {
        return axis == 0 ? jb.src[((int64_t)p * jb.n1 + ln.a) * jb.n2 + ln.b] : cf[p * step];
    };
    const float z = kPole, s0 = ld(0), sl = ld(n - 1), g0 = 6.f * s0, gl = 6.f * sl;
    float c = long_causal_start(g0, n, ld);
    for (int p0 = -2; p0 < n + 2; p0 += kLongBatch) {                 // causal: c+ over p = -2 .. n + 1
        float x[kLongBatch];
#pragma unroll
        for (int k = 0; k < kLongBatch; ++k) {
            const int p = p0 + k;
            x[k] = p < 0 ? s0 : (p < n ? ld(p) : sl);
        }
#pragma unroll
        for (int k = 0; k < kLongBatch; ++k) {
            const int p = p0 + k;
            if (p < n + 2) {
                c = 6.f * x[k] + z * c;
                cf[p * step] = c;
            }
        }
    }
    float tail[kEdgePad - 2];                                         // c+ at p = n + 2 .. n + 11
#pragma unroll
    for (int k = 0; k < kEdgePad - 2; ++k) tail[k] = c = gl + z * c;
    float d = tail[kEdgePad - 3] * (z / (z - 1.f));                   // anticausal
#pragma unroll
    for (int k = kEdgePad - 4; k >= 0; --k) d = z * (d - tail[k]);
    for (int p0 = n + 1; p0 >= -2; p0 -= kLongBatch) {
        float x[kLongBatch];
#pragma unroll
        for (int k = 0; k < kLongBatch; ++k) x[k] = p0 - k >= -2 ? cf[(p0 - k) * step] : 0.f;
#pragma unroll
        for (int k = 0; k < kLongBatch; ++k)
            if (p0 - k >= -2) {
                d = z * (d - x[k]);
                cf[(p0 - k) * step] = d;
            }
    }
}

// axis 2 (contiguous lines): a warp stages 32 lines x 32 samples transposed in shared memory, lane t runs the recursion of line t
__global__ void __launch_bounds__(kLongThreads) prefilter_long_rows_kernel(Jobs<smb_aug_prefilter_job> jobs) {
    __shared__ float tile[kLongThreads / 32][32][33];
    const smb_aug_prefilter_job jb = jobs.j[blockIdx.y];
    const int n = jb.n2, E2 = n + 4;
    if (n <= kAugShortLine) return;
    const int lane = threadIdx.x & 31;
    const int64_t lines = long_lines(jb, 2), l0 = ((int64_t)blockIdx.x * kLongThreads + threadIdx.x) - lane;
    if (l0 >= lines) return;                                          // the whole warp
    float(*T)[33] = tile[threadIdx.x >> 5];
    const bool live = l0 + lane < lines;
    const int64_t base = live ? long_line(jb, 2, l0 + lane).base : 0;
    const int nl = lines - l0 < 32 ? (int)(lines - l0) : 32;
    float *row = jb.coef + base;                                      // row[p + 2]: grid position p of this lane's line
    const float z = kPole;
    float c = 0.f, s0 = 0.f, sl = 0.f;
    if (live) {
        s0 = row[2];
        sl = row[n + 1];
        c = long_causal_start(6.f * s0, n, [&](int p) { return row[p + 2]; });
    }
    const float g0 = 6.f * s0, gl = 6.f * sl;
    for (int e0 = 0; e0 < E2; e0 += 32) {                            // causal, tiles of grid index e = p + 2
        for (int u = 0; u < nl; ++u) {
            const int64_t bu = __shfl_sync(0xffffffffu, base, u);
            const int e = e0 + lane;
            if (e >= 2 && e < n + 2) T[u][lane] = jb.coef[bu + e];
        }
        __syncwarp();
        if (live)
            for (int k = 0; k < 32 && e0 + k < E2; ++k) {
                const int p = e0 + k - 2;
                c = (p < 0 ? g0 : (p < n ? 6.f * T[lane][k] : gl)) + z * c;
                T[lane][k] = c;
            }
        __syncwarp();
        for (int u = 0; u < nl; ++u) {
            const int64_t bu = __shfl_sync(0xffffffffu, base, u);
            if (e0 + lane < E2) jb.coef[bu + e0 + lane] = T[u][lane];
        }
        __syncwarp();
    }
    float tail[kEdgePad - 2];
#pragma unroll
    for (int k = 0; k < kEdgePad - 2; ++k) tail[k] = c = gl + z * c;
    float d = tail[kEdgePad - 3] * (z / (z - 1.f));
#pragma unroll
    for (int k = kEdgePad - 4; k >= 0; --k) d = z * (d - tail[k]);
    for (int e0 = (E2 - 1) / 32 * 32; e0 >= 0; e0 -= 32) {            // anticausal, tiles backward
        for (int u = 0; u < nl; ++u) {
            const int64_t bu = __shfl_sync(0xffffffffu, base, u);
            if (e0 + lane < E2) T[u][lane] = jb.coef[bu + e0 + lane];
        }
        __syncwarp();
        if (live)
            for (int k = (E2 - 1 - e0 < 31 ? E2 - 1 - e0 : 31); k >= 0; --k) {
                d = z * (d - T[lane][k]);
                T[lane][k] = d;
            }
        __syncwarp();
        for (int u = 0; u < nl; ++u) {
            const int64_t bu = __shfl_sync(0xffffffffu, base, u);
            if (e0 + lane < E2) jb.coef[bu + e0 + lane] = T[u][lane];
        }
        __syncwarp();
    }
}

// ---- resample ---------------------------------------------------------------------------------------------------------------
__device__ inline void map_coord(const smb_aug_resample_job &jb, int i, int j, int k, double x[3]) {
    if (jb.map == SMB_AUG_ZOOM) {
        x[0] = ((double)i + 0.5) * jb.a00 - 0.5;
        x[1] = ((double)j + 0.5) * jb.a11 - 0.5;
        x[2] = ((double)k + 0.5) * jb.a22 - 0.5;
    } else {
        x[0] = jb.a00 * i + jb.a01 * j + jb.a02 * k + jb.a03;
        x[1] = jb.a10 * i + jb.a11 * j + jb.a12 * k + jb.a13;
        x[2] = jb.a20 * i + jb.a21 * j + jb.a22 * k + jb.a23;
    }
}

__global__ void __launch_bounds__(256) resample_kernel(Jobs<smb_aug_resample_job> jobs) {
    const smb_aug_resample_job jb = jobs.j[blockIdx.y];
    const int n[3] = {jb.n0, jb.n1, jb.n2};
    const int64_t vol = (int64_t)jb.m0 * jb.m1 * jb.m2;
    const bool zoom = jb.map == SMB_AUG_ZOOM;
    float lo = -INFINITY, hi = INFINITY;
    if (jb.clip) { lo = (float)jb.clip[2]; hi = (float)jb.clip[3]; }
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < vol; v += (int64_t)gridDim.x * blockDim.x) {
        const int k = (int)(v % jb.m2), j = (int)((v / jb.m2) % jb.m1), i = (int)(v / ((int64_t)jb.m2 * jb.m1));
        double x[3];
        map_coord(jb, i, j, k, x);
        bool inside = true;
        for (int d = 0; d < 3; ++d) {
            if (zoom) x[d] = x[d] < -1.0 ? -1.0 : (x[d] > n[d] - 0.5 ? n[d] - 0.5 : x[d]);   // a zoom by n/m stays inside; taps stay on the border
            else inside = inside && x[d] >= 0.0 && x[d] <= (double)(n[d] - 1);
        }
        if (jb.order == 0) {
            float r = 0.f;
            if (inside) {
                int ix[3];
                for (int d = 0; d < 3; ++d) {
                    int q = (int)floor(x[d] + 0.5);
                    ix[d] = q < 0 ? 0 : (q > n[d] - 1 ? n[d] - 1 : q);
                }
                r = reinterpret_cast<const float *>(jb.src)[((int64_t)ix[0] * n[1] + ix[1]) * n[2] + ix[2]];
            }
            reinterpret_cast<float *>(jb.dst)[v] = fminf(fmaxf(r, lo), hi);
        } else if (jb.order == 3) {
            float r = 0.f;
            if (inside) {
                const int E1 = n[1] + 4, E2 = n[2] + 4;
                int f[3];
                float w[3][4];
                for (int d = 0; d < 3; ++d) {
                    const double fl = floor(x[d]);
                    f[d] = (int)fl - 1 + 2;                              // first tap, on the border-extended grid
                    bspline3((float)(x[d] - fl), w[d]);
                }
                const float *cf = reinterpret_cast<const float *>(jb.src);
                for (int a = 0; a < 4; ++a) {
                    float ra = 0.f;
                    for (int b = 0; b < 4; ++b) {
                        const float *row = cf + ((int64_t)(f[0] + a) * E1 + (f[1] + b)) * E2 + f[2];
                        const float rb = w[2][0] * row[0] + w[2][1] * row[1] + w[2][2] * row[2] + w[2][3] * row[3];
                        ra += w[1][b] * rb;
                    }
                    r += w[0][a] * ra;
                }
                r = fminf(fmaxf(r, lo), hi);
            }
            reinterpret_cast<float *>(jb.dst)[v] = r;
        } else {                                                         // order 1, labels
            int8_t best = 0;
            if (inside) {
                const int8_t *sg = reinterpret_cast<const int8_t *>(jb.src);
                int f[3], g[3];
                float t[3];
                for (int d = 0; d < 3; ++d) {
                    const double fl = floor(x[d]);
                    f[d] = (int)fl;
                    g[d] = f[d] + 1 > n[d] - 1 ? n[d] - 1 : f[d] + 1;      // the tap past the last sample has weight 0
                    t[d] = (float)(x[d] - fl);
                }
                int8_t lab[8];
                float wt[8];
                for (int c = 0; c < 8; ++c) {
                    const int zz = c & 4 ? g[0] : f[0], yy = c & 2 ? g[1] : f[1], xx = c & 1 ? g[2] : f[2];
                    lab[c] = sg[((int64_t)zz * n[1] + yy) * n[2] + xx];
                    wt[c] = (c & 4 ? t[0] : 1.f - t[0]) * (c & 2 ? t[1] : 1.f - t[1]) * (c & 1 ? t[2] : 1.f - t[2]);
                }
                float bw = 0.5f;
                for (int c = 0; c < 8; ++c) {
                    bool seen = false;
                    for (int e = 0; e < c; ++e) seen = seen || lab[e] == lab[c];
                    if (seen) continue;
                    float ind = 0.f;
                    for (int e = c; e < 8; ++e) ind += lab[e] == lab[c] ? wt[e] : 0.f;
                    if (ind >= bw) { bw = ind; best = lab[c]; }
                }
            }
            reinterpret_cast<int8_t *>(jb.dst)[v] = best;
        }
    }
}

// ---- separable Gaussian, reflect boundary -------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) blur_kernel(Jobs<smb_aug_blur_job> jobs, int axis) {
    __shared__ float w[17];
    __shared__ int rad;
    const smb_aug_blur_job jb = jobs.j[blockIdx.y];
    if (threadIdx.x == 0) {                                          // scipy _gaussian_kernel1d, in double
        const double sd = (double)jb.sigma;
        const int r = (int)(4.0 * sd + 0.5);
        double sum = 0.0, p[17];
        for (int q = -r; q <= r; ++q) { p[q + r] = exp(-0.5 / (sd * sd) * (double)(q * q)); sum += p[q + r]; }
        for (int q = 0; q <= 2 * r; ++q) w[q] = (float)(p[q] / sum);
        rad = r;
    }
    __syncthreads();
    const int n[3] = {jb.n0, jb.n1, jb.n2};
    const int64_t vol = (int64_t)n[0] * n[1] * n[2];
    const int64_t st[3] = {(int64_t)n[1] * n[2], n[2], 1};
    const float *src = axis == 0 ? jb.x : (axis == 1 ? jb.tmp : jb.tmp + vol);
    float *dst = axis == 0 ? jb.tmp : (axis == 1 ? jb.tmp + vol : jb.x);
    const int r = rad, na = n[axis];
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < vol; v += (int64_t)gridDim.x * blockDim.x) {
        const int p = (int)((v / st[axis]) % na);
        const int64_t base = v - (int64_t)p * st[axis];
        float acc = 0.f;
        for (int q = -r; q <= r; ++q) acc += w[q + r] * src[base + (int64_t)reflect_index(p + q, na) * st[axis]];
        dst[v] = acc;
    }
}

// ---- statistics ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) stats_partial_kernel(Jobs<smb_aug_stats_job> jobs) {
    __shared__ double red[8][4];
    const smb_aug_stats_job jb = jobs.j[blockIdx.y];
    double s = 0.0, s2 = 0.0;
    float mn = INFINITY, mx = -INFINITY;
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < jb.n; v += (int64_t)gridDim.x * blockDim.x) {
        const float a = jb.x[v];
        s += a;
        s2 += (double)a * a;
        mn = fminf(mn, a);
        mx = fmaxf(mx, a);
    }
    for (int o = 16; o; o >>= 1) {
        s += __shfl_down_sync(0xffffffffu, s, o);
        s2 += __shfl_down_sync(0xffffffffu, s2, o);
        mn = fminf(mn, __shfl_down_sync(0xffffffffu, mn, o));
        mx = fmaxf(mx, __shfl_down_sync(0xffffffffu, mx, o));
    }
    const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { red[wid][0] = s; red[wid][1] = s2; red[wid][2] = mn; red[wid][3] = mx; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double a = 0.0, b = 0.0, c = INFINITY, d = -INFINITY;
        for (int q = 0; q < (int)(blockDim.x >> 5); ++q) {
            a += red[q][0]; b += red[q][1];
            c = red[q][2] < c ? red[q][2] : c;
            d = red[q][3] > d ? red[q][3] : d;
        }
        double *o = jb.scratch + 4 * blockIdx.x;
        o[0] = a; o[1] = b; o[2] = c; o[3] = d;
    }
}

__global__ void __launch_bounds__(32) stats_final_kernel(Jobs<smb_aug_stats_job> jobs, int nblk) {
    const smb_aug_stats_job jb = jobs.j[blockIdx.x];
    if (threadIdx.x != 0) return;
    double a = 0.0, b = 0.0, c = INFINITY, d = -INFINITY;
    for (int q = 0; q < nblk; ++q) {
        const double *p = jb.scratch + 4 * q;
        a += p[0]; b += p[1];
        c = p[2] < c ? p[2] : c;
        d = p[3] > d ? p[3] : d;
    }
    jb.stats[0] = a; jb.stats[1] = b; jb.stats[2] = c; jb.stats[3] = d;
}

// ---- pointwise chain ----------------------------------------------------------------------------------------------------------
struct Moments {
    double mean, sd, mn, mx;
};

__device__ inline Moments moments(const double *st, int64_t n) {
    Moments m;
    m.mean = st[0] / (double)n;
    const double var = st[1] / (double)n - m.mean * m.mean;
    m.sd = sqrt(var > 0.0 ? var : 0.0);
    m.mn = st[2];
    m.mx = st[3];
    return m;
}

__device__ inline void box_muller4(uint32_t c[4], double out[4]) {
    const double k = 2.3283064365386963e-10;                          // 2^-32
    for (int h = 0; h < 2; ++h) {
        const double u1 = ((double)c[2 * h] + 0.5) * k, u2 = ((double)c[2 * h + 1] + 0.5) * k;
        const double rr = sqrt(-2.0 * log(u1)), th = 6.283185307179586 * u2;
        out[2 * h] = rr * cos(th);
        out[2 * h + 1] = rr * sin(th);
    }
}

__global__ void __launch_bounds__(256) pointwise_kernel(Jobs<smb_aug_point_job> jobs) {
    const smb_aug_point_job jb = jobs.j[blockIdx.y];
    const int ops = jb.ops;
    Moments m = {0.0, 0.0, 0.0, 0.0};
    if (jb.stats) m = moments(jb.stats, jb.n);
    float ra = 1.f, rb = 0.f;                                         // RETAIN as x * ra + rb after subtracting the mean
    float rmean = 0.f;
    if (ops & SMB_AUG_OP_RETAIN) {
        Moments r = moments(jb.retain_ref, jb.n);
        const double mn_r = (ops & SMB_AUG_OP_UNINVERT) ? -r.mean : r.mean;
        rmean = (float)m.mean;
        ra = (float)(r.sd / (m.sd + 1e-8));
        rb = (float)mn_r;
        // statistics after the step (used only by a later linear step)
        m.mn = (m.mn - m.mean) * ra + mn_r;
        m.mx = (m.mx - m.mean) * ra + mn_r;
        m.sd *= ra;
        m.mean = mn_r;
    }
    if (ops & SMB_AUG_OP_UNINVERT) { const double t = m.mn; m.mn = -m.mx; m.mx = -t; m.mean = -m.mean; }
    if (ops & SMB_AUG_OP_BRIGHT) { m.mean *= jb.brightness; m.mn *= jb.brightness; m.mx *= jb.brightness; m.sd *= jb.brightness; }
    const float cmean = (float)m.mean, cmin = (float)m.mn, cmax = (float)m.mx;
    if (ops & SMB_AUG_OP_INVERT) { const double t = m.mn; m.mn = -m.mx; m.mx = -t; m.mean = -m.mean; }
    const float gmin = (float)m.mn, grng = (float)(m.mx - m.mn);
    const float gden = grng + 1e-7f;
    const uint32_t k0 = (uint32_t)(uint64_t)jb.seed, k1 = (uint32_t)((uint64_t)jb.seed >> 32);
    const int64_t quads = (jb.n + 3) / 4;
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < quads; q += (int64_t)gridDim.x * blockDim.x) {
        double nz[4] = {0.0, 0.0, 0.0, 0.0};
        if (ops & SMB_AUG_OP_NOISE) {
            uint32_t c[4] = {(uint32_t)q, (uint32_t)jb.step, (uint32_t)jb.sample, (uint32_t)jb.channel};
            philox4x32_10(c, k0, k1);
            box_muller4(c, nz);
        }
        for (int e = 0; e < 4; ++e) {
            const int64_t v = 4 * q + e;
            if (v >= jb.n) break;
            float x = jb.x[v];
            if (ops & SMB_AUG_OP_RETAIN) x = (x - rmean) * ra + rb;
            if (ops & SMB_AUG_OP_UNINVERT) x = -x;
            if (ops & SMB_AUG_OP_NOISE) x += (float)((double)jb.noise_std * nz[e]);
            if (ops & SMB_AUG_OP_BRIGHT) x *= jb.brightness;
            if (ops & SMB_AUG_OP_CONTRAST) x = fminf(fmaxf((x - cmean) * jb.contrast + cmean, cmin), cmax);
            if (ops & SMB_AUG_OP_INVERT) x = -x;
            if (ops & SMB_AUG_OP_GAMMA) {
                const float b = fmaxf((x - gmin) / gden, 0.f);
                x = powf(b, jb.gamma) * grng + gmin;
            }
            jb.x[v] = x;
        }
    }
}

// ---- emit -------------------------------------------------------------------------------------------------------------------
template <typename T> __device__ inline T to_out(float v);
template <> __device__ inline float to_out<float>(float v) { return v; }
template <> __device__ inline __half to_out<__half>(float v) { return __float2half_rn(v); }
template <> __device__ inline __nv_bfloat16 to_out<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

template <typename T>
__global__ void __launch_bounds__(256) emit_kernel(Jobs<smb_aug_emit_sample> smp, int C, int pd, int ph, int pw, int channels_last,
                                                   T *__restrict__ image, int64_t *__restrict__ label, int sample0) {
    const smb_aug_emit_sample e = smp.j[blockIdx.y];
    const int s = sample0 + (int)blockIdx.y;
    const int64_t vol = (int64_t)pd * ph * pw;
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < vol; v += (int64_t)gridDim.x * blockDim.x) {
        int k = (int)(v % pw), j = (int)((v / pw) % ph), i = (int)(v / ((int64_t)pw * ph));
        if (e.flip & 1) i = pd - 1 - i;
        if (e.flip & 2) j = ph - 1 - j;
        if (e.flip & 4) k = pw - 1 - k;
        const int64_t src = ((int64_t)i * ph + j) * pw + k;
        for (int c = 0; c < C; ++c) {
            const int64_t o = channels_last ? ((int64_t)s * vol + v) * C + c : ((int64_t)s * C + c) * vol + v;
            image[o] = to_out<T>(e.data[c * vol + src]);
        }
        const int8_t l = reinterpret_cast<const int8_t *>(e.seg)[src];
        label[(int64_t)s * vol + v] = l == -1 ? 0 : (int64_t)l;
    }
}

unsigned grid_for(int64_t work, int per_block, int jobs) {
    int64_t b = (work + per_block - 1) / per_block;
    const int64_t cap = (132 * 16 + jobs - 1) / jobs;                  // about 16 blocks per SM over all jobs of a launch
    if (b > cap) b = cap;
    return (unsigned)(b < 1 ? 1 : b);
}

template <class T, class F> cudaError_t for_chunks(const T *jobs, int n, F &&launch) {
    for (int base = 0; base < n; base += kAugMaxJobs) {
        Jobs<T> js;
        js.n = n - base < kAugMaxJobs ? n - base : kAugMaxJobs;
        for (int q = 0; q < js.n; ++q) js.j[q] = jobs[base + q];
        for (int q = js.n; q < kAugMaxJobs; ++q) js.j[q] = jobs[base];
        cudaError_t e = launch(js, base);
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

}  // namespace

cudaError_t aug_crop_launch(const smb_aug_crop_args &a, cudaStream_t st) {
    const int64_t vol = (int64_t)a.pd * a.ph * a.pw;
    return for_chunks(a.cases, a.batch, [&](const Jobs<smb_aug_case> &js, int base) {
        crop_kernel<<<dim3(grid_for(vol, 256, js.n), js.n), 256, 0, st>>>(js, a.channels, a.pd, a.ph, a.pw, a.data,
                                                                         reinterpret_cast<int8_t *>(a.seg), base);
        count_launch();
        return cudaGetLastError();
    });
}

cudaError_t aug_prefilter_launch(const smb_aug_prefilter_job *jobs, int n, cudaStream_t st) {
    // per axis, each job's lines go to the staged kernel (n <= kAugShortLine) or to the streaming one (longer, edge boundary)
    return for_chunks(jobs, n, [&](const Jobs<smb_aug_prefilter_job> &js, int) {
        for (int axis = 0; axis < 3; ++axis) {
            int maxn = 0;
            int64_t short_lines = 0, long_lines = 0;
            for (int q = 0; q < js.n; ++q) {
                const smb_aug_prefilter_job &j = js.j[q];
                const int na = axis == 0 ? j.n0 : (axis == 1 ? j.n1 : j.n2);
                const int64_t l = axis == 0 ? (int64_t)j.n1 * j.n2 : (int64_t)(j.n0 + 4) * (axis == 1 ? j.n2 : j.n1 + 4);
                if (na <= kAugShortLine) {
                    maxn = na > maxn ? na : maxn;
                    short_lines = l > short_lines ? l : short_lines;
                } else {
                    long_lines = l > long_lines ? l : long_lines;
                }
            }
            if (short_lines) {
                const size_t smem = sizeof(float) * 33 * (size_t)(maxn + 24);
                prefilter_kernel<<<dim3((unsigned)((short_lines + 31) / 32), js.n), 32, smem, st>>>(js, axis);
                count_launch();
                cudaError_t e = cudaGetLastError();
                if (e != cudaSuccess) return e;
            }
            if (long_lines) {
                const dim3 grid((unsigned)((long_lines + kLongThreads - 1) / kLongThreads), js.n);
                if (axis == 2)
                    prefilter_long_rows_kernel<<<grid, kLongThreads, 0, st>>>(js);
                else
                    prefilter_long_strided_kernel<<<grid, kLongThreads, 0, st>>>(js, axis);
                count_launch();
                cudaError_t e = cudaGetLastError();
                if (e != cudaSuccess) return e;
            }
        }
        return cudaSuccess;
    });
}

cudaError_t aug_resample_launch(const smb_aug_resample_job *jobs, int n, cudaStream_t st) {
    return for_chunks(jobs, n, [&](const Jobs<smb_aug_resample_job> &js, int) {
        int64_t vol = 0;
        for (int q = 0; q < js.n; ++q) {
            const int64_t v = (int64_t)js.j[q].m0 * js.j[q].m1 * js.j[q].m2;
            vol = v > vol ? v : vol;
        }
        resample_kernel<<<dim3(grid_for(vol, 256, js.n), js.n), 256, 0, st>>>(js);
        count_launch();
        return cudaGetLastError();
    });
}

cudaError_t aug_blur_launch(const smb_aug_blur_job *jobs, int n, cudaStream_t st) {
    return for_chunks(jobs, n, [&](const Jobs<smb_aug_blur_job> &js, int) {
        int64_t vol = 0;
        for (int q = 0; q < js.n; ++q) {
            const int64_t v = (int64_t)js.j[q].n0 * js.j[q].n1 * js.j[q].n2;
            vol = v > vol ? v : vol;
        }
        for (int axis = 0; axis < 3; ++axis) {
            blur_kernel<<<dim3(grid_for(vol, 256, js.n), js.n), 256, 0, st>>>(js, axis);
            count_launch();
            cudaError_t e = cudaGetLastError();
            if (e != cudaSuccess) return e;
        }
        return cudaSuccess;
    });
}

cudaError_t aug_stats_launch(const smb_aug_stats_job *jobs, int n, cudaStream_t st) {
    return for_chunks(jobs, n, [&](const Jobs<smb_aug_stats_job> &js, int) {
        stats_partial_kernel<<<dim3(kAugStatsBlocks, js.n), 256, 0, st>>>(js);
        count_launch();
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
        stats_final_kernel<<<js.n, 32, 0, st>>>(js, kAugStatsBlocks);
        count_launch();
        return cudaGetLastError();
    });
}

cudaError_t aug_pointwise_launch(const smb_aug_point_job *jobs, int n, cudaStream_t st) {
    return for_chunks(jobs, n, [&](const Jobs<smb_aug_point_job> &js, int) {
        int64_t quads = 0;
        for (int q = 0; q < js.n; ++q) quads = (js.j[q].n + 3) / 4 > quads ? (js.j[q].n + 3) / 4 : quads;
        pointwise_kernel<<<dim3(grid_for(quads, 256, js.n), js.n), 256, 0, st>>>(js);
        count_launch();
        return cudaGetLastError();
    });
}

cudaError_t aug_emit_launch(const smb_aug_emit_args &a, cudaStream_t st) {
    const int64_t vol = (int64_t)a.pd * a.ph * a.pw;
    return for_chunks(a.samples, a.batch, [&](const Jobs<smb_aug_emit_sample> &js, int base) {
        const dim3 grid(grid_for(vol, 256, js.n), js.n);
        if (a.out_dtype == SMB_F32)
            emit_kernel<float><<<grid, 256, 0, st>>>(js, a.channels, a.pd, a.ph, a.pw, a.channels_last, reinterpret_cast<float *>(a.image),
                                                      a.label, base);
        else if (a.out_dtype == SMB_F16)
            emit_kernel<__half><<<grid, 256, 0, st>>>(js, a.channels, a.pd, a.ph, a.pw, a.channels_last, reinterpret_cast<__half *>(a.image),
                                                       a.label, base);
        else
            emit_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>(js, a.channels, a.pd, a.ph, a.pw, a.channels_last,
                                                              reinterpret_cast<__nv_bfloat16 *>(a.image), a.label, base);
        count_launch();
        return cudaGetLastError();
    });
}

}  // namespace smb
