// Dice and Hausdorff-percentile evaluation (medpy.metric.binary.dc / hd95 / hd, connectivity 1, as the reference's
// 5_compute_metrics.py and validation_step use them) on region bitmasks.
//
// The distance transform is exact and separable: a 1-D nearest-feature sweep along axis 0, then two lower-envelope passes
// (Meijster et al., 2000) along axes 2 and 1 in fp64 with the voxel spacing.  Each voxel carries the linear index of its
// nearest feature so the last pass can form the distance from the offsets the way scipy does.  A lower-envelope pass runs one
// thread per line; the line and its envelope stack share one 8-byte slot per position in shared memory (the stack never
// grows past the position being read, and the answers overwrite dead stack slots).
//
// The EDT runs over a list of jobs, each a box of one sample's border maps: smb_metric_edt makes one whole-volume job per
// (sample, region, direction); smb_metric_class_edt reads a job table from device memory, one box per (sample, class,
// direction), and also writes each axis-1 line's sum and maximum of its distances so that the means reduce in a fixed order.
//
// What bounds them: the count / border pass and the sweeps stream bytes and int32 features through HBM; the envelope passes
// are latency-bound sequential loops over shared memory (one line per thread, a few warps per SM for lack of shared memory).
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>

#include "metrics_internal.h"

namespace smb {
void count_launch();

namespace {

constexpr int kEnvSmem = 200 * 1024;                                   // shared-memory budget of an envelope block

template <typename T> __device__ inline float as_float(T v);
template <> __device__ inline float as_float<float>(float v) { return v; }
template <> __device__ inline float as_float<__half>(__half v) { return __half2float(v); }
template <> __device__ inline float as_float<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

// ---- region bits ------------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) label_bits_kernel(smb_metric_bits_args a) {
    const int b = blockIdx.y;
    const T *src = reinterpret_cast<const T *>(a.src) + (int64_t)b * a.sample_stride;
    uint8_t *bits = reinterpret_cast<uint8_t *>(a.bits) + (int64_t)b * a.voxels;
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < a.voxels; v += (int64_t)gridDim.x * blockDim.x) {
        const int64_t l = (int64_t)src[v * a.voxel_stride];
        bits[v] = (l >= 0 && l < 256) ? a.lut[l] : (uint8_t)0;
    }
}

template <typename T>
__global__ void __launch_bounds__(256) logit_bits_kernel(smb_metric_bits_args a) {
    const int b = blockIdx.y;
    const T *src = reinterpret_cast<const T *>(a.src) + (int64_t)b * a.sample_stride;
    uint8_t *bits = reinterpret_cast<uint8_t *>(a.bits) + (int64_t)b * a.voxels;
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < a.voxels; v += (int64_t)gridDim.x * blockDim.x) {
        const T *p = src + v * a.voxel_stride;
        float best = as_float<T>(p[0]);
        int arg = 0;
        for (int c = 1; c < a.classes && best == best; ++c) {           // the first maximum; a NaN is the maximum
            const float x = as_float<T>(p[(int64_t)c * a.class_stride]);
            if (x > best || x != x) { best = x; arg = c; }
        }
        bits[v] = arg < 256 ? a.lut[arg] : (uint8_t)0;
    }
}

// ---- counts and borders -----------------------------------------------------------------------------------------------------
__device__ inline uint8_t interior(const uint8_t *m, int z, int y, int x, int d, int h, int w, int64_t v) {
    uint8_t in = m[v];
    in &= z > 0 ? m[v - (int64_t)h * w] : 0;
    in &= z < d - 1 ? m[v + (int64_t)h * w] : 0;
    in &= y > 0 ? m[v - w] : 0;
    in &= y < h - 1 ? m[v + w] : 0;
    in &= x > 0 ? m[v - 1] : 0;
    in &= x < w - 1 ? m[v + 1] : 0;
    return in;
}

__global__ void __launch_bounds__(256) count_kernel(smb_metric_count_args a) {
    const int b = blockIdx.y;
    const int64_t n = (int64_t)a.d * a.h * a.w;
    const uint8_t *P = reinterpret_cast<const uint8_t *>(a.pred) + (int64_t)b * n;
    const uint8_t *G = reinterpret_cast<const uint8_t *>(a.target) + (int64_t)b * n;
    uint8_t *PB = reinterpret_cast<uint8_t *>(a.pred_border) + (int64_t)b * n;
    uint8_t *GB = reinterpret_cast<uint8_t *>(a.target_border) + (int64_t)b * n;
    unsigned cnt[5][SMB_METRIC_MAX_REGIONS] = {};
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < n; v += (int64_t)gridDim.x * blockDim.x) {
        const int x = (int)(v % a.w), y = (int)((v / a.w) % a.h), z = (int)(v / ((int64_t)a.w * a.h));
        const uint8_t p = P[v], g = G[v];
        const uint8_t pb = p & ~interior(P, z, y, x, a.d, a.h, a.w, v), gb = g & ~interior(G, z, y, x, a.d, a.h, a.w, v);
        PB[v] = pb;
        GB[v] = gb;
        const uint8_t m[5] = {p, g, (uint8_t)(p & g), pb, gb};
#pragma unroll
        for (int k = 0; k < 5; ++k)
#pragma unroll
            for (int r = 0; r < SMB_METRIC_MAX_REGIONS; ++r) cnt[k][r] += (m[k] >> r) & 1u;
    }
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int k = 0; k < 5; ++k)
#pragma unroll
        for (int r = 0; r < SMB_METRIC_MAX_REGIONS; ++r) {
            unsigned c = cnt[k][r];
            for (int o = 16; o; o >>= 1) c += __shfl_down_sync(0xffffffffu, c, o);
            if (lane == 0 && r < a.regions && c)
                atomicAdd(reinterpret_cast<unsigned long long *>(a.counts) + ((int64_t)b * a.regions + r) * SMB_METRIC_NCOUNTS + k,
                          (unsigned long long)c);
        }
}

// ---- exact EDT ----------------------------------------------------------------------------------------------------------------
// A job is a box of one sample's border maps.  Feature indices are linear indices inside the box; the maps are read through the
// box origin and their row / slice strides.  smb_metric_edt's jobs are whole volumes, smb_metric_class_edt's come from a table.
struct Job {
    const uint8_t *src, *tgt;
    int32_t *feat;
    double *pool;
    unsigned long long *fill;
    double2 *lines;
    int64_t ys, zs;                                                    // map strides
    int bd, bh, bw;
    uint8_t smask, sval, tmask, tval;
    __device__ bool is_src(int64_t o) const { return (src[o] & smask) == sval; }
    __device__ bool is_tgt(int64_t o) const { return (tgt[o] & tmask) == tval; }
};

// smb_metric_edt: job j = (b * regions + r) * 2 + dir; dir 0: source P's border, target G's border; dir 1 the other way round
struct RegionJobs {
    static constexpr bool kLines = false;                              // no per-line sums
    smb_metric_edt_args a;
    __device__ Job operator()(int j) const {
        Job o;
        const int64_t n = (int64_t)a.d * a.h * a.w;
        const int pair = j >> 1, dir = j & 1, b = pair / a.regions, r = pair % a.regions;
        const uint8_t *pb = reinterpret_cast<const uint8_t *>(a.pred_border) + (int64_t)b * n;
        const uint8_t *gb = reinterpret_cast<const uint8_t *>(a.target_border) + (int64_t)b * n;
        o.src = dir ? gb : pb;
        o.tgt = dir ? pb : gb;
        o.feat = a.feat + (int64_t)j * n;
        o.pool = a.pool + (int64_t)pair * a.pool_cap;
        o.fill = reinterpret_cast<unsigned long long *>(a.counts) + (int64_t)pair * SMB_METRIC_NCOUNTS + 5;
        o.lines = nullptr;
        o.ys = a.w;
        o.zs = (int64_t)a.h * a.w;
        o.bd = a.d;
        o.bh = a.h;
        o.bw = a.w;
        o.smask = o.sval = o.tmask = o.tval = (uint8_t)(1u << r);
        return o;
    }
};

// smb_metric_class_edt: the job table in device memory
struct TableJobs {
    static constexpr bool kLines = true;
    smb_metric_class_edt_args a;
    __device__ Job operator()(int j) const {
        const smb_metric_edt_job &t = a.jobs[j];
        Job o;
        o.src = reinterpret_cast<const uint8_t *>(t.src);
        o.tgt = reinterpret_cast<const uint8_t *>(t.tgt);
        o.feat = t.feat;
        o.pool = t.pool;
        o.fill = reinterpret_cast<unsigned long long *>(t.fill);
        o.lines = reinterpret_cast<double2 *>(t.lines);
        o.ys = a.row_stride;
        o.zs = a.slice_stride;
        o.bd = t.bd;
        o.bh = t.bh;
        o.bw = t.bw;
        o.smask = (uint8_t)t.src_mask;
        o.sval = (uint8_t)t.src_val;
        o.tmask = (uint8_t)t.tgt_mask;
        o.tval = (uint8_t)t.tgt_val;
        return o;
    }
};

// axis 0: feat = index of the nearest target voxel in the voxel's column (ties: the lower z), -1 if none
template <class Jobs>
__global__ void __launch_bounds__(256) edt_axis0_kernel(Jobs jobs) {
    const Job jb = jobs(blockIdx.y);
    const int64_t hw = (int64_t)jb.bh * jb.bw;
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < hw; c += (int64_t)gridDim.x * blockDim.x) {
        const int64_t m = (c / jb.bw) * jb.ys + c % jb.bw;           // the column in the maps
        int last = -1;
        for (int z = 0; z < jb.bd; ++z) {
            if (jb.is_tgt(z * jb.zs + m)) last = z;
            jb.feat[z * hw + c] = last;
        }
        int next = -1;
        for (int z = jb.bd - 1; z >= 0; --z) {
            if (jb.is_tgt(z * jb.zs + m)) next = z;
            const int prev = jb.feat[z * hw + c];
            const int f = (next >= 0 && (prev < 0 || next - z < z - prev)) ? next : prev;
            jb.feat[z * hw + c] = f < 0 ? -1 : (int32_t)(f * hw + c);
        }
    }
}

// Lower envelope of the parabolas g(i) + ((u - i) h)^2 over one line of n positions.  slot(p) is the 8-byte shared slot of
// position p: on entry .x holds the feature index at p (-1: none); on exit .x holds the feature of the nearest parabola at p.
// The stack entry q lives in slot q (.x its feature, .y its position | its first position << 16); q <= the position read.
template <class Cost>
__device__ inline void envelope(int2 *s, int stride, int n, double h2, Cost cost) {
    int q = -1;
    double gq = 0.0;                                                   // g of the stack top
    for (int u = 0; u < n; ++u) {
        const int fu = s[u * stride].x;
        if (fu < 0) continue;
        const double gu = cost(fu);
        double sep = 0.0;
        int tq = 0;
        while (q >= 0) {
            const int2 e = s[q * stride];
            const int sq = e.y & 0xffff;
            tq = e.y >> 16;
            const double dq = (double)(tq - sq), du = (double)(tq - u);
            if (gq + dq * dq * h2 <= gu + du * du * h2) {
                sep = (gu - gq + h2 * ((double)u * u - (double)sq * sq)) / (2.0 * h2 * (double)(u - sq));
                break;
            }
            if (--q >= 0) gq = cost(s[q * stride].x);
        }
        if (q < 0) {
            q = 0;
            s[0] = make_int2(fu, u);
            gq = gu;
        } else {
            // the top wins at tq, so u's segment starts after it even where rounding puts the intersection a hair below tq
            const double w = fmax(floor(sep) + 1.0, (double)(tq + 1));
            if (w < (double)n) {
                ++q;
                s[q * stride] = make_int2(fu, u | ((int)w << 16));
                gq = gu;
            }
        }
    }
    for (int u = n - 1; u >= 0; --u) {
        if (q < 0) { s[u * stride].x = -1; continue; }
        const int2 e = s[q * stride];
        s[u * stride].x = e.x;                                         // u >= q: slot u is dead or is the entry just read
        if (u == (e.y >> 16)) --q;
    }
}

__device__ inline double sq(double v) { return __dmul_rn(v, v); }

// axis 2 (rows, contiguous): lanes stage rows cooperatively, each thread runs the envelope of one row
template <class Jobs>
__global__ void __launch_bounds__(128) edt_axis2_kernel(Jobs jobs, double s0, double s2) {
    extern __shared__ int2 env[];
    const Job jb = jobs(blockIdx.y);
    const int T = blockDim.x, stride = T + 1, n = jb.bw;
    const int64_t lines = (int64_t)jb.bd * jb.bh, l0 = (int64_t)blockIdx.x * T;
    if (l0 >= lines) return;
    const int nl = (int)(lines - l0 < T ? lines - l0 : T);
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5, nwarps = T >> 5;
    for (int u = warp; u < nl; u += nwarps)
        for (int p = lane; p < n; p += 32) env[p * stride + u].x = jb.feat[(l0 + u) * n + p];
    __syncthreads();
    if (t < nl) {
        const int z = (int)((l0 + t) / jb.bh);
        const int64_t hw = (int64_t)jb.bh * jb.bw;
        envelope(env + t, stride, n, s2 * s2, [=](int f) { return sq((double)((int)(f / hw) - z) * s0); });
    }
    __syncthreads();
    for (int u = warp; u < nl; u += nwarps)
        for (int p = lane; p < n; p += 32) jb.feat[(l0 + u) * n + p] = env[p * stride + u].x;
}

// axis 1 (columns of a z slice), the last pass: each thread stages and walks one column; distances at the source voxels go to
// the job's pool, and the column's sum (in order of y) and maximum of them to its line slot
template <class Jobs>
__global__ void __launch_bounds__(128) edt_axis1_kernel(Jobs jobs, double s0, double s1, double s2) {
    extern __shared__ int2 env[];
    const Job jb = jobs(blockIdx.y);
    const int T = blockDim.x, stride = T + 1, n = jb.bh, t = threadIdx.x;
    const int64_t lines = (int64_t)jb.bd * jb.bw, l = (int64_t)blockIdx.x * T + t;
    if (l >= lines) return;
    const int z = (int)(l / jb.bw), x = (int)(l % jb.bw);
    const int64_t hw = (int64_t)jb.bh * jb.bw, base = z * hw + x, mbase = z * jb.zs + x;
    int2 *s = env + t;
    for (int p = 0; p < n; ++p) s[p * stride].x = jb.feat[base + (int64_t)p * jb.bw];
    const int bw = jb.bw;
    envelope(s, stride, n, s1 * s1, [=](int f) {
        return __dadd_rn(sq((double)((int)(f / hw) - z) * s0), sq((double)((int)(f % bw) - x) * s2));
    });
    double sum = 0.0, mx = 0.0;
    for (int p = 0; p < n; ++p) {
        if (!jb.is_src(mbase + (int64_t)p * jb.ys)) continue;
        const int f = s[p * stride].x;
        if (f < 0) continue;
        const int fz = (int)(f / hw), fy = (int)((f / jb.bw) % jb.bh), fx = (int)(f % jb.bw);
        const double d0 = (double)(fz - z) * s0, d1 = (double)(fy - p) * s1, d2 = (double)(fx - x) * s2;
        const double dist = sqrt(__dadd_rn(__dadd_rn(sq(d0), sq(d1)), sq(d2)));
        jb.pool[atomicAdd(jb.fill, 1ull)] = dist;
        if (Jobs::kLines) {
            sum = __dadd_rn(sum, dist);
            mx = fmax(mx, dist);
        }
    }
    if (Jobs::kLines && jb.lines) jb.lines[l] = make_double2(sum, mx);
}

// ---- percentile ---------------------------------------------------------------------------------------------------------------
// One block per (b, r): a radix select, 8 bits per pass from the top, over the bit patterns of the non-negative distances
// (their order is the order of the values) finds the value of rank kp; rank kp + 1 is that value again or the smallest above it.
constexpr int kSelThreads = 512;

__device__ inline unsigned long long block_min(unsigned long long v, unsigned long long *red) {
    for (int o = 16; o; o >>= 1) {
        const unsigned long long w = __shfl_down_sync(0xffffffffu, v, o);
        v = w < v ? w : v;
    }
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int q = 1; q < (int)(blockDim.x >> 5); ++q) v = red[q] < v ? red[q] : v;
        red[0] = v;
    }
    __syncthreads();
    return red[0];
}

struct SelectSmem {
    unsigned hist[256];
    unsigned long long red[kSelThreads / 32];
    unsigned long long pre, k, eq;
};

// numpy.percentile(key[0..n), 100 * frac) with method 'linear' (n > 0), for thread 0; every thread of the block must call it
__device__ double select_value(const unsigned long long *key, int64_t n, double frac, SelectSmem &sm) {
    // numpy 'linear': virtual index (n - 1) q; at or past the last index both neighbours are the maximum
    const double vi = (double)(n - 1) * frac;
    int64_t kp;
    double gamma = 0.0;
    if (vi >= (double)(n - 1)) {
        kp = n - 1;
    } else {
        const double fl = floor(vi);
        kp = (int64_t)fl;
        gamma = vi - fl;
    }
    if (threadIdx.x == 0) { sm.pre = 0; sm.k = (unsigned long long)kp; }
    unsigned long long mask = 0;
    for (int shift = 56; shift >= 0; shift -= 8) {
        for (int i = threadIdx.x; i < 256; i += blockDim.x) sm.hist[i] = 0;
        __syncthreads();
        const unsigned long long pre = sm.pre;
        for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
            const unsigned long long k = key[i];
            if ((k & mask) == pre) atomicAdd(&sm.hist[(k >> shift) & 255], 1u);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned long long k = sm.k;
            int d = 0;
            while (sm.hist[d] <= k) k -= sm.hist[d++];
            sm.k = k;
            sm.pre = pre | ((unsigned long long)d << shift);
            sm.eq = sm.hist[d];
        }
        mask |= 255ull << shift;
        __syncthreads();
    }
    const unsigned long long va = sm.pre;
    unsigned long long vb = va;
    if (kp + 1 < n && gamma != 0.0 && sm.k + 1 >= sm.eq) {              // rank kp + 1 lies above the run of va
        unsigned long long m = ~0ull;
        for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
            const unsigned long long k = key[i];
            if (k > va && k < m) m = k;
        }
        vb = block_min(m, sm.red);
    }
    double x, y;
    memcpy(&x, &va, 8);
    memcpy(&y, &vb, 8);
    // numpy's _lerp, both branches, without contraction
    const double diff = __dsub_rn(y, x);
    return gamma >= 0.5 ? __dsub_rn(y, __dmul_rn(diff, __dsub_rn(1.0, gamma))) : __dadd_rn(x, __dmul_rn(diff, gamma));
}

__global__ void __launch_bounds__(kSelThreads) select_kernel(smb_metric_select_args a) {
    __shared__ SelectSmem sm;
    const int pr = blockIdx.x;
    const int64_t *c = a.counts + (int64_t)pr * SMB_METRIC_NCOUNTS;
    if (c[0] == 0 || c[1] == 0) {
        if (threadIdx.x == 0) a.out[pr] = NAN;
        return;
    }
    const unsigned long long *key = reinterpret_cast<const unsigned long long *>(a.pool + (int64_t)pr * a.pool_cap);
    const double v = select_value(key, c[5], a.frac, sm);
    if (threadIdx.x == 0) a.out[pr] = v;
}

// sum and maximum of (sum, max) line pairs in a fixed order: each thread walks its stride sequentially, then a fixed tree
__device__ double2 reduce_lines(const double2 *lines, int n, double2 *red) {
    double sum = 0.0, mx = 0.0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const double2 v = lines[i];
        sum = __dadd_rn(sum, v.x);
        mx = fmax(mx, v.y);
    }
    red[threadIdx.x] = make_double2(sum, mx);
    __syncthreads();
    for (int o = blockDim.x >> 1; o; o >>= 1) {
        if ((int)threadIdx.x < o) {
            const double2 u = red[threadIdx.x], v = red[threadIdx.x + o];
            red[threadIdx.x] = make_double2(__dadd_rn(u.x, v.x), fmax(u.y, v.y));
        }
        __syncthreads();
    }
    const double2 r = red[0];
    __syncthreads();
    return r;
}

// one block per pool of smb_metric_class_reduce
__global__ void __launch_bounds__(kSelThreads) class_reduce_kernel(smb_metric_class_reduce_args a) {
    __shared__ SelectSmem sm;
    __shared__ double2 red[kSelThreads];
    const smb_metric_pool pl = a.pools[blockIdx.x];
    const double2 *lines = reinterpret_cast<const double2 *>(pl.lines);
    const double2 r0 = reduce_lines(lines, pl.lines0, red), r1 = reduce_lines(lines + pl.lines0, pl.lines1, red);
    const double q = select_value(reinterpret_cast<const unsigned long long *>(pl.dist), pl.n0 + pl.n1, a.frac, sm);
    if (threadIdx.x == 0) {
        const double asd0 = r0.x / (double)pl.n0, asd1 = r1.x / (double)pl.n1;
        double *o = a.out + (int64_t)blockIdx.x * 4;
        o[0] = fmax(r0.y, r1.y);
        o[1] = q;
        o[2] = asd0;
        o[3] = __dadd_rn(asd0, asd1) / 2.0;
    }
}

// ---- per-class counts, borders and boxes ----------------------------------------------------------------------------------------
// true when the voxel has class c (nonzero) and a 6-neighbour of another class or outside the volume
__device__ inline bool class_border(const uint8_t *m, uint8_t c, int z, int y, int x, int d, int h, int w, int64_t v) {
    const int64_t hw = (int64_t)h * w;
    bool in = true;
    in &= z > 0 && m[v - hw] == c;
    in &= z < d - 1 && m[v + hw] == c;
    in &= y > 0 && m[v - w] == c;
    in &= y < h - 1 && m[v + w] == c;
    in &= x > 0 && m[v - 1] == c;
    in &= x < w - 1 && m[v + 1] == c;
    return c != 0 && !in;
}

// adds 1 to cnt[c - 1] for every lane whose c is nonzero: one shared atomic per distinct value in the warp
__device__ inline void warp_count(unsigned *cnt, unsigned c) {
    const unsigned peers = __match_any_sync(0xffffffffu, c);
    if (c != 0 && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&cnt[c - 1], (unsigned)__popc(peers));
}

__device__ inline void box_add(unsigned (*cnt)[SMB_METRIC_MAX_CLASSES], unsigned c, int z, int y, int x, int d, int h, int w) {
    const int k = (int)c - 1;
    atomicMax(&cnt[5][k], (unsigned)(d - z));
    atomicMax(&cnt[6][k], (unsigned)(h - y));
    atomicMax(&cnt[7][k], (unsigned)(w - x));
    atomicMax(&cnt[8][k], (unsigned)(z + 1));
    atomicMax(&cnt[9][k], (unsigned)(y + 1));
    atomicMax(&cnt[10][k], (unsigned)(x + 1));
}

// grid (blocks, batch); each block keeps its counters in shared memory and adds them to the record once
__global__ void __launch_bounds__(256) class_count_kernel(smb_metric_class_count_args a) {
    __shared__ unsigned cnt[SMB_METRIC_CLASS_NREC][SMB_METRIC_MAX_CLASSES];
    const int b = blockIdx.y, K = a.classes;
    const int64_t n = (int64_t)a.d * a.h * a.w;
    const uint8_t *P = reinterpret_cast<const uint8_t *>(a.pred) + (int64_t)b * n;
    const uint8_t *G = reinterpret_cast<const uint8_t *>(a.target) + (int64_t)b * n;
    uint8_t *PB = reinterpret_cast<uint8_t *>(a.pred_border) + (int64_t)b * n;
    uint8_t *GB = reinterpret_cast<uint8_t *>(a.target_border) + (int64_t)b * n;
    for (int i = threadIdx.x; i < SMB_METRIC_CLASS_NREC * SMB_METRIC_MAX_CLASSES; i += blockDim.x) (&cnt[0][0])[i] = 0;
    __syncthreads();
    // the loop bound is uniform across the warp, so the warp is converged at every __match_any_sync
    for (int64_t v0 = (int64_t)blockIdx.x * blockDim.x; v0 < n; v0 += (int64_t)gridDim.x * blockDim.x) {
        const int64_t v = v0 + threadIdx.x;
        unsigned p = 0, g = 0, pb = 0, gb = 0;
        int x = 0, y = 0, z = 0;
        if (v < n) {
            x = (int)(v % a.w);
            y = (int)((v / a.w) % a.h);
            z = (int)(v / ((int64_t)a.w * a.h));
            p = P[v];
            g = G[v];
            if (p > (unsigned)K) p = 0;                              // not a class of this call
            if (g > (unsigned)K) g = 0;
            pb = class_border(P, (uint8_t)p, z, y, x, a.d, a.h, a.w, v) ? p : 0;
            gb = class_border(G, (uint8_t)g, z, y, x, a.d, a.h, a.w, v) ? g : 0;
            PB[v] = (uint8_t)pb;
            GB[v] = (uint8_t)gb;
            if (pb) box_add(cnt, pb, z, y, x, a.d, a.h, a.w);
            if (gb) box_add(cnt, gb, z, y, x, a.d, a.h, a.w);
        }
        warp_count(cnt[0], p);
        warp_count(cnt[1], g);
        warp_count(cnt[2], p == g ? p : 0);
        warp_count(cnt[3], pb);
        warp_count(cnt[4], gb);
    }
    __syncthreads();
    unsigned long long *rec = reinterpret_cast<unsigned long long *>(a.record) + (int64_t)b * K * SMB_METRIC_CLASS_NREC;
    for (int i = threadIdx.x; i < SMB_METRIC_CLASS_NREC * K; i += blockDim.x) {
        const int k = i / SMB_METRIC_CLASS_NREC, q = i % SMB_METRIC_CLASS_NREC;
        const unsigned c = cnt[q][k];
        if (c == 0) continue;
        if (q < 5) atomicAdd(rec + i, (unsigned long long)c);
        else atomicMax(rec + i, (unsigned long long)c);
    }
}

unsigned grid_for(int64_t work, int per_block, int jobs) {
    int64_t b = (work + per_block - 1) / per_block;
    const int64_t cap = (132 * 16 + jobs - 1) / jobs;
    if (b > cap) b = cap;
    return (unsigned)(b < 1 ? 1 : b);
}

int env_threads(int n) {                                               // threads (lines) per envelope block
    int t = (int)(kEnvSmem / (8 * (int64_t)(n + 0)) - 1) / 32 * 32;
    return t > 128 ? 128 : (t < 32 ? 32 : t);
}

}  // namespace

cudaError_t metric_bits_launch(const smb_metric_bits_args &a, cudaStream_t st) {
    const dim3 grid(grid_for(a.voxels, 256, a.batch), a.batch);
    if (a.kind == SMB_METRIC_LOGITS) {
        if (a.dtype == SMB_F32) logit_bits_kernel<float><<<grid, 256, 0, st>>>(a);
        else if (a.dtype == SMB_F16) logit_bits_kernel<__half><<<grid, 256, 0, st>>>(a);
        else logit_bits_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>(a);
    } else if (a.kind == SMB_METRIC_I8) {
        label_bits_kernel<int8_t><<<grid, 256, 0, st>>>(a);
    } else if (a.kind == SMB_METRIC_U8) {
        label_bits_kernel<uint8_t><<<grid, 256, 0, st>>>(a);
    } else if (a.kind == SMB_METRIC_I16) {
        label_bits_kernel<int16_t><<<grid, 256, 0, st>>>(a);
    } else if (a.kind == SMB_METRIC_I32) {
        label_bits_kernel<int32_t><<<grid, 256, 0, st>>>(a);
    } else {
        label_bits_kernel<int64_t><<<grid, 256, 0, st>>>(a);
    }
    count_launch();
    return cudaGetLastError();
}

cudaError_t metric_count_launch(const smb_metric_count_args &a, cudaStream_t st) {
    const int64_t n = (int64_t)a.d * a.h * a.w;
    count_kernel<<<dim3(grid_for(n, 256, a.batch), a.batch), 256, 0, st>>>(a);
    count_launch();
    return cudaGetLastError();
}

namespace {

// the three EDT passes over `njobs` jobs whose boxes lie within max_d x max_h x max_w: one launch per pass
template <class Jobs>
cudaError_t edt_launch(const Jobs &jobs, int njobs, int max_d, int max_h, int max_w, double s0, double s1, double s2, cudaStream_t st) {
    edt_axis0_kernel<Jobs><<<dim3(grid_for((int64_t)max_h * max_w, 256, 1), njobs), 256, 0, st>>>(jobs);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    const int t2 = env_threads(max_w), t1 = env_threads(max_h);
    const size_t sm2 = sizeof(int2) * (size_t)max_w * (t2 + 1), sm1 = sizeof(int2) * (size_t)max_h * (t1 + 1);
    e = cudaFuncSetAttribute(edt_axis2_kernel<Jobs>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm2);
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(edt_axis1_kernel<Jobs>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm1);
    if (e != cudaSuccess) return e;
    const int64_t l2 = (int64_t)max_d * max_h, l1 = (int64_t)max_d * max_w;
    edt_axis2_kernel<Jobs><<<dim3((unsigned)((l2 + t2 - 1) / t2), njobs), t2, sm2, st>>>(jobs, s0, s2);
    count_launch();
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    edt_axis1_kernel<Jobs><<<dim3((unsigned)((l1 + t1 - 1) / t1), njobs), t1, sm1, st>>>(jobs, s0, s1, s2);
    count_launch();
    return cudaGetLastError();
}

}  // namespace

cudaError_t metric_edt_launch(const smb_metric_edt_args &a, cudaStream_t st) {
    return edt_launch(RegionJobs{a}, a.batch * a.regions * 2, a.d, a.h, a.w, a.s0, a.s1, a.s2, st);
}

cudaError_t metric_select_launch(const smb_metric_select_args &a, cudaStream_t st) {
    select_kernel<<<a.batch * a.regions, kSelThreads, 0, st>>>(a);
    count_launch();
    return cudaGetLastError();
}

cudaError_t metric_class_count_launch(const smb_metric_class_count_args &a, cudaStream_t st) {
    const int64_t n = (int64_t)a.d * a.h * a.w;
    class_count_kernel<<<dim3(grid_for(n, 256, a.batch), a.batch), 256, 0, st>>>(a);
    count_launch();
    return cudaGetLastError();
}

cudaError_t metric_class_edt_launch(const smb_metric_class_edt_args &a, cudaStream_t st) {
    return edt_launch(TableJobs{a}, a.njobs, a.max_d, a.max_h, a.max_w, a.s0, a.s1, a.s2, st);
}

cudaError_t metric_class_reduce_launch(const smb_metric_class_reduce_args &a, cudaStream_t st) {
    class_reduce_kernel<<<a.npools, kSelThreads, 0, st>>>(a);
    count_launch();
    return cudaGetLastError();
}

}  // namespace smb
