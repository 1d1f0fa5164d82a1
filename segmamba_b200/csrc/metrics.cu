// Dice and Hausdorff-percentile evaluation (medpy.metric.binary.dc / hd95 / hd, connectivity 1, as the reference's
// 5_compute_metrics.py and validation_step use them) on region bitmasks.
//
// The distance transform is exact and separable: a 1-D nearest-feature sweep along axis 0, then two lower-envelope passes
// (Meijster et al., 2000) along axes 2 and 1 in fp64 with the voxel spacing.  Each voxel carries the linear index of its
// nearest feature so the last pass can form the distance from the offsets the way scipy does.  A lower-envelope pass runs one
// thread per line; the line and its envelope stack share one 8-byte slot per position in shared memory (the stack never
// grows past the position being read, and the answers overwrite dead stack slots).
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
// job j = (b * regions + r) * 2 + dir; dir 0: source P's border, target G's border; dir 1 the other way round
struct Job {
    const uint8_t *src, *tgt;
    int32_t *feat;
    int b, r, bit;
};

__device__ inline Job job_of(const smb_metric_edt_args &a, int j) {
    Job o;
    const int64_t n = (int64_t)a.d * a.h * a.w;
    const int pair = j >> 1, dir = j & 1;
    o.b = pair / a.regions;
    o.r = pair % a.regions;
    o.bit = 1 << o.r;
    const uint8_t *pb = reinterpret_cast<const uint8_t *>(a.pred_border) + (int64_t)o.b * n;
    const uint8_t *gb = reinterpret_cast<const uint8_t *>(a.target_border) + (int64_t)o.b * n;
    o.src = dir ? gb : pb;
    o.tgt = dir ? pb : gb;
    o.feat = a.feat + (int64_t)j * n;
    return o;
}

// axis 0: feat = linear index of the nearest target voxel in the voxel's column (ties: the lower z), -1 if none
__global__ void __launch_bounds__(256) edt_axis0_kernel(smb_metric_edt_args a) {
    const Job jb = job_of(a, blockIdx.y);
    const int64_t hw = (int64_t)a.h * a.w;
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < hw; c += (int64_t)gridDim.x * blockDim.x) {
        int last = -1;
        for (int z = 0; z < a.d; ++z) {
            if (jb.tgt[z * hw + c] & jb.bit) last = z;
            jb.feat[z * hw + c] = last;
        }
        int next = -1;
        for (int z = a.d - 1; z >= 0; --z) {
            if (jb.tgt[z * hw + c] & jb.bit) next = z;
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
__global__ void __launch_bounds__(128) edt_axis2_kernel(smb_metric_edt_args a) {
    extern __shared__ int2 env[];
    const Job jb = job_of(a, blockIdx.y);
    const int T = blockDim.x, stride = T + 1, n = a.w;
    const int64_t lines = (int64_t)a.d * a.h, l0 = (int64_t)blockIdx.x * T;
    if (l0 >= lines) return;
    const int nl = (int)(lines - l0 < T ? lines - l0 : T);
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5, nwarps = T >> 5;
    for (int u = warp; u < nl; u += nwarps)
        for (int p = lane; p < n; p += 32) env[p * stride + u].x = jb.feat[(l0 + u) * n + p];
    __syncthreads();
    if (t < nl) {
        const int z = (int)((l0 + t) / a.h);
        const int64_t hw = (int64_t)a.h * a.w;
        const double s0 = a.s0;
        envelope(env + t, stride, n, a.s2 * a.s2, [&](int f) { return sq((double)((int)(f / hw) - z) * s0); });
    }
    __syncthreads();
    for (int u = warp; u < nl; u += nwarps)
        for (int p = lane; p < n; p += 32) jb.feat[(l0 + u) * n + p] = env[p * stride + u].x;
}

// axis 1 (columns of a z slice), the last pass: each thread stages and walks one column; distances at the source voxels go to
// the pool of (b, r)
__global__ void __launch_bounds__(128) edt_axis1_kernel(smb_metric_edt_args a) {
    extern __shared__ int2 env[];
    const Job jb = job_of(a, blockIdx.y);
    const int T = blockDim.x, stride = T + 1, n = a.h, t = threadIdx.x;
    const int64_t lines = (int64_t)a.d * a.w, l = (int64_t)blockIdx.x * T + t;
    if (l >= lines) return;
    const int z = (int)(l / a.w), x = (int)(l % a.w);
    const int64_t hw = (int64_t)a.h * a.w, base = z * hw + x;
    int2 *s = env + t;
    for (int p = 0; p < n; ++p) s[p * stride].x = jb.feat[base + (int64_t)p * a.w];
    const double s0 = a.s0, s1 = a.s1, s2 = a.s2;
    envelope(s, stride, n, s1 * s1, [&](int f) {
        return __dadd_rn(sq((double)((int)(f / hw) - z) * s0), sq((double)((int)(f % a.w) - x) * s2));
    });
    unsigned long long *fill = reinterpret_cast<unsigned long long *>(a.counts) + ((int64_t)jb.b * a.regions + jb.r) * SMB_METRIC_NCOUNTS + 5;
    double *pool = a.pool + ((int64_t)jb.b * a.regions + jb.r) * a.pool_cap;
    for (int p = 0; p < n; ++p) {
        if (!(jb.src[base + (int64_t)p * a.w] & jb.bit)) continue;
        const int f = s[p * stride].x;
        if (f < 0) continue;
        const int fz = (int)(f / hw), fy = (int)((f / a.w) % a.h), fx = (int)(f % a.w);
        const double d0 = (double)(fz - z) * s0, d1 = (double)(fy - p) * s1, d2 = (double)(fx - x) * s2;
        const double dist = sqrt(__dadd_rn(__dadd_rn(sq(d0), sq(d1)), sq(d2)));
        pool[atomicAdd(fill, 1ull)] = dist;
    }
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

__global__ void __launch_bounds__(kSelThreads) select_kernel(smb_metric_select_args a) {
    __shared__ unsigned hist[256];
    __shared__ unsigned long long red[kSelThreads / 32];
    __shared__ unsigned long long pre_s, k_s, eq_s;
    const int pr = blockIdx.x;
    const int64_t *c = a.counts + (int64_t)pr * SMB_METRIC_NCOUNTS;
    if (c[0] == 0 || c[1] == 0) {
        if (threadIdx.x == 0) a.out[pr] = NAN;
        return;
    }
    const int64_t n = c[5];
    const unsigned long long *key = reinterpret_cast<const unsigned long long *>(a.pool + (int64_t)pr * a.pool_cap);
    // numpy 'linear': virtual index (n - 1) q; at or past the last index both neighbours are the maximum
    const double vi = (double)(n - 1) * a.frac;
    int64_t kp;
    double gamma = 0.0;
    if (vi >= (double)(n - 1)) {
        kp = n - 1;
    } else {
        const double fl = floor(vi);
        kp = (int64_t)fl;
        gamma = vi - fl;
    }
    if (threadIdx.x == 0) { pre_s = 0; k_s = (unsigned long long)kp; }
    unsigned long long mask = 0;
    for (int shift = 56; shift >= 0; shift -= 8) {
        for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
        __syncthreads();
        const unsigned long long pre = pre_s;
        for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
            const unsigned long long k = key[i];
            if ((k & mask) == pre) atomicAdd(&hist[(k >> shift) & 255], 1u);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned long long k = k_s;
            int d = 0;
            while (hist[d] <= k) k -= hist[d++];
            k_s = k;
            pre_s = pre | ((unsigned long long)d << shift);
            eq_s = hist[d];
        }
        mask |= 255ull << shift;
        __syncthreads();
    }
    const unsigned long long va = pre_s;
    unsigned long long vb = va;
    if (kp + 1 < n && gamma != 0.0 && k_s + 1 >= eq_s) {                 // rank kp + 1 lies above the run of va
        unsigned long long m = ~0ull;
        for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
            const unsigned long long k = key[i];
            if (k > va && k < m) m = k;
        }
        vb = block_min(m, red);
    }
    if (threadIdx.x == 0) {
        double x, y;
        memcpy(&x, &va, 8);
        memcpy(&y, &vb, 8);
        // numpy's _lerp, both branches, without contraction
        const double diff = __dsub_rn(y, x);
        a.out[pr] = gamma >= 0.5 ? __dsub_rn(y, __dmul_rn(diff, __dsub_rn(1.0, gamma))) : __dadd_rn(x, __dmul_rn(diff, gamma));
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

cudaError_t metric_edt_launch(const smb_metric_edt_args &a, cudaStream_t st) {
    const int jobs = a.batch * a.regions * 2;
    edt_axis0_kernel<<<dim3(grid_for((int64_t)a.h * a.w, 256, 1), jobs), 256, 0, st>>>(a);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    const int t2 = env_threads(a.w), t1 = env_threads(a.h);
    const size_t sm2 = sizeof(int2) * (size_t)a.w * (t2 + 1), sm1 = sizeof(int2) * (size_t)a.h * (t1 + 1);
    e = cudaFuncSetAttribute(edt_axis2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm2);
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(edt_axis1_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm1);
    if (e != cudaSuccess) return e;
    const int64_t l2 = (int64_t)a.d * a.h, l1 = (int64_t)a.d * a.w;
    edt_axis2_kernel<<<dim3((unsigned)((l2 + t2 - 1) / t2), jobs), t2, sm2, st>>>(a);
    count_launch();
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    edt_axis1_kernel<<<dim3((unsigned)((l1 + t1 - 1) / t1), jobs), t1, sm1, st>>>(a);
    count_launch();
    return cudaGetLastError();
}

cudaError_t metric_select_launch(const smb_metric_select_args &a, cudaStream_t st) {
    select_kernel<<<a.batch * a.regions, kSelThreads, 0, st>>>(a);
    count_launch();
    return cudaGetLastError();
}

}  // namespace smb
