// Case preprocessing (the reference's DefaultPreprocessor.run_case_npy and collect_foreground_intensities) as GPU stages;
// segmamba_b200/preprocess.py composes them with the hole filling of predict.cu and the cubic resize of augment.cu.
//
//   mask       one read of the channels: the nonzero mask, the labels as int8, and one record with the bbox, the
//              foreground count, NaN and bad-label counts (per-warp reductions, one atomic per warp and field)
//   crop       the bbox of the data and the labels into contiguous buffers, with crop_to_nonzero's -1 relabel
//   normalize  the z-score of a channel from its fp64 smb_aug_stats record
//   labels     resize_segmentation(order=1): fp64 trilinear indicators over the 8 taps, the highest label >= 0.5 wins
//   compaction per job, matching voxels counted per 1024-voxel chunk, an ordered scan of the chunk counts, then a ballot
//              scan inside each chunk writes the linear indices in raster order (predict.cu's numbering scheme)
//   gather     drawn positions of a compaction -> argwhere rows or per-channel values
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>

#include "prep_internal.h"

namespace smb {
void count_launch();

namespace {

constexpr int kThreads = 256, kChunk = SMB_PREP_CHUNK, kScanThreads = 1024;
constexpr int64_t kFlip = 1ll << 31;

template <class T> struct Jobs {
    T j[SMB_PREP_MAX_JOBS];
    int n;
};

unsigned grid_for(int64_t work, int per_block, int jobs) {
    int64_t b = (work + per_block - 1) / per_block;
    const int64_t cap = (132 * 16 + jobs - 1) / jobs;
    if (b > cap) b = cap;
    return (unsigned)(b < 1 ? 1 : b);
}

__device__ inline unsigned long long warp_max(unsigned long long v) {
    for (int o = 16; o; o >>= 1) {
        const unsigned long long y = __shfl_down_sync(0xffffffffu, v, o);
        v = y > v ? y : v;
    }
    return v;
}

__device__ inline unsigned long long warp_sum(unsigned long long v) {
    for (int o = 16; o; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    return v;
}

// ---- mask pass ----------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) mask_kernel(smb_prep_mask_args a) {
    const int64_t n = (int64_t)a.d * a.h * a.w;
    unsigned long long lo[3] = {0, 0, 0}, hi[3] = {0, 0, 0}, fg = 0, nan = 0, bad = 0;
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < n; v += (int64_t)gridDim.x * blockDim.x) {
        bool nz = false, isnan = false;
        for (int c = 0; c < a.channels; ++c) {
            const float x = a.data[(int64_t)c * n + v];
            nz = nz || x != 0.f;
            isnan = isnan || x != x;
        }
        a.mask[v] = nz;
        nan += isnan;
        if (nz) {
            const int64_t p[3] = {v / ((int64_t)a.h * a.w), (v / a.w) % a.h, v % a.w};
            for (int q = 0; q < 3; ++q) {
                const unsigned long long f = (unsigned long long)(kFlip - p[q]), e = (unsigned long long)(p[q] + 1);
                lo[q] = f > lo[q] ? f : lo[q];
                hi[q] = e > hi[q] ? e : hi[q];
            }
        }
        int8_t l = 0;
        if (a.seg) {
            const float s = a.seg[v];
            const bool ok = s >= 0.f && s <= 127.f && s == floorf(s);   // false for NaN
            bad += !ok;
            fg += s > 0.f;
            l = ok ? (int8_t)s : (int8_t)0;
        }
        a.seg8[v] = l;
    }
    unsigned long long *r = reinterpret_cast<unsigned long long *>(a.record);
    for (int q = 0; q < 3; ++q) {
        lo[q] = warp_max(lo[q]);
        hi[q] = warp_max(hi[q]);
    }
    fg = warp_sum(fg);
    nan = warp_sum(nan);
    bad = warp_sum(bad);
    if ((threadIdx.x & 31) == 0) {
        for (int q = 0; q < 3; ++q) {
            if (lo[q]) atomicMax(r + q, lo[q]);
            if (hi[q]) atomicMax(r + 3 + q, hi[q]);
        }
        if (fg) atomicAdd(r + 6, fg);
        if (nan) atomicAdd(r + 7, nan);
        if (bad) atomicAdd(r + 8, bad);
    }
}

// ---- crop + relabel -------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) crop_kernel(smb_prep_crop_args a) {
    const int64_t n = (int64_t)a.d * a.h * a.w, m = (int64_t)a.cd * a.ch * a.cw;
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < m; v += (int64_t)gridDim.x * blockDim.x) {
        const int x = (int)(v % a.cw), y = (int)((v / a.cw) % a.ch), z = (int)(v / ((int64_t)a.cw * a.ch));
        const int64_t s = ((int64_t)(z + a.z0) * a.h + (y + a.y0)) * a.w + (x + a.x0);
        for (int c = 0; c < a.channels; ++c) a.out[(int64_t)c * m + v] = a.data[(int64_t)c * n + s];
        const int8_t l = a.seg8[s];
        a.seg_out[v] = (l == 0 && !a.mask[s]) ? (int8_t)a.nonzero_label : l;
    }
}

// ---- z-score ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) normalize_kernel(Jobs<smb_prep_norm_job> jobs) {
    const smb_prep_norm_job jb = jobs.j[blockIdx.y];
    const double mean = jb.stats[0] / (double)jb.n;
    const double var = jb.stats[1] / (double)jb.n - mean * mean;
    const double sd = sqrt(var > 0.0 ? var : 0.0);
    const double div = sd > 1e-8 ? sd : 1e-8;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        jb.moments[0] = mean;
        jb.moments[1] = sd;
    }
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < jb.n; v += (int64_t)gridDim.x * blockDim.x)
        jb.dst[v] = (float)(((double)jb.src[v] - mean) / div);
}

// ---- CT normalisation -----------------------------------------------------------------------------------------------------------
// numpy's clip (maximum, then minimum; a NaN passes through, -0 stays -0) and two fp32 operations: a subtraction and an IEEE
// division cannot contract into an FMA, so the result is bit-equal to numpy's float32 arithmetic
__global__ void __launch_bounds__(kThreads) ct_normalize_kernel(Jobs<smb_prep_ct_norm_job> jobs) {
    const smb_prep_ct_norm_job jb = jobs.j[blockIdx.y];
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < jb.n; v += (int64_t)gridDim.x * blockDim.x) {
        float x = jb.src[v];
        x = x < jb.lo ? jb.lo : x;
        x = x > jb.hi ? jb.hi : x;
        jb.dst[v] = (x - jb.mean) / jb.div;
    }
}

// ---- order-1 label resize -------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) label_resize_kernel(smb_prep_label_resize_args a) {
    const int n[3] = {a.n0, a.n1, a.n2};
    const int m[3] = {a.m0, a.m1, a.m2};
    const int64_t vol = (int64_t)a.m0 * a.m1 * a.m2;
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < vol; v += (int64_t)gridDim.x * blockDim.x) {
        const int o[3] = {(int)(v / ((int64_t)a.m1 * a.m2)), (int)((v / a.m2) % a.m1), (int)(v % a.m2)};
        int i0[3], i1[3];
        double w[3][2];
        for (int d = 0; d < 3; ++d) {
            double x = __dadd_rn(__dmul_rn((double)o[d] + 0.5, (double)n[d] / (double)m[d]), -0.5);   // no contraction
            x = x < 0.0 ? 0.0 : (x > (double)(n[d] - 1) ? (double)(n[d] - 1) : x);   // scipy's map_coordinate, mode 'nearest'
            const double fl = floor(x);
            i0[d] = (int)fl;
            i1[d] = i0[d] + 1 > n[d] - 1 ? n[d] - 1 : i0[d] + 1;
            w[d][1] = x - fl;
            w[d][0] = 1.0 - w[d][1];
        }
        int8_t lab[8];
        double wt[8];
        for (int c = 0; c < 8; ++c) {                                   // taps in scipy's order: the last axis fastest
            const int a0 = c >> 2, a1 = (c >> 1) & 1, a2 = c & 1;
            const int zz = a0 ? i1[0] : i0[0], yy = a1 ? i1[1] : i0[1], xx = a2 ? i1[2] : i0[2];
            lab[c] = a.src[((int64_t)zz * n[1] + yy) * n[2] + xx];
            wt[c] = __dmul_rn(__dmul_rn(w[0][a0], w[1][a1]), w[2][a2]);
        }
        int best = 0;
        bool won = false;
        for (int c = 0; c < 8; ++c) {
            bool seen = false;
            for (int e = 0; e < c; ++e) seen = seen || lab[e] == lab[c];
            if (seen) continue;
            double ind = 0.0;
            for (int e = c; e < 8; ++e) ind = __dadd_rn(ind, lab[e] == lab[c] ? wt[e] : 0.0);
            if (ind >= 0.5 && (!won || lab[c] > best)) { best = lab[c]; won = true; }   // ascending labels, later ones overwrite
        }
        a.dst[v] = (int8_t)best;
    }
}

// ---- ordered compaction ---------------------------------------------------------------------------------------------------------
// the label set is staged in shared memory: indexing the by-value job record with a label would put it in local memory
__device__ inline const unsigned *stage_set(const smb_prep_compact_job &jb, unsigned *set) {
    if (threadIdx.x < 8) set[threadIdx.x] = jb.set[threadIdx.x];
    __syncthreads();
    return set;
}

__device__ inline bool in_set(const smb_prep_compact_job &jb, const unsigned *set, int64_t v) {
    const unsigned l = (uint8_t)jb.seg[v];
    return (set[l >> 5] >> (l & 31)) & 1u;
}

// one block per chunk and job: chunk[k] = matching voxels of chunk k
__global__ void __launch_bounds__(kThreads) count_kernel(Jobs<smb_prep_compact_job> jobs) {
    __shared__ int red[kThreads / 32];
    __shared__ unsigned set_s[8];
    const smb_prep_compact_job &jb = jobs.j[blockIdx.y];
    const unsigned *set = stage_set(jb, set_s);
    const int64_t chunks = (jb.n + kChunk - 1) / kChunk;
    for (int64_t k = blockIdx.x; k < chunks; k += gridDim.x) {
        int s = 0;
        for (int q = 0; q < kChunk / kThreads; ++q) {
            const int64_t v = k * kChunk + q * kThreads + threadIdx.x;
            s += v < jb.n && in_set(jb, set, v);
        }
        for (int o = 16; o; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
        __syncthreads();
        if (threadIdx.x == 0) {
            int t = 0;
            for (int q = 0; q < kThreads / 32; ++q) t += red[q];
            jb.chunk[k] = t;
        }
        __syncthreads();
    }
}

// one block per job: exclusive scan of the chunk counts in place, the total to *count
__global__ void __launch_bounds__(kScanThreads) scan_kernel(Jobs<smb_prep_compact_job> jobs) {
    __shared__ int64_t wsum[kScanThreads / 32];
    const smb_prep_compact_job jb = jobs.j[blockIdx.x];
    const int64_t nchunks = (jb.n + kChunk - 1) / kChunk;
    const int64_t per = (nchunks + kScanThreads - 1) / kScanThreads;
    const int64_t lo = min((int64_t)threadIdx.x * per, nchunks), hi = min(lo + per, nchunks);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int64_t s = 0;
    for (int64_t i = lo; i < hi; ++i) s += jb.chunk[i];
    int64_t incl = s;
    for (int o = 1; o < 32; o <<= 1) {
        const int64_t y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
    }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        const int64_t ws = wsum[lane];
        int64_t wi = ws;
        for (int o = 1; o < 32; o <<= 1) {
            const int64_t y = __shfl_up_sync(0xffffffffu, wi, o);
            if (lane >= o) wi += y;
        }
        wsum[lane] = wi - ws;
    }
    __syncthreads();
    int64_t run = wsum[warp] + incl - s;
    for (int64_t i = lo; i < hi; ++i) {
        const int t = jb.chunk[i];
        jb.chunk[i] = (int)run;
        run += t;
    }
    if (threadIdx.x == kScanThreads - 1) *jb.count = run;
}

// one block per chunk and job: matching voxels written at the chunk offset plus their rank inside the chunk
__global__ void __launch_bounds__(kThreads) compact_kernel(Jobs<smb_prep_compact_job> jobs) {
    __shared__ int wsum[kThreads / 32];
    __shared__ unsigned set_s[8];
    const smb_prep_compact_job &jb = jobs.j[blockIdx.y];
    const unsigned *set = stage_set(jb, set_s);
    const int64_t chunks = (jb.n + kChunk - 1) / kChunk;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int64_t k = blockIdx.x; k < chunks; k += gridDim.x) {
        int base = jb.chunk[k];
        for (int q = 0; q < kChunk / kThreads; ++q) {
            const int64_t v = k * kChunk + q * kThreads + threadIdx.x;
            const bool hit = v < jb.n && in_set(jb, set, v);
            const unsigned b = __ballot_sync(0xffffffffu, hit);
            if (lane == 0) wsum[warp] = __popc(b);
            __syncthreads();
            int before = 0, total = 0;
            for (int w = 0; w < kThreads / 32; ++w) {
                before += w < warp ? wsum[w] : 0;
                total += wsum[w];
            }
            if (hit) jb.index[base + before + __popc(b & ((1u << lane) - 1u))] = (int32_t)v;
            base += total;
            __syncthreads();
        }
    }
}

// ---- gather -----------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) gather_kernel(smb_prep_gather_args a) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * blockDim.x) {
        if (a.rows) {
            const int64_t p = a.index[a.select ? a.select[i] : i];
            int64_t *r = a.rows + 4 * i;
            r[0] = 0;
            r[1] = p / ((int64_t)a.h * a.w);
            r[2] = (p / a.w) % a.h;
            r[3] = p % a.w;
        }
        if (a.values)
            for (int c = 0; c < a.channels; ++c) {
                const int64_t p = a.index[a.select ? a.select[(int64_t)c * a.select_channel_stride + i] : i];
                a.values[(int64_t)c * a.n + i] = a.data[(int64_t)c * a.channel_stride + p];
            }
    }
}

template <class T, class F> cudaError_t for_chunks(const T *jobs, int n, F &&launch) {
    for (int base = 0; base < n; base += SMB_PREP_MAX_JOBS) {
        Jobs<T> js;
        js.n = n - base < SMB_PREP_MAX_JOBS ? n - base : SMB_PREP_MAX_JOBS;
        for (int q = 0; q < js.n; ++q) js.j[q] = jobs[base + q];
        for (int q = js.n; q < SMB_PREP_MAX_JOBS; ++q) js.j[q] = jobs[base];
        cudaError_t e = launch(js);
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

template <class T> int64_t max_n(const Jobs<T> &js) {
    int64_t m = 0;
    for (int q = 0; q < js.n; ++q) m = js.j[q].n > m ? js.j[q].n : m;
    return m;
}

}  // namespace

cudaError_t prep_mask_launch(const smb_prep_mask_args &a, cudaStream_t st) {
    cudaError_t e = cudaMemsetAsync(a.record, 0, sizeof(smb_prep_record), st);
    if (e != cudaSuccess) return e;
    mask_kernel<<<grid_for((int64_t)a.d * a.h * a.w, kThreads, 1), kThreads, 0, st>>>(a);
    count_launch();
    return cudaGetLastError();
}

cudaError_t prep_crop_launch(const smb_prep_crop_args &a, cudaStream_t st) {
    crop_kernel<<<grid_for((int64_t)a.cd * a.ch * a.cw, kThreads, 1), kThreads, 0, st>>>(a);
    count_launch();
    return cudaGetLastError();
}

cudaError_t prep_normalize_launch(const smb_prep_norm_job *jobs, int n, cudaStream_t st) {
    return for_chunks(jobs, n, [&](const Jobs<smb_prep_norm_job> &js) {
        normalize_kernel<<<dim3(grid_for(max_n(js), kThreads, js.n), js.n), kThreads, 0, st>>>(js);
        count_launch();
        return cudaGetLastError();
    });
}

cudaError_t prep_ct_normalize_launch(const smb_prep_ct_norm_job *jobs, int n, cudaStream_t st) {
    return for_chunks(jobs, n, [&](const Jobs<smb_prep_ct_norm_job> &js) {
        ct_normalize_kernel<<<dim3(grid_for(max_n(js), kThreads, js.n), js.n), kThreads, 0, st>>>(js);
        count_launch();
        return cudaGetLastError();
    });
}

cudaError_t prep_label_resize_launch(const smb_prep_label_resize_args &a, cudaStream_t st) {
    label_resize_kernel<<<grid_for((int64_t)a.m0 * a.m1 * a.m2, kThreads, 1), kThreads, 0, st>>>(a);
    count_launch();
    return cudaGetLastError();
}

cudaError_t prep_count_launch(const smb_prep_compact_job *jobs, int n, cudaStream_t st) {
    return for_chunks(jobs, n, [&](const Jobs<smb_prep_compact_job> &js) {
        count_kernel<<<dim3(grid_for(max_n(js), kChunk, js.n), js.n), kThreads, 0, st>>>(js);
        count_launch();
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
        scan_kernel<<<js.n, kScanThreads, 0, st>>>(js);
        count_launch();
        return cudaGetLastError();
    });
}

cudaError_t prep_compact_launch(const smb_prep_compact_job *jobs, int n, cudaStream_t st) {
    return for_chunks(jobs, n, [&](const Jobs<smb_prep_compact_job> &js) {
        compact_kernel<<<dim3(grid_for(max_n(js), kChunk, js.n), js.n), kThreads, 0, st>>>(js);
        count_launch();
        return cudaGetLastError();
    });
}

cudaError_t prep_gather_launch(const smb_prep_gather_args &a, cudaStream_t st) {
    gather_kernel<<<grid_for(a.n, kThreads, 1), kThreads, 0, st>>>(a);
    count_launch();
    return cudaGetLastError();
}

}  // namespace smb
