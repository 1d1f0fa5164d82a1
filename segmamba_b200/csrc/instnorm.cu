// Fused InstanceNorm3d (+ optional second operand, + ReLU / LeakyReLU) forward / backward for sm_90a,
// on channels-last activations viewed as (batch, spatial, channels).
//
// Replaces the reference's nn.InstanceNorm3d(affine=False, eps=1e-5) + activation + residual-add chains:
//   GSC            ReLU(IN(conv(x)))                                   model_segmamba/segmamba.py:111-130
//   UnetResBlock   LReLU(IN(conv1)),  LReLU(IN(conv2) + IN(conv3(res))) or LReLU(IN(conv2) + res)
//                                                                      monai/networks/blocks/dynunet_block.py:98-111
//   downsample / norm{i}   IN(x)                                       segmamba.py:147,171
// which the reference runs as ATen batch_norm kernels in fp32 plus separate elementwise kernels (38 % of its
// training step).  These are pure HBM streaming ops:
//   forward : 1 read for the statistics + 1 read + 1 write for the apply     (per operand)
//   backward: reads dy, x (, x2) twice (sums, then apply), writes dx (, dx2)
// Mapping: a CTA owns a contiguous range of rows (voxels); thread (r, cv) owns the 16-byte column vector cv of
// rows r, r+RB, ...; so every global access is a full coalesced row segment and per-channel statistics live in
// registers.  Variance uses per-CTA centred sums merged with Chan's formula (no E[x^2]-E[x]^2 cancellation
// across the 2 M-voxel reduction).
#include "norm_internal.h"

namespace smb {

constexpr int kNormThreads = 256;
#ifndef SMB_IN_FWD_MINB
#define SMB_IN_FWD_MINB 3
#endif
// backward kernels, by second-operand mode (tools/norm_bench.py sweeps them; the values below were not re-swept on H100; the
// two-norm one spills beyond 2 and stays there)
#ifndef SMB_IN_BWD_MINB0
#define SMB_IN_BWD_MINB0 5
#endif
#ifndef SMB_IN_BWD_MINB1
#define SMB_IN_BWD_MINB1 4
#endif
#ifndef SMB_IN_BWD_MINB2
#define SMB_IN_BWD_MINB2 2
#endif
// rows in flight per thread in the apply / backward-sum passes (memory-level parallelism against registers)
#ifndef SMB_IN_U_FWD
#define SMB_IN_U_FWD 2
#endif
#ifndef SMB_IN_U_BWD0
#define SMB_IN_U_BWD0 1
#endif
#ifndef SMB_IN_U_BWD2
#define SMB_IN_U_BWD2 1
#endif

// Non-finite semantics are torch's: ReLU is threshold(v, 0, 0), so NaN passes through it, and its backward
// (threshold_backward) selects rather than multiplies -- g passes where v is NaN and is dropped, even if non-finite, where
// v <= 0.  LeakyReLU's backward multiplies (g * slope), as leaky_relu_backward does.
__device__ __forceinline__ float act_fwd(float v, int act, float slope) {
    if (act == 1) return v <= 0.f ? 0.f : v;
    if (act == 2) return v > 0.f ? v : slope * v;
    return v;
}
// g * act'(v), for the incoming gradient g and the pre-activation v
__device__ __forceinline__ float act_bwd(float g, float v, int act, float slope) {
    if (act == 1) return v <= 0.f ? 0.f : g;
    if (act == 2) return v > 0.f ? g : g * slope;
    return g;
}

// Build-time knob (tools/build_variants.py in_rev): the apply passes walk their row range from the top down.  The statistics pass
// that precedes them streams the same range bottom-up, so what is still in the 126 MB L2 when it ends is the TOP of every CTA's
// range; reading that first turns part of the second read of a > L2 tensor into L2 hits.  Default off (unmeasured).
#ifndef SMB_IN_APPLY_REVERSE
#define SMB_IN_APPLY_REVERSE 0
#endif
#if SMB_IN_APPLY_REVERSE
#define SMB_APPLY_ROW(m, row) ((m).row_lo + (m).row_hi - 1 - (row))
#else
#define SMB_APPLY_ROW(m, row) (row)
#endif
// The mirror image (variant in_rev_stats): the STATISTICS passes walk top-down, so they start with what the producer of the
// tensor (a cuDNN convolution, if it writes in row order) left in L2, and end where the bottom-up apply pass starts.
#ifndef SMB_IN_STATS_REVERSE
#define SMB_IN_STATS_REVERSE 0
#endif
#if SMB_IN_STATS_REVERSE
#define SMB_STATS_ROW(m, row) ((m).row_lo + (m).row_hi - 1 - (row))
#else
#define SMB_STATS_ROW(m, row) (row)
#endif

struct RowMap {
    int cv, r, RB;
    int64_t row_lo, row_hi;
    bool active;
};
// thread -> (column vector, first row, row step) for the CTA's row range
__device__ __forceinline__ RowMap row_map(const NormP &p, int CV) {
    RowMap m;
    m.RB = kNormThreads / CV;
    m.cv = threadIdx.x % CV;
    m.r = threadIdx.x / CV;
    m.active = m.r < m.RB;
    m.row_lo = (int64_t)blockIdx.x * p.rows_per_cta;
    m.row_hi = min(p.spatial, m.row_lo + p.rows_per_cta);
    return m;
}

// ---------------------------------------------------------------------------------------------
// forward statistics: per-CTA (count, mean, M2) per channel, for x and optionally x2
// partial layout: [which][batch][cta][3][C]
// ---------------------------------------------------------------------------------------------
template <typename T, bool kTwo>
__global__ void __launch_bounds__(kNormThreads) in_stats_fwd_kernel(const NormP p) {
    constexpr int V = VecOf<T>::V;
    extern __shared__ float sm[];                        // [RB][C] x (2 or 4)
    const int C = p.channels, CV = C / V;
    const RowMap m = row_map(p, CV);
    const int b = blockIdx.y;
    const T *x = reinterpret_cast<const T *>(p.x) + (int64_t)b * p.spatial * C;
    const T *x2 = kTwo ? reinterpret_cast<const T *>(p.x2) + (int64_t)b * p.spatial * C : nullptr;
    float s1[V], q1[V], s2[V], q2[V];
#pragma unroll
    for (int v = 0; v < V; ++v) { s1[v] = q1[v] = s2[v] = q2[v] = 0.f; }
    // centre on the first row of the CTA's range to keep the sums small (shift invariance of the variance)
    float c1[V], c2[V];
    if (m.row_lo < m.row_hi) {
        loadv<T, V>(x + m.row_lo * C + m.cv * V, c1);
        if (kTwo) loadv<T, V>(x2 + m.row_lo * C + m.cv * V, c2);
    }
    if (m.active) {
        constexpr int U = 4;                             // rows in flight per thread (memory-level parallelism)
        int64_t row = m.row_lo + m.r;
        for (; row + (int64_t)(U - 1) * m.RB < m.row_hi; row += (int64_t)U * m.RB) {
            float a[U][V], a2[U][V];
#pragma unroll
            for (int k = 0; k < U; ++k) {
                const int64_t sr = SMB_STATS_ROW(m, row + (int64_t)k * m.RB);
                loadv<T, V>(x + sr * C + m.cv * V, a[k]);
                if (kTwo) loadv<T, V>(x2 + sr * C + m.cv * V, a2[k]);
            }
#pragma unroll
            for (int k = 0; k < U; ++k) {
#pragma unroll
                for (int v = 0; v < V; ++v) {
                    const float d = a[k][v] - c1[v]; s1[v] += d; q1[v] = fmaf(d, d, q1[v]);
                    if (kTwo) { const float e = a2[k][v] - c2[v]; s2[v] += e; q2[v] = fmaf(e, e, q2[v]); }
                }
            }
        }
        for (; row < m.row_hi; row += m.RB) {
            float a[V];
            loadv<T, V>(x + SMB_STATS_ROW(m, row) * C + m.cv * V, a);
#pragma unroll
            for (int v = 0; v < V; ++v) { const float d = a[v] - c1[v]; s1[v] += d; q1[v] = fmaf(d, d, q1[v]); }
            if (kTwo) {
                loadv<T, V>(x2 + SMB_STATS_ROW(m, row) * C + m.cv * V, a);
#pragma unroll
                for (int v = 0; v < V; ++v) { const float d = a[v] - c2[v]; s2[v] += d; q2[v] = fmaf(d, d, q2[v]); }
            }
        }
    }
    const int RB = m.RB;
    float *S1 = sm, *Q1 = sm + RB * C, *S2 = sm + 2 * RB * C, *Q2 = sm + 3 * RB * C;
    if (m.active) {
#pragma unroll
        for (int v = 0; v < V; ++v) {
            S1[m.r * C + m.cv * V + v] = s1[v];
            Q1[m.r * C + m.cv * V + v] = q1[v];
            if (kTwo) { S2[m.r * C + m.cv * V + v] = s2[v]; Q2[m.r * C + m.cv * V + v] = q2[v]; }
        }
    }
    __syncthreads();
    const float n = (float)(m.row_hi - m.row_lo);
    for (int c = threadIdx.x; c < C; c += kNormThreads) {
        float a = 0.f, q = 0.f, a2 = 0.f, qq2 = 0.f;
        for (int r = 0; r < RB; ++r) {
            a += S1[r * C + c]; q += Q1[r * C + c];
            if (kTwo) { a2 += S2[r * C + c]; qq2 += Q2[r * C + c]; }
        }
        // shift back: mean = centre + a/n ; M2 = q - a^2/n
        const float ctr = n > 0.f ? to_f32<T>(x[m.row_lo * C + c]) : 0.f;
        float *o = p.partial + (((int64_t)b * gridDim.x + blockIdx.x) * 3) * C + c;
        o[0] = n;
        o[C] = n > 0.f ? ctr + a / n : 0.f;
        o[2 * C] = n > 0.f ? q - a * a / n : 0.f;
        if (kTwo) {
            const float ctr2 = n > 0.f ? to_f32<T>(x2[m.row_lo * C + c]) : 0.f;
            float *o2 = o + (int64_t)p.batch * gridDim.x * 3 * C;
            o2[0] = n;
            o2[C] = n > 0.f ? ctr2 + a2 / n : 0.f;
            o2[2 * C] = n > 0.f ? qq2 - a2 * a2 / n : 0.f;
        }
    }
}

// merge the per-CTA (n, mean, M2) with Chan's parallel formula -> (mean, rstd).
// Block = 32 channels x 32 partial-groups (coalesced 128-byte reads along the channel axis); grid = (C/32, batch, which).
__global__ void __launch_bounds__(1024) in_finalize_fwd_kernel(const float *__restrict__ partial, float *__restrict__ stats,
                                                              float *__restrict__ stats2, int batch, int C, int n_cta, float eps) {
    __shared__ float sn[32][33], smean[32][33], sm2[32][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + tx, b = blockIdx.y, which = blockIdx.z;
    float n = 0.f, mean = 0.f, M2 = 0.f;
    if (c < C) {
        const float *pp = partial + (int64_t)which * batch * n_cta * 3 * C + ((int64_t)b * n_cta * 3) * C + c;
        for (int k = ty; k < n_cta; k += 32) {
            const float nk = pp[(int64_t)k * 3 * C], mk = pp[(int64_t)k * 3 * C + C], qk = pp[(int64_t)k * 3 * C + 2 * C];
            if (nk > 0.f) {
                const float nt = n + nk, dlt = mk - mean;
                mean += dlt * (nk / nt);
                M2 += qk + dlt * dlt * (n * nk / nt);
                n = nt;
            }
        }
    }
    sn[ty][tx] = n; smean[ty][tx] = mean; sm2[ty][tx] = M2;
    __syncthreads();
    if (ty == 0 && c < C) {
        double dn = 0.0, dmean = 0.0, dM2 = 0.0;
        for (int g = 0; g < 32; ++g) {
            const double nk = sn[g][tx], mk = smean[g][tx], qk = sm2[g][tx];
            if (nk <= 0.0) continue;
            const double nt = dn + nk, dlt = mk - dmean;
            dmean += dlt * nk / nt;
            dM2 += qk + dlt * dlt * dn * nk / nt;
            dn = nt;
        }
        const double var = dn > 0.0 ? dM2 / dn : 0.0;    // biased, as InstanceNorm uses
        float *o = (which ? stats2 : stats) + ((int64_t)b * C + c) * 2;
        o[0] = (float)dmean;
        o[1] = (float)(1.0 / sqrt(var + (double)eps));
    }
}

// ---------------------------------------------------------------------------------------------
// forward apply: y = act( (x - mean) rstd  [+ (x2 - mean2) rstd2 | + x2] )
// ---------------------------------------------------------------------------------------------
template <typename T, int MODE2>
__global__ void __launch_bounds__(kNormThreads, SMB_IN_FWD_MINB) in_apply_fwd_kernel(const NormP p) {
    constexpr int V = VecOf<T>::V;
    const int C = p.channels, CV = C / V;
    const RowMap m = row_map(p, CV);
    if (!m.active) return;
    const int b = blockIdx.y;
    const int64_t base = (int64_t)b * p.spatial * C;
    const T *x = reinterpret_cast<const T *>(p.x) + base;
    const T *x2 = MODE2 ? reinterpret_cast<const T *>(p.x2) + base : nullptr;
    T *y = reinterpret_cast<T *>(p.y) + base;
    float mu[V], rs[V], mu2[V], rs2[V];
#pragma unroll
    for (int v = 0; v < V; ++v) {
        const int c = m.cv * V + v;
        mu[v] = p.stats[((int64_t)b * C + c) * 2];
        rs[v] = p.stats[((int64_t)b * C + c) * 2 + 1];
        mu2[v] = 0.f; rs2[v] = 1.f;
        if (MODE2 == 2) {
            mu2[v] = p.stats2[((int64_t)b * C + c) * 2];
            rs2[v] = p.stats2[((int64_t)b * C + c) * 2 + 1];
        }
    }
    constexpr int U = SMB_IN_U_FWD;
    for (int64_t row0 = m.row_lo + m.r; row0 < m.row_hi; row0 += (int64_t)U * m.RB) {
        float a[U][V], b2[U][V];
#pragma unroll
        for (int k = 0; k < U; ++k) {
            const int64_t row = row0 + (int64_t)k * m.RB;
            if (row < m.row_hi) {
                const int64_t ar = SMB_APPLY_ROW(m, row);
                loadv<T, V>(x + ar * C + m.cv * V, a[k]);
                if (MODE2) loadv<T, V>(x2 + ar * C + m.cv * V, b2[k]);
            }
        }
#pragma unroll
        for (int k = 0; k < U; ++k) {
            const int64_t row = row0 + (int64_t)k * m.RB;
            if (row < m.row_hi) {
                float o[V];
#pragma unroll
                for (int v = 0; v < V; ++v) {
                    float t = (a[k][v] - mu[v]) * rs[v];
                    if (MODE2) t += (b2[k][v] - mu2[v]) * rs2[v];
                    o[v] = act_fwd(t, p.act, p.slope);
                }
                storev<T, V>(y + SMB_APPLY_ROW(m, row) * C + m.cv * V, o);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// backward sums: per-CTA  sum g, sum g*xhat1 (, sum g*xhat2)  with g = dy * act'(pre-activation)
// partial layout: [batch][cta][3][C]
// ---------------------------------------------------------------------------------------------
template <typename T, int MODE2>
__global__ void __launch_bounds__(kNormThreads, (MODE2 == 0 ? SMB_IN_BWD_MINB0 : (MODE2 == 1 ? SMB_IN_BWD_MINB1 : SMB_IN_BWD_MINB2))) in_stats_bwd_kernel(const NormP p) {
    constexpr int V = VecOf<T>::V;
    extern __shared__ float sm[];
    const int C = p.channels, CV = C / V;
    const RowMap m = row_map(p, CV);
    const int b = blockIdx.y;
    const int64_t base = (int64_t)b * p.spatial * C;
    const T *x = reinterpret_cast<const T *>(p.x) + base;
    const T *x2 = MODE2 ? reinterpret_cast<const T *>(p.x2) + base : nullptr;
    const T *dy = reinterpret_cast<const T *>(p.dy) + base;
    float mu[V], rs[V], mu2[V], rs2[V], sg[V], sgx[V], sgx2[V];
#pragma unroll
    for (int v = 0; v < V; ++v) {
        const int c = m.cv * V + v;
        mu[v] = p.stats[((int64_t)b * C + c) * 2];
        rs[v] = p.stats[((int64_t)b * C + c) * 2 + 1];
        mu2[v] = 0.f; rs2[v] = 1.f;
        if (MODE2 == 2) {
            mu2[v] = p.stats2[((int64_t)b * C + c) * 2];
            rs2[v] = p.stats2[((int64_t)b * C + c) * 2 + 1];
        }
        sg[v] = sgx[v] = sgx2[v] = 0.f;
    }
    if (m.active) {
        constexpr int U = MODE2 == 0 ? SMB_IN_U_BWD0 : SMB_IN_U_BWD2;
        for (int64_t row0 = m.row_lo + m.r; row0 < m.row_hi; row0 += (int64_t)U * m.RB) {
            float a[U][V], a2[U][V], g[U][V];
#pragma unroll
            for (int k = 0; k < U; ++k) {
                const int64_t row = row0 + (int64_t)k * m.RB;
                if (row < m.row_hi) {
                    const int64_t sr = SMB_STATS_ROW(m, row);
                    loadv<T, V>(x + sr * C + m.cv * V, a[k]);
                    loadv<T, V>(dy + sr * C + m.cv * V, g[k]);
                    if (MODE2) loadv<T, V>(x2 + sr * C + m.cv * V, a2[k]);
                }
            }
#pragma unroll
            for (int k = 0; k < U; ++k) {
                const int64_t row = row0 + (int64_t)k * m.RB;
                if (row < m.row_hi) {
#pragma unroll
                    for (int v = 0; v < V; ++v) {
                        const float xh = (a[k][v] - mu[v]) * rs[v];
                        float pre = xh, xh2 = 0.f;
                        if (MODE2) { xh2 = (a2[k][v] - mu2[v]) * rs2[v]; pre += xh2; }
                        const float gg = act_bwd(g[k][v], pre, p.act, p.slope);
                        sg[v] += gg;
                        sgx[v] = fmaf(gg, xh, sgx[v]);
                        if (MODE2 == 2) sgx2[v] = fmaf(gg, xh2, sgx2[v]);
                    }
                }
            }
        }
    }
    const int RB = m.RB;
    float *A = sm, *Bq = sm + RB * C, *Cq = sm + 2 * RB * C;
    if (m.active) {
#pragma unroll
        for (int v = 0; v < V; ++v) {
            A[m.r * C + m.cv * V + v] = sg[v];
            Bq[m.r * C + m.cv * V + v] = sgx[v];
            Cq[m.r * C + m.cv * V + v] = sgx2[v];
        }
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += kNormThreads) {
        float a = 0.f, q = 0.f, q2 = 0.f;
        for (int r = 0; r < RB; ++r) { a += A[r * C + c]; q += Bq[r * C + c]; q2 += Cq[r * C + c]; }
        float *o = p.partial + (((int64_t)b * gridDim.x + blockIdx.x) * 3) * C + c;
        o[0] = a; o[C] = q; o[2 * C] = q2;
    }
}

// sums[b][c] = (mean g, mean g*xhat1, mean g*xhat2); same 32 x 8 mapping as the forward finalize
__global__ void __launch_bounds__(1024) in_finalize_bwd_kernel(const float *__restrict__ partial, float *__restrict__ sums, int batch,
                                                              int C, int n_cta, float inv_n) {
    __shared__ float sa[32][33], sq[32][33], sq2[32][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + tx, b = blockIdx.y;
    float a = 0.f, q = 0.f, q2 = 0.f;
    if (c < C) {
        const float *pp = partial + ((int64_t)b * n_cta * 3) * C + c;
        for (int k = ty; k < n_cta; k += 32) {
            a += pp[(int64_t)k * 3 * C]; q += pp[(int64_t)k * 3 * C + C]; q2 += pp[(int64_t)k * 3 * C + 2 * C];
        }
    }
    sa[ty][tx] = a; sq[ty][tx] = q; sq2[ty][tx] = q2;
    __syncthreads();
    if (ty == 0 && c < C) {
        double da = 0.0, dq = 0.0, dq2 = 0.0;
        for (int g = 0; g < 32; ++g) { da += sa[g][tx]; dq += sq[g][tx]; dq2 += sq2[g][tx]; }
        float *o = sums + ((int64_t)b * C + c) * 3;
        o[0] = (float)(da * inv_n); o[1] = (float)(dq * inv_n); o[2] = (float)(dq2 * inv_n);
    }
}

// backward apply: dx = rstd (g - mean g - xhat mean(g xhat)) ;  dx2 likewise (mode 2) or dx2 = g (mode 1)
template <typename T, int MODE2>
__global__ void __launch_bounds__(kNormThreads, (MODE2 == 0 ? SMB_IN_BWD_MINB0 : (MODE2 == 1 ? SMB_IN_BWD_MINB1 : SMB_IN_BWD_MINB2))) in_apply_bwd_kernel(const NormP p) {
    constexpr int V = VecOf<T>::V;
    const int C = p.channels, CV = C / V;
    const RowMap m = row_map(p, CV);
    if (!m.active) return;
    const int b = blockIdx.y;
    const int64_t base = (int64_t)b * p.spatial * C;
    const T *x = reinterpret_cast<const T *>(p.x) + base;
    const T *x2 = MODE2 ? reinterpret_cast<const T *>(p.x2) + base : nullptr;
    const T *dy = reinterpret_cast<const T *>(p.dy) + base;
    T *dx = reinterpret_cast<T *>(p.dx) + base;
    T *dx2 = (MODE2 && p.dx2) ? reinterpret_cast<T *>(p.dx2) + base : nullptr;
    float mu[V], rs[V], mu2[V], rs2[V], mg[V], mgx[V], mgx2[V];
#pragma unroll
    for (int v = 0; v < V; ++v) {
        const int c = m.cv * V + v;
        mu[v] = p.stats[((int64_t)b * C + c) * 2];
        rs[v] = p.stats[((int64_t)b * C + c) * 2 + 1];
        mu2[v] = 0.f; rs2[v] = 1.f;
        if (MODE2 == 2) {
            mu2[v] = p.stats2[((int64_t)b * C + c) * 2];
            rs2[v] = p.stats2[((int64_t)b * C + c) * 2 + 1];
        }
        mg[v] = p.sums[((int64_t)b * C + c) * 3];
        mgx[v] = p.sums[((int64_t)b * C + c) * 3 + 1];
        mgx2[v] = p.sums[((int64_t)b * C + c) * 3 + 2];
    }
    constexpr int U = MODE2 == 0 ? SMB_IN_U_BWD0 : SMB_IN_U_BWD2;
    for (int64_t row0 = m.row_lo + m.r; row0 < m.row_hi; row0 += (int64_t)U * m.RB) {
        float a[U][V], a2[U][V], g[U][V];
#pragma unroll
        for (int k = 0; k < U; ++k) {
            const int64_t row = row0 + (int64_t)k * m.RB;
            if (row < m.row_hi) {
                const int64_t ar = SMB_APPLY_ROW(m, row);
                loadv<T, V>(x + ar * C + m.cv * V, a[k]);
                loadv<T, V>(dy + ar * C + m.cv * V, g[k]);
                if (MODE2) loadv<T, V>(x2 + ar * C + m.cv * V, a2[k]);
            }
        }
#pragma unroll
        for (int k = 0; k < U; ++k) {
            const int64_t row = row0 + (int64_t)k * m.RB;
            if (row < m.row_hi) {
                float o[V], o2[V];
#pragma unroll
                for (int v = 0; v < V; ++v) {
                    const float xh = (a[k][v] - mu[v]) * rs[v];
                    float pre = xh, xh2 = 0.f;
                    if (MODE2) { xh2 = (a2[k][v] - mu2[v]) * rs2[v]; pre += xh2; }
                    const float gg = act_bwd(g[k][v], pre, p.act, p.slope);
                    o[v] = rs[v] * (gg - mg[v] - xh * mgx[v]);
                    o2[v] = MODE2 == 2 ? rs2[v] * (gg - mg[v] - xh2 * mgx2[v]) : gg;
                }
                storev<T, V>(dx + SMB_APPLY_ROW(m, row) * C + m.cv * V, o);
                if (dx2) storev<T, V>(dx2 + SMB_APPLY_ROW(m, row) * C + m.cv * V, o2);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
template <typename T>
static cudaError_t norm_fwd_t(NormP p, cudaStream_t st) {
    constexpr int V = VecOf<T>::V;
    const int CV = p.channels / V, RB = kNormThreads / CV;
    dim3 grid(p.n_cta, p.batch);
    const bool two = p.mode2 == 2;
    const size_t smem = (size_t)RB * p.channels * (two ? 4 : 2) * sizeof(float);
    if (two) in_stats_fwd_kernel<T, true><<<grid, kNormThreads, smem, st>>>(p);
    else in_stats_fwd_kernel<T, false><<<grid, kNormThreads, smem, st>>>(p);
    count_launch();
    dim3 fg((p.channels + 31) / 32, p.batch, two ? 2 : 1);
    in_finalize_fwd_kernel<<<fg, 1024, 0, st>>>(p.partial, p.stats, p.stats2, p.batch, p.channels, p.n_cta, p.eps);
    count_launch();
    if (p.mode2 == 0) in_apply_fwd_kernel<T, 0><<<grid, kNormThreads, 0, st>>>(p);
    else if (p.mode2 == 1) in_apply_fwd_kernel<T, 1><<<grid, kNormThreads, 0, st>>>(p);
    else in_apply_fwd_kernel<T, 2><<<grid, kNormThreads, 0, st>>>(p);
    count_launch();
    return cudaGetLastError();
}

template <typename T>
static cudaError_t norm_bwd_t(NormP p, cudaStream_t st) {
    constexpr int V = VecOf<T>::V;
    const int CV = p.channels / V, RB = kNormThreads / CV;
    dim3 grid(p.n_cta, p.batch);
    const size_t smem = (size_t)RB * p.channels * 3 * sizeof(float);
    if (p.mode2 == 0) in_stats_bwd_kernel<T, 0><<<grid, kNormThreads, smem, st>>>(p);
    else if (p.mode2 == 1) in_stats_bwd_kernel<T, 1><<<grid, kNormThreads, smem, st>>>(p);
    else in_stats_bwd_kernel<T, 2><<<grid, kNormThreads, smem, st>>>(p);
    count_launch();
    dim3 fg((p.channels + 31) / 32, p.batch);
    in_finalize_bwd_kernel<<<fg, 1024, 0, st>>>(p.partial, p.sums, p.batch, p.channels, p.n_cta, (float)(1.0 / (double)p.spatial));
    count_launch();
    if (p.mode2 == 0) in_apply_bwd_kernel<T, 0><<<grid, kNormThreads, 0, st>>>(p);
    else if (p.mode2 == 1) in_apply_bwd_kernel<T, 1><<<grid, kNormThreads, 0, st>>>(p);
    else in_apply_bwd_kernel<T, 2><<<grid, kNormThreads, 0, st>>>(p);
    count_launch();
    return cudaGetLastError();
}

cudaError_t instnorm_dispatch(const NormP &p, int dtype, bool bwd, cudaStream_t st) {
    switch (dtype) {
        case 0: return bwd ? norm_bwd_t<float>(p, st) : norm_fwd_t<float>(p, st);
        case 1: return bwd ? norm_bwd_t<__half>(p, st) : norm_fwd_t<__half>(p, st);
        default: return bwd ? norm_bwd_t<__nv_bfloat16>(p, st) : norm_fwd_t<__nv_bfloat16>(p, st);
    }
}

}  // namespace smb
