// Depthwise causal conv1d (+SiLU) forward / backward for sm_90a, and the inter-slice sequence permutation.
//
// Restates causal_conv1d_fwd_kernel / causal_conv1d_bwd_kernel (causal-conv1d/csrc/causal_conv1d_fwd.cu:39-130,
// causal_conv1d_bwd.cu:46-240).  The reference runs one CTA per (batch, channel) that walks L serially in
// 512..1024-element chunks; here the grid also spans L (each thread owns a run of 8 scan positions, the
// 3-element halo comes from the neighbouring lane by shuffle), so a 96-channel x 262144-token call fills
// the chip.  Any width 2..4 is handled as width 4 with leading zero taps.
#include <cstdlib>

#include "conv_internal.h"

namespace smb {

#ifndef SMB_CONV_THREADS
#define SMB_CONV_THREADS 128
#endif
constexpr int kConvThreads = SMB_CONV_THREADS;

__device__ __forceinline__ float silu_grad(float o) {   // d/do [o * sigmoid(o)]
    const float s = sigmoidf(o);
    return s * (1.f + o * (1.f - s));
}

template <typename T>
__global__ void __launch_bounds__(kConvThreads) conv1d_fwd_kernel(const ConvP p) {
    const int lane = threadIdx.x & 31;
    const int d = blockIdx.y, b = blockIdx.z;
    const int j = (blockIdx.x * kConvThreads + threadIdx.x) * kRun;       // first scan position of this run
    const int L = p.L;
    const T *xr = reinterpret_cast<const T *>(p.x) + b * p.x_bs + (int64_t)d * p.x_ds;
    T *outr = reinterpret_cast<T *>(p.out) + b * p.out_bs + (int64_t)d * p.out_ds;

    float w4[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int kk = k - (4 - p.width);
        w4[k] = kk >= 0 ? p.weight[(int64_t)d * p.w_ds + (int64_t)kk * p.w_ws] : 0.f;
    }
    const float bias = p.bias ? p.bias[d] : 0.f;

    float x[kRun + 3];                                   // x[3 + i] = position j + i ; x[0..2] = halo
    load_run8<T>(xr, j, L, p.reverse, x + 3);
    // halo from the previous lane's last three positions; lane 0 reads them from memory
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float up = __shfl_up_sync(0xffffffffu, x[3 + kRun - 3 + k], 1);
        float v = up;
        if (lane == 0) {
            const int jj = j - 3 + k;
            v = (jj >= 0 && jj < L) ? to_f32<T>(xr[pos_to_tok(jj, L, p.reverse)]) : 0.f;
        }
        x[k] = v;
    }
    if (j >= L) return;
    float o[kRun];
#pragma unroll
    for (int i = 0; i < kRun; ++i) {
        float acc = bias;
#pragma unroll
        for (int k = 0; k < 4; ++k) acc = fmaf(w4[k], x[i + k], acc);
        o[i] = p.silu ? acc * sigmoidf(acc) : acc;
    }
    store_run8<T>(outr, j, L, p.reverse, o);
}

template <typename T>
__global__ void __launch_bounds__(kConvThreads) conv1d_bwd_kernel(const ConvP p) {
    __shared__ float red[kConvThreads / 32][5];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int d = blockIdx.y, b = blockIdx.z;
    const int j = (blockIdx.x * kConvThreads + threadIdx.x) * kRun;
    const int L = p.L;
    const T *xr = reinterpret_cast<const T *>(p.x) + b * p.x_bs + (int64_t)d * p.x_ds;
    const T *gr = reinterpret_cast<const T *>(p.dout) + b * p.dout_bs + (int64_t)d * p.dout_ds;
    T *dxr = reinterpret_cast<T *>(p.dx) + b * p.dx_bs + (int64_t)d * p.dx_ds;

    float w4[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int kk = k - (4 - p.width);
        w4[k] = kk >= 0 ? p.weight[(int64_t)d * p.w_ds + (int64_t)kk * p.w_ws] : 0.f;
    }
    const float bias = p.bias ? p.bias[d] : 0.f;

    float x[kRun + 3], gh[kRun + 3];                     // gh[i] = g-hat at position j + i, i in [0, 11)
    load_run8<T>(xr, j, L, p.reverse, x + 3);
    load_run8<T>(gr, j, L, p.reverse, gh);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float up = __shfl_up_sync(0xffffffffu, x[3 + kRun - 3 + k], 1);
        float v = up;
        if (lane == 0) {
            const int jj = j - 3 + k;
            v = (jj >= 0 && jj < L) ? to_f32<T>(xr[pos_to_tok(jj, L, p.reverse)]) : 0.f;
        }
        x[k] = v;
    }
    // g-hat = dout * silu'(pre-activation)  (causal_conv1d_bwd.cu:153-164); positions >= L have dout == 0
    if (p.silu) {
#pragma unroll
        for (int i = 0; i < kRun; ++i) {
            float acc = bias;
#pragma unroll
            for (int k = 0; k < 4; ++k) acc = fmaf(w4[k], x[i + k], acc);
            gh[i] *= silu_grad(acc);
        }
    }
    // right halo: g-hat of the next lane's first three positions; lane 31 recomputes them
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float dn = __shfl_down_sync(0xffffffffu, gh[k], 1);
        gh[kRun + k] = dn;
    }
    if (lane == 31) {
        float xn[3], gn[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const int jj = j + kRun + k;
            const bool ok = jj < L;
            xn[k] = ok ? to_f32<T>(xr[pos_to_tok(jj, L, p.reverse)]) : 0.f;
            gn[k] = ok ? to_f32<T>(gr[pos_to_tok(jj, L, p.reverse)]) : 0.f;
        }
        // window for position j+8+k is x at j+5+k .. j+8+k = {x[8+k], x[9+k], x[10+k] (own), xn[..]}
        const float xe[6] = {x[kRun], x[kRun + 1], x[kRun + 2], xn[0], xn[1], xn[2]};   // positions j+5 .. j+10
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            float gv = gn[k];
            if (p.silu) {
                float acc = bias;
#pragma unroll
                for (int t = 0; t < 4; ++t) acc = fmaf(w4[t], xe[k + t], acc);
                gv *= silu_grad(acc);
            }
            gh[kRun + k] = gv;
        }
    }
    // dx[j+i] = sum_k w4[k] * ghat[j+i + (3-k)]   (causal_conv1d_bwd.cu:197-204)
    float dxv[kRun];
    float dw[4] = {0.f, 0.f, 0.f, 0.f}, db = 0.f;
#pragma unroll
    for (int i = 0; i < kRun; ++i) {
        float acc = 0.f;
#pragma unroll
        for (int k = 0; k < 4; ++k) acc = fmaf(w4[k], gh[i + 3 - k], acc);
        dxv[i] = acc;
        // causal_conv1d_bwd.cu:216-222; a tap over the zero padding before position 0 is skipped rather than multiplied by 0,
        // so a non-finite g-hat at the first positions reaches only the taps that read input, as in the reference
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float t = x[i + k] * gh[i];
            dw[k] += (j + i + k >= 3) ? t : 0.f;
        }
        db += gh[i];
    }
    store_run8<T>(dxr, j, L, p.reverse, dxv);
    // block reduction of dW / dbias, then one fp32 atomic per block (causal_conv1d_bwd.cu:225-239)
#pragma unroll
    for (int k = 0; k < 4; ++k) dw[k] = warp_sum(dw[k]);
    db = warp_sum(db);
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < 4; ++k) red[warp][k] = dw[k];
        red[warp][4] = db;
    }
    __syncthreads();
    if (threadIdx.x < 5) {
        float s = 0.f;
#pragma unroll
        for (int w2 = 0; w2 < kConvThreads / 32; ++w2) s += red[w2][threadIdx.x];
        if (threadIdx.x < 4) {
            const int kk = threadIdx.x - (4 - p.width);
            if (kk >= 0) atomicAdd(p.dweight + (int64_t)d * p.width + kk, s);
        } else if (p.dbias) {
            atomicAdd(p.dbias + d, s);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// inter-slice permutation: per row, view L as (ns, Lp) and transpose to (Lp, ns) (or back)
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) seq_permute_kernel(const T *__restrict__ src, T *__restrict__ dst, int64_t src_rs,
                                                          int64_t dst_rs, int n_src_rows, int n_src_cols, int accumulate) {
    // src row r (of the matrix view): [n_src_rows][n_src_cols] -> dst [n_src_cols][n_src_rows]
    __shared__ float tile[32][33];
    const int row = blockIdx.z;
    const T *s = src + (int64_t)row * src_rs;
    T *o = dst + (int64_t)row * dst_rs;
    const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 32 x 8
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int r = r0 + ty + 8 * k, c = c0 + tx;
        if (r < n_src_rows && c < n_src_cols) tile[ty + 8 * k][tx] = to_f32<T>(s[(int64_t)r * n_src_cols + c]);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int c = c0 + ty + 8 * k, r = r0 + tx;               // dst[c][r]
        if (r < n_src_rows && c < n_src_cols) {
            float v = tile[tx][ty + 8 * k];
            T *q = o + (int64_t)c * n_src_rows + r;
            if (accumulate) v += to_f32<T>(*q);
            *q = from_f32<T>(v);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
template <typename T>
static cudaError_t conv_launch_t(const ConvP &p, bool bwd, cudaStream_t st) {
    const int per_block = kConvThreads * kRun;
    dim3 grid((p.L + per_block - 1) / per_block, p.dim, p.batch);
    if (!bwd) conv1d_fwd_kernel<T><<<grid, kConvThreads, 0, st>>>(p);
    else conv1d_bwd_kernel<T><<<grid, kConvThreads, 0, st>>>(p);
    count_launch();
    return cudaGetLastError();
}

cudaError_t conv1d_dispatch(const ConvP &p, int dtype, bool bwd, cudaStream_t st) {
    {   // 16-bit activations: 16 positions per thread (conv1d_v2.cu); SMB_CONV_V2=0 keeps 8 per thread (A/B switch, read per call)
        const char *v2 = getenv("SMB_CONV_V2");
        if (dtype != 0 && !(v2 && v2[0] == '0')) return conv1d_v2_dispatch(p, dtype, bwd, st);
    }
    switch (dtype) {
        case 0: return conv_launch_t<float>(p, bwd, st);
        case 1: return conv_launch_t<__half>(p, bwd, st);
        default: return conv_launch_t<__nv_bfloat16>(p, bwd, st);
    }
}

template <typename T>
static cudaError_t permute_launch_t(const void *src, void *dst, int64_t src_rs, int64_t dst_rs, int rows, int L, int ns,
                                    int inverse, int accumulate, cudaStream_t st) {
    // to_slices: src viewed (ns, Lp) -> dst (Lp, ns);  from_slices: src viewed (Lp, ns) -> dst (ns, Lp)
    const int Lp = L / ns;
    const int nr = inverse ? Lp : ns, nc = inverse ? ns : Lp;
    dim3 grid((nc + 31) / 32, (nr + 31) / 32, rows);
    seq_permute_kernel<T><<<grid, 256, 0, st>>>(reinterpret_cast<const T *>(src), reinterpret_cast<T *>(dst), src_rs, dst_rs,
                                                nr, nc, accumulate); count_launch();
    return cudaGetLastError();
}

cudaError_t seq_permute_dispatch(const void *src, void *dst, int64_t src_rs, int64_t dst_rs, int rows, int L, int ns,
                                 int inverse, int accumulate, int dtype, cudaStream_t st) {
    {   // 16-bit activations: 4-byte accesses (conv1d_v2.cu); SMB_PERMUTE_V2=0 keeps the 2-byte kernel (A/B switch, read per call)
        const char *v2 = getenv("SMB_PERMUTE_V2");
        if (dtype != 0 && !(v2 && v2[0] == '0')) {
            const cudaError_t e = seq_permute_v2_dispatch(src, dst, src_rs, dst_rs, rows, L, ns, inverse, accumulate, dtype, st);
            if (e != cudaErrorNotSupported) return e;
        }
    }
    switch (dtype) {
        case 0: return permute_launch_t<float>(src, dst, src_rs, dst_rs, rows, L, ns, inverse, accumulate, st);
        case 1: return permute_launch_t<__half>(src, dst, src_rs, dst_rs, rows, L, ns, inverse, accumulate, st);
        default: return permute_launch_t<__nv_bfloat16>(src, dst, src_rs, dst_rs, rows, L, ns, inverse, accumulate, st);
    }
}

}  // namespace smb
