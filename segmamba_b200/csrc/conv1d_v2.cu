// Depthwise causal conv1d forward / backward with 16 scan positions per thread for 16-bit activations
// (opt-in: SMB_CONV_V2=1).  Same arithmetic as conv1d.cu.  Why: with 8 positions per thread a bf16 / fp16 thread moves only
// 16 bytes each way, half of what the fp32 instantiation (32 bytes per thread) keeps in flight; 16 positions give the 16-bit types the same bytes in flight per thread.
#include "conv_internal.h"

#include <cstdint>

namespace smb {

constexpr int kConv2Threads = 128;
constexpr int kRun2 = 16;

__device__ __forceinline__ float silu_grad2(float o) {   // d/do [o * sigmoid(o)]
    const float s = sigmoidf(o);
    return s * (1.f + o * (1.f - s));
}

template <typename T> __device__ __forceinline__ void load_run16(const T *row, int j, int L, bool reverse, float v[kRun2]) {
    load_run8<T>(row, j, L, reverse, v);
    load_run8<T>(row, j + kRun, L, reverse, v + kRun);
}
template <typename T> __device__ __forceinline__ void store_run16(T *row, int j, int L, bool reverse, const float v[kRun2]) {
    store_run8<T>(row, j, L, reverse, v);
    store_run8<T>(row, j + kRun, L, reverse, v + kRun);
}

template <typename T>
__global__ void __launch_bounds__(kConv2Threads) conv1d_fwd16_kernel(const ConvP p) {
    const int lane = threadIdx.x & 31;
    const int d = blockIdx.y, b = blockIdx.z;
    const int j = (blockIdx.x * kConv2Threads + threadIdx.x) * kRun2;      // first scan position of this run
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

    float x[kRun2 + 3];                                  // x[3 + i] = position j + i ; x[0..2] = halo
    load_run16<T>(xr, j, L, p.reverse, x + 3);
#pragma unroll
    for (int k = 0; k < 3; ++k) {                        // halo: previous lane's last three positions; lane 0 reads memory
        const float up = __shfl_up_sync(0xffffffffu, x[3 + kRun2 - 3 + k], 1);
        float v = up;
        if (lane == 0) {
            const int jj = j - 3 + k;
            v = (jj >= 0 && jj < L) ? to_f32<T>(xr[pos_to_tok(jj, L, p.reverse)]) : 0.f;
        }
        x[k] = v;
    }
    if (j >= L) return;
    float o[kRun2];
#pragma unroll
    for (int i = 0; i < kRun2; ++i) {
        float acc = bias;
#pragma unroll
        for (int k = 0; k < 4; ++k) acc = fmaf(w4[k], x[i + k], acc);
        o[i] = p.silu ? acc * sigmoidf(acc) : acc;
    }
    store_run16<T>(outr, j, L, p.reverse, o);
}

template <typename T>
__global__ void __launch_bounds__(kConv2Threads) conv1d_bwd16_kernel(const ConvP p) {
    __shared__ float red[kConv2Threads / 32][5];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int d = blockIdx.y, b = blockIdx.z;
    const int j = (blockIdx.x * kConv2Threads + threadIdx.x) * kRun2;
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

    float x[kRun2 + 3], gh[kRun2 + 3];                   // gh[i] = g-hat at position j + i
    load_run16<T>(xr, j, L, p.reverse, x + 3);
    load_run16<T>(gr, j, L, p.reverse, gh);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float up = __shfl_up_sync(0xffffffffu, x[3 + kRun2 - 3 + k], 1);
        float v = up;
        if (lane == 0) {
            const int jj = j - 3 + k;
            v = (jj >= 0 && jj < L) ? to_f32<T>(xr[pos_to_tok(jj, L, p.reverse)]) : 0.f;
        }
        x[k] = v;
    }
    if (p.silu) {                                        // g-hat = dout * silu'(pre-activation); positions >= L have dout == 0
#pragma unroll
        for (int i = 0; i < kRun2; ++i) {
            float acc = bias;
#pragma unroll
            for (int k = 0; k < 4; ++k) acc = fmaf(w4[k], x[i + k], acc);
            gh[i] *= silu_grad2(acc);
        }
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {                        // right halo: next lane's first three g-hats; lane 31 recomputes them
        const float dn = __shfl_down_sync(0xffffffffu, gh[k], 1);
        gh[kRun2 + k] = dn;
    }
    if (lane == 31) {
        float xn[3], gn[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const int jj = j + kRun2 + k;
            const bool ok = jj < L;
            xn[k] = ok ? to_f32<T>(xr[pos_to_tok(jj, L, p.reverse)]) : 0.f;
            gn[k] = ok ? to_f32<T>(gr[pos_to_tok(jj, L, p.reverse)]) : 0.f;
        }
        // window of position j+R+k is x at j+R+k-3 .. j+R+k = {own x[R], x[R+1], x[R+2] (positions j+R-3..j+R-1), xn[..]}
        const float xe[6] = {x[kRun2], x[kRun2 + 1], x[kRun2 + 2], xn[0], xn[1], xn[2]};
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            float gv = gn[k];
            if (p.silu) {
                float acc = bias;
#pragma unroll
                for (int t = 0; t < 4; ++t) acc = fmaf(w4[t], xe[k + t], acc);
                gv *= silu_grad2(acc);
            }
            gh[kRun2 + k] = gv;
        }
    }
    float dxv[kRun2];
    float dw[4] = {0.f, 0.f, 0.f, 0.f}, db = 0.f;
#pragma unroll
    for (int i = 0; i < kRun2; ++i) {
        float acc = 0.f;
#pragma unroll
        for (int k = 0; k < 4; ++k) acc = fmaf(w4[k], gh[i + 3 - k], acc);     // dx[j+i] = sum_k w4[k] ghat[j+i+3-k]
        dxv[i] = acc;
        // x[i + k] is position j + i + k - 3: a tap over the zero padding before position 0 is selected away, not multiplied
        // by 0, so a non-finite g-hat at the first positions reaches only the taps that read input, as in the reference
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float t = x[i + k] * gh[i];
            dw[k] += (j + i + k >= 3) ? t : 0.f;
        }
        db += gh[i];
    }
    store_run16<T>(dxr, j, L, p.reverse, dxv);
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
        for (int w2 = 0; w2 < kConv2Threads / 32; ++w2) s += red[w2][threadIdx.x];
        if (threadIdx.x < 4) {
            const int kk = threadIdx.x - (4 - p.width);
            if (kk >= 0) atomicAdd(p.dweight + (int64_t)d * p.width + kk, s);
        } else if (p.dbias) {
            atomicAdd(p.dbias + d, s);
        }
    }
}

template <typename T>
static cudaError_t conv2_launch_t(const ConvP &p, bool bwd, cudaStream_t st) {
    const int per_block = kConv2Threads * kRun2;
    dim3 grid((p.L + per_block - 1) / per_block, p.dim, p.batch);
    if (!bwd) conv1d_fwd16_kernel<T><<<grid, kConv2Threads, 0, st>>>(p);
    else conv1d_bwd16_kernel<T><<<grid, kConv2Threads, 0, st>>>(p);
    count_launch();
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// inter-slice permutation for 16-bit activations with 4-byte accesses (opt-in: SMB_PERMUTE_V2=1).
// The default kernel (conv1d.cu) moves one 2-byte element per thread and access: a warp touches 64 bytes per row segment.
// Here a CTA transposes a 64 x 64 tile held as
// 64 x 32 words: every global access is a 128-byte row segment of 32 element pairs; the pair that leaves along the
// destination row is assembled from the same half of two vertically adjacent words (one PRMT).
// Requires even n_src_rows / n_src_cols and 4-byte aligned rows; the dispatcher falls back to the default kernel otherwise.
// ---------------------------------------------------------------------------------------------
template <typename T> __device__ __forceinline__ unsigned add_pair(unsigned a, unsigned b);
template <> __device__ __forceinline__ unsigned add_pair<__nv_bfloat16>(unsigned a, unsigned b) {
    const float lo = __uint_as_float(a << 16) + __uint_as_float(b << 16);
    const float hi = __uint_as_float(a & 0xffff0000u) + __uint_as_float(b & 0xffff0000u);
    const __nv_bfloat162 r = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<const unsigned *>(&r);
}
template <> __device__ __forceinline__ unsigned add_pair<__half>(unsigned a, unsigned b) {
    const float2 fa = __half22float2(*reinterpret_cast<const __half2 *>(&a)), fb = __half22float2(*reinterpret_cast<const __half2 *>(&b));
    const __half2 r = __floats2half2_rn(fa.x + fb.x, fa.y + fb.y);
    return *reinterpret_cast<const unsigned *>(&r);
}

template <typename T>
__global__ void __launch_bounds__(256) seq_permute2_kernel(const T *__restrict__ src, T *__restrict__ dst, int64_t src_rs,
                                                           int64_t dst_rs, int n_src_rows, int n_src_cols, int accumulate) {
    __shared__ unsigned tile[64][33];                      // tile[r][w]: elements (r, 2w) and (r, 2w + 1) of the source tile
    const int row = blockIdx.z;
    const T *s = src + (int64_t)row * src_rs;
    T *o = dst + (int64_t)row * dst_rs;
    const int c0 = blockIdx.x * 64, r0 = blockIdx.y * 64;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 32 x 8
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int r = r0 + ty + 8 * k, c = c0 + 2 * tx;
        unsigned w = 0u;
        if (r < n_src_rows && c < n_src_cols) w = *reinterpret_cast<const unsigned *>(s + (int64_t)r * n_src_cols + c);
        tile[ty + 8 * k][tx] = w;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int cl = ty + 8 * k;                          // destination row inside the tile = source column
        const int c = c0 + cl, r = r0 + 2 * tx;             // dst[c][r], dst[c][r + 1]
        if (r < n_src_rows && c < n_src_cols) {
            const unsigned w0 = tile[2 * tx][cl >> 1], w1 = tile[2 * tx + 1][cl >> 1];
            unsigned v = (cl & 1) ? ((w0 >> 16) | (w1 & 0xffff0000u)) : ((w0 & 0xffffu) | (w1 << 16));
            unsigned *q = reinterpret_cast<unsigned *>(o + (int64_t)c * n_src_rows + r);
            if (accumulate) v = add_pair<T>(v, *q);
            *q = v;
        }
    }
}

template <typename T>
static cudaError_t permute2_launch_t(const void *src, void *dst, int64_t src_rs, int64_t dst_rs, int rows, int nr, int nc,
                                     int accumulate, cudaStream_t st) {
    dim3 grid((nc + 63) / 64, (nr + 63) / 64, rows);
    seq_permute2_kernel<T><<<grid, 256, 0, st>>>(reinterpret_cast<const T *>(src), reinterpret_cast<T *>(dst), src_rs, dst_rs, nr, nc,
                                                 accumulate); count_launch();
    return cudaGetLastError();
}

// returns cudaErrorNotSupported when the shape / alignment does not allow 4-byte accesses (caller then uses the default kernel)
cudaError_t seq_permute_v2_dispatch(const void *src, void *dst, int64_t src_rs, int64_t dst_rs, int rows, int L, int ns, int inverse,
                                    int accumulate, int dtype, cudaStream_t st) {
    const int Lp = L / ns;
    const int nr = inverse ? Lp : ns, nc = inverse ? ns : Lp;
    if (dtype == 0 || (nr & 1) || (nc & 1) || (src_rs & 1) || (dst_rs & 1) ||
        ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 3))
        return cudaErrorNotSupported;
    if (dtype == 1) return permute2_launch_t<__half>(src, dst, src_rs, dst_rs, rows, nr, nc, accumulate, st);
    return permute2_launch_t<__nv_bfloat16>(src, dst, src_rs, dst_rs, rows, nr, nc, accumulate, st);
}

cudaError_t conv1d_v2_dispatch(const ConvP &p, int dtype, bool bwd, cudaStream_t st) {
    if (dtype == 1) return conv2_launch_t<__half>(p, bwd, st);
    return conv2_launch_t<__nv_bfloat16>(p, bwd, st);
}

}  // namespace smb
