// Fused LayerNorm over the channel axis of the (tokens, C) matrix that feeds every Mamba mixer, forward and backward,
// for sm_90a.
//
// Replaces nn.LayerNorm(dim) in MambaLayer.forward (model_segmamba/segmamba.py:54,70): under autocast the reference runs
// it as ATen fp32 kernels (bf16 -> fp32 input cast, vectorized_layer_norm_kernel, fp32 -> bf16 cast before in_proj; in
// backward layer_norm_grad_input + GammaBetaBackward).
// The op is a pure HBM stream:
//   forward : read x, write y                      2 * s * rows * C bytes
//   backward: read x, dy, write dx (+ C floats)    3 * s * rows * C bytes   (statistics are recomputed, nothing is saved)
// Mapping: a row (token) is C/V 16-byte vectors; LPR = the next power of two >= C/V lanes (at most 32) own one row, each
// lane VPL vectors of it, so a warp covers 32/LPR consecutive rows with fully coalesced 16-byte accesses.  Row statistics
// are two-pass in registers (mean, then centred variance) with xor-shuffles inside the LPR group; gamma / beta and the
// per-channel gradient accumulators live in registers for the whole kernel.  dgamma / dbeta: lane accumulators ->
// shuffle-reduce over the warp's row groups -> shared-memory reduce over the CTA's warps -> one fp32 atomic per channel
// and CTA.
#include "norm_internal.h"

namespace smb {

constexpr int kLnThreads = 256;
constexpr int kLnWarps = kLnThreads / 32;


__device__ __forceinline__ float group_sum(float v, int lpr) {
    for (int o = lpr >> 1; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

struct LnMap {
    int lpr, rows_per_warp, gl, sub;     // lanes per row, rows per warp, lane within the row group, row group within the warp
    int64_t warp_row0, warp_stride;
};
__device__ __forceinline__ LnMap ln_map(int lpr) {
    LnMap m;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    m.lpr = lpr;
    m.rows_per_warp = 32 / lpr;
    m.gl = lane & (lpr - 1);
    m.sub = lane / lpr;
    m.warp_row0 = ((int64_t)blockIdx.x * kLnWarps + warp) * m.rows_per_warp;
    m.warp_stride = (int64_t)gridDim.x * kLnWarps * m.rows_per_warp;
    return m;
}

template <typename T, int VPL>
__global__ void __launch_bounds__(kLnThreads) ln_fwd_kernel(const LnP p, int lpr) {
    constexpr int V = VecOf<T>::V;
    const int CV = p.C / V;
    const LnMap m = ln_map(lpr);
    const T *x = reinterpret_cast<const T *>(p.x);
    T *y = reinterpret_cast<T *>(p.y);
    const float invC = 1.f / (float)p.C;
    float ga[VPL][V], be[VPL][V];
#pragma unroll
    for (int k = 0; k < VPL; ++k) {
        const int cv = m.gl + k * lpr;
#pragma unroll
        for (int v = 0; v < V; ++v) {
            ga[k][v] = cv < CV ? p.gamma[cv * V + v] : 0.f;
            be[k][v] = cv < CV && p.beta ? p.beta[cv * V + v] : 0.f;
        }
    }
    for (int64_t r0 = m.warp_row0; r0 < p.rows; r0 += m.warp_stride) {      // warp-uniform trip count
        const int64_t row = r0 + m.sub;
        const bool live = row < p.rows;
        float xv[VPL][V];
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
            const int cv = m.gl + k * lpr;
            if (live && cv < CV) {
                loadv<T, V>(x + row * p.C + cv * V, xv[k]);
            } else {
#pragma unroll
                for (int v = 0; v < V; ++v) xv[k][v] = 0.f;
            }
#pragma unroll
            for (int v = 0; v < V; ++v) s += xv[k][v];
        }
        const float mean = group_sum(s, lpr) * invC;
        float q = 0.f;
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
            const int cv = m.gl + k * lpr;
#pragma unroll
            for (int v = 0; v < V; ++v) {
                const float d = cv < CV ? xv[k][v] - mean : 0.f;
                xv[k][v] = d;
                q = fmaf(d, d, q);
            }
        }
        const float rstd = rsqrtf(group_sum(q, lpr) * invC + p.eps);
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
            const int cv = m.gl + k * lpr;
            if (live && cv < CV) {
                float o[V];
#pragma unroll
                for (int v = 0; v < V; ++v) o[v] = fmaf(xv[k][v] * rstd, ga[k][v], be[k][v]);
                storev<T, V>(y + row * p.C + cv * V, o);
            }
        }
    }
}

template <typename T, int VPL>
__global__ void __launch_bounds__(kLnThreads) ln_bwd_kernel(const LnP p, int lpr) {
    constexpr int V = VecOf<T>::V;
    extern __shared__ float red[];                       // [2][kLnWarps][C]
    const int CV = p.C / V;
    const LnMap m = ln_map(lpr);
    const T *x = reinterpret_cast<const T *>(p.x);
    const T *dy = reinterpret_cast<const T *>(p.dy);
    T *dx = reinterpret_cast<T *>(p.dx);
    const float invC = 1.f / (float)p.C;
    float ga[VPL][V], dga[VPL][V], dbe[VPL][V];
#pragma unroll
    for (int k = 0; k < VPL; ++k) {
        const int cv = m.gl + k * lpr;
#pragma unroll
        for (int v = 0; v < V; ++v) {
            ga[k][v] = cv < CV ? p.gamma[cv * V + v] : 0.f;
            dga[k][v] = 0.f;
            dbe[k][v] = 0.f;
        }
    }
    for (int64_t r0 = m.warp_row0; r0 < p.rows; r0 += m.warp_stride) {
        const int64_t row = r0 + m.sub;
        const bool live = row < p.rows;
        float xv[VPL][V], gv[VPL][V];
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
            const int cv = m.gl + k * lpr;
            if (live && cv < CV) {
                loadv<T, V>(x + row * p.C + cv * V, xv[k]);
                loadv<T, V>(dy + row * p.C + cv * V, gv[k]);
            } else {
#pragma unroll
                for (int v = 0; v < V; ++v) { xv[k][v] = 0.f; gv[k][v] = 0.f; }
            }
#pragma unroll
            for (int v = 0; v < V; ++v) s += xv[k][v];
        }
        const float mean = group_sum(s, lpr) * invC;
        float q = 0.f;
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
            const int cv = m.gl + k * lpr;
#pragma unroll
            for (int v = 0; v < V; ++v) {
                const float d = cv < CV ? xv[k][v] - mean : 0.f;
                xv[k][v] = d;
                q = fmaf(d, d, q);
            }
        }
        const float rstd = rsqrtf(group_sum(q, lpr) * invC + p.eps);
        // xhat = d * rstd;  g = dy * gamma;  dx = rstd * (g - mean(g) - xhat * mean(g * xhat))
        float sg = 0.f, sgx = 0.f;
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
#pragma unroll
            for (int v = 0; v < V; ++v) {
                const float xh = xv[k][v] * rstd;
                xv[k][v] = xh;
                dga[k][v] = fmaf(gv[k][v], xh, dga[k][v]);       // dead rows / columns contribute dy = 0
                dbe[k][v] += gv[k][v];
                const float g = gv[k][v] * ga[k][v];
                gv[k][v] = g;
                sg += g;
                sgx = fmaf(g, xh, sgx);
            }
        }
        const float mg = group_sum(sg, lpr) * invC;
        const float mgx = group_sum(sgx, lpr) * invC;
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
            const int cv = m.gl + k * lpr;
            if (live && cv < CV) {
                float o[V];
#pragma unroll
                for (int v = 0; v < V; ++v) o[v] = rstd * (gv[k][v] - mg - xv[k][v] * mgx);
                storev<T, V>(dx + row * p.C + cv * V, o);
            }
        }
    }
    // per-channel gradients: over the warp's row groups (lanes with equal gl), then over the CTA's warps, then one atomic
    const int warp = threadIdx.x >> 5;
    float *rg = red + (size_t)warp * p.C;
    float *rb = red + (size_t)(kLnWarps + warp) * p.C;
#pragma unroll
    for (int k = 0; k < VPL; ++k) {
        const int cv = m.gl + k * lpr;
#pragma unroll
        for (int v = 0; v < V; ++v) {
            float a = dga[k][v], b = dbe[k][v];
            for (int o = 16; o >= lpr; o >>= 1) {
                a += __shfl_xor_sync(0xffffffffu, a, o);
                b += __shfl_xor_sync(0xffffffffu, b, o);
            }
            if (m.sub == 0 && cv < CV) {
                rg[cv * V + v] = a;
                rb[cv * V + v] = b;
            }
        }
    }
    __syncthreads();
    for (int c = threadIdx.x; c < p.C; c += kLnThreads) {
        float a = 0.f, b = 0.f;
#pragma unroll
        for (int w = 0; w < kLnWarps; ++w) {
            a += red[(size_t)w * p.C + c];
            b += red[(size_t)(kLnWarps + w) * p.C + c];
        }
        atomicAdd(p.dgamma + c, a);
        if (p.dbeta) atomicAdd(p.dbeta + c, b);
    }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
template <typename T, int VPL>
static cudaError_t ln_launch(const LnP &p, bool bwd, int lpr, cudaStream_t st) {
    const int rows_per_cta = kLnWarps * (32 / lpr);
    int64_t ctas = (p.rows + rows_per_cta - 1) / rows_per_cta;
    const int64_t cap = 132 * 8;                                  // persistent-style grid: 8 CTAs of 8 warps per SM at most
    if (ctas > cap) ctas = cap;
    if (!bwd) {
        ln_fwd_kernel<T, VPL><<<(unsigned)ctas, kLnThreads, 0, st>>>(p, lpr);
    } else {
        const size_t smem = (size_t)2 * kLnWarps * p.C * sizeof(float);
        ln_bwd_kernel<T, VPL><<<(unsigned)ctas, kLnThreads, smem, st>>>(p, lpr);
    }
    count_launch();
    return cudaGetLastError();
}

template <typename T>
static cudaError_t ln_t(const LnP &p, bool bwd, cudaStream_t st) {
    constexpr int V = VecOf<T>::V;
    const int CV = p.C / V;
    int lpr = 1;
    while (lpr < CV && lpr < 32) lpr <<= 1;
    const int vpl = (CV + lpr - 1) / lpr;
    switch (vpl) {
        case 1: return ln_launch<T, 1>(p, bwd, lpr, st);
        case 2: return ln_launch<T, 2>(p, bwd, lpr, st);
        case 3: return ln_launch<T, 3>(p, bwd, lpr, st);
        case 4: return ln_launch<T, 4>(p, bwd, lpr, st);
        default: return cudaErrorInvalidValue;                  // capi.cu rejects C > 4 * 32 * V before getting here
    }
}

cudaError_t layernorm_dispatch(const LnP &p, int dtype, bool bwd, cudaStream_t st) {
    switch (dtype) {
        case 0: return ln_t<float>(p, bwd, st);
        case 1: return ln_t<__half>(p, bwd, st);
        default: return ln_t<__nv_bfloat16>(p, bwd, st);
    }
}

}  // namespace smb
