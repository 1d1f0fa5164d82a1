// Internal parameter block for the fused instance-norm kernels.
#pragma once

#include "common.cuh"

namespace smb {

struct NormP {
    int batch, channels;
    int64_t spatial;
    int act, mode2;              // act: 0 none, 1 relu, 2 leaky relu; mode2: 0 none, 1 raw add, 2 normalised add
    float slope, eps;
    int n_cta;
    int64_t rows_per_cta;
    const void *x, *x2, *dy;
    void *y, *dx, *dx2;
    float *stats, *stats2;       // (batch, channels, 2): mean, rstd
    float *partial, *sums;       // workspace
};

// rows per CTA / CTA count: >= 8 CTAs per SM in total, at least 8 row-iterations per thread
inline void norm_plan(int batch, int channels, int64_t spatial, int elem_bytes, int *n_cta, int64_t *rows_per_cta) {
    const int V = 16 / elem_bytes;
    const int CV = channels / V;
    const int RB = 256 / CV;
    const int64_t target = (132 * 8 + batch - 1) / batch;
    int64_t rows = (spatial + target - 1) / target;
    if (rows < (int64_t)RB * 8) rows = (int64_t)RB * 8;
    *rows_per_cta = rows;
    *n_cta = (int)((spatial + rows - 1) / rows);
}

cudaError_t instnorm_dispatch(const NormP &p, int dtype, bool bwd, cudaStream_t st);

// ---- 16-byte vector <-> fp32 registers, shared by the instance-norm and layer-norm kernels ----
template <typename T> struct VecOf { static constexpr int V = 16 / sizeof(T); };

template <typename T, int V> __device__ __forceinline__ void loadv(const T *p, float v[V]);
template <> __device__ __forceinline__ void loadv<float, 4>(const float *p, float v[4]) {
    const float4 a = *reinterpret_cast<const float4 *>(p);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
}
template <> __device__ __forceinline__ void loadv<__half, 8>(const __half *p, float v[8]) {
    const float4 a = load4<__half>(p), b = load4<__half>(p + 4);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
template <> __device__ __forceinline__ void loadv<__nv_bfloat16, 8>(const __nv_bfloat16 *p, float v[8]) {
    const uint4 r = *reinterpret_cast<const uint4 *>(p);
    const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {   // bf16 -> fp32 is a 16-bit shift
        v[2 * i] = __uint_as_float(w[i] << 16);
        v[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
    }
}
template <typename T, int V> __device__ __forceinline__ void storev(T *p, const float v[V]);
template <> __device__ __forceinline__ void storev<float, 4>(float *p, const float v[4]) {
    *reinterpret_cast<float4 *>(p) = make_float4(v[0], v[1], v[2], v[3]);
}
template <> __device__ __forceinline__ void storev<__half, 8>(__half *p, const float v[8]) {
    store4<__half>(p, make_float4(v[0], v[1], v[2], v[3]));
    store4<__half>(p + 4, make_float4(v[4], v[5], v[6], v[7]));
}
template <> __device__ __forceinline__ void storev<__nv_bfloat16, 8>(__nv_bfloat16 *p, const float v[8]) {
    uint4 r;
    __nv_bfloat162 a = __floats2bfloat162_rn(v[0], v[1]), b = __floats2bfloat162_rn(v[2], v[3]);
    __nv_bfloat162 c = __floats2bfloat162_rn(v[4], v[5]), d = __floats2bfloat162_rn(v[6], v[7]);
    r.x = *reinterpret_cast<uint32_t *>(&a); r.y = *reinterpret_cast<uint32_t *>(&b);
    r.z = *reinterpret_cast<uint32_t *>(&c); r.w = *reinterpret_cast<uint32_t *>(&d);
    *reinterpret_cast<uint4 *>(p) = r;
}

// Fused LayerNorm over the last axis of a (rows, C) matrix (csrc/layernorm.cu)
struct LnP {
    int64_t rows;
    int C;
    float eps;
    const void *x, *dy;
    const float *gamma, *beta;
    void *y, *dx;
    float *dgamma, *dbeta;       // fp32 accumulators, zero-initialised by the caller
};
cudaError_t layernorm_dispatch(const LnP &p, int dtype, bool bwd, cudaStream_t st);

}  // namespace smb
