// Shared device helpers for the sm_90a scan / conv kernels.
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace smb {

// host-side launch accounting (smb_launch_count)
void count_launch();

// opt a kernel into > 48 KB dynamic shared memory once per device (the attribute is per context)
#define SMB_SET_SMEM_ONCE(kernel, bytes)                                                                        \
    do {                                                                                                        \
        static bool done_[64] = {};                                                                             \
        int dv_ = 0;                                                                                            \
        cudaGetDevice(&dv_);                                                                                    \
        if (!done_[dv_ & 63]) {                                                                                 \
            e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bytes));       \
            if (e != cudaSuccess) return e;                                                                     \
            done_[dv_ & 63] = true;                                                                             \
        }                                                                                                       \
    } while (0)

constexpr int kTile = 32;         // scan positions per warp-private shared-memory tile
constexpr int kCkpt = 256;        // state checkpoint interval (scan positions) shared by fwd and bwd
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

// ---------------------------------------------------------------------------------------------
// math.  The decay uses the MUFU ex2 path with A pre-scaled by log2(e), as the reference kernel
// does (selective_scan_fwd_kernel.cuh:169-171,216).
// ---------------------------------------------------------------------------------------------
#ifdef SMB_EMU   // host build for tools/simt_emu (functional tests without a GPU): no PTX
__device__ __forceinline__ float ex2(float x) { return exp2f(x); }
#else
__device__ __forceinline__ float ex2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
#endif
// ---- fp32 pairs: the kernels keep two states per float2; sm_90 has no packed fp32 arithmetic, so each op is two scalar ones ----
__device__ __forceinline__ float2 f2(float a, float b) { return make_float2(a, b); }
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(a.x * b.x, a.y * b.y); }
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 ex2x2_mufu(float2 x) { return make_float2(ex2(x.x), ex2(x.y)); }
// 2^x for x <= 0 on the FMA pipe (Cody-Waite split + degree-6 polynomial, rel. error ~2e-7, same class as MUFU.EX2):
// lets a fraction of the decays move off the MUFU pipe (see SMB_POLY_MASK below).
__device__ __forceinline__ float2 ex2x2_poly(float2 x) {
    x.x = fmaxf(x.x, -126.f);
    x.y = fmaxf(x.y, -126.f);
    const float2 t = fadd2(x, f2(12582912.f, 12582912.f));          // round to nearest integer in the low mantissa bits
    const float2 n = fadd2(t, f2(-12582912.f, -12582912.f));
    const float2 f = ffma2(n, f2(-1.f, -1.f), x);                    // f in [-0.5, 0.5]
    float2 p = f2(1.535336188319500e-4f, 1.535336188319500e-4f);
    p = ffma2(p, f, f2(1.339887440266574e-3f, 1.339887440266574e-3f));
    p = ffma2(p, f, f2(9.618437357674640e-3f, 9.618437357674640e-3f));
    p = ffma2(p, f, f2(5.550332471162809e-2f, 5.550332471162809e-2f));
    p = ffma2(p, f, f2(2.402264791363012e-1f, 2.402264791363012e-1f));
    p = ffma2(p, f, f2(6.931472028550421e-1f, 6.931472028550421e-1f));
    p = ffma2(p, f, f2(1.f, 1.f));
    return make_float2(__int_as_float(__float_as_int(p.x) + (__float_as_int(t.x) << 23)),
                       __int_as_float(__float_as_int(p.y) + (__float_as_int(t.y) << 23)));
}
// which state pairs take the polynomial path (bit m = pair m).  The default keeps every decay on the MUFU; other masks have not
// been measured on H100.
#ifndef SMB_POLY_MASK
#define SMB_POLY_MASK 0x00
#endif
template <int M> __device__ __forceinline__ float2 decay2(float2 arg) {
    if ((SMB_POLY_MASK >> M) & 1) return ex2x2_poly(arg);
    return ex2x2_mufu(arg);
}

// softplus with the reference's threshold (selective_scan_fwd_kernel.cuh:155), branch-free and ~14 instructions:
//   softplus(x) = max(x, 0) + log1p(t),  t = exp(-|x|) in (0, 1]
//   log1p(t)    = 2 atanh(s),  s = t / (2 + t) <= 1/3  ->  2 s (1 + w/3 + w^2/5 + ... + w^6/13),  w = s^2
// (series remainder < 2e-8 relative; for x > 20 the log term is < 2.1e-9, i.e. the reference's `x` branch in fp32).
__device__ __forceinline__ float softplus20(float x) {
    const float t = __expf(-fabsf(x));
    const float s = __fdividef(t, 2.f + t);
    const float w = s * s;
    float p = fmaf(w, 1.f / 13.f, 1.f / 11.f);
    p = fmaf(p, w, 1.f / 9.f);
    p = fmaf(p, w, 1.f / 7.f);
    p = fmaf(p, w, 1.f / 5.f);
    p = fmaf(p, w, 1.f / 3.f);
    p = fmaf(p, w, 1.f);
    return fmaf(2.f * s, p, fmaxf(x, 0.f));
}
__device__ __forceinline__ float sigmoidf(float x) { return __fdividef(1.f, 1.f + __expf(-x)); }
// 1 - exp(-x) for x >= 0 (= sigmoid(raw) when x = softplus(raw)): Taylor polynomial below 1/8 (remainder x^6/720 < 6e-9
// relative), 1 - ex2 above (cancellation error < 6e-8 / 0.117); ~9 instructions against expm1f's ~25
__device__ __forceinline__ float one_minus_exp_neg(float x) {
    float p = fmaf(x, -1.f / 120.f, 1.f / 24.f);
    p = fmaf(p, -x, 1.f / 6.f);
    p = fmaf(p, -x, 0.5f);
    p = fmaf(p, -x, 1.f);
    const float big = 1.f - __expf(-x);
    return x < 0.125f ? p * x : big;
}

// ---------------------------------------------------------------------------------------------
// element conversion
// ---------------------------------------------------------------------------------------------
template <typename T> __device__ __forceinline__ float to_f32(T v);
template <> __device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f32<__half>(__half v) { return __half2float(v); }
template <> __device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ __half from_f32<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

// 4 consecutive elements <-> float4; the pointer must be aligned to 4 elements.
template <typename T> __device__ __forceinline__ float4 load4(const T *p);
template <> __device__ __forceinline__ float4 load4<float>(const float *p) { return *reinterpret_cast<const float4 *>(p); }
template <> __device__ __forceinline__ float4 load4<__half>(const __half *p) {
    uint2 r = *reinterpret_cast<const uint2 *>(p);
    __half2 a = *reinterpret_cast<__half2 *>(&r.x), b = *reinterpret_cast<__half2 *>(&r.y);
    float2 fa = __half22float2(a), fb = __half22float2(b);
    return make_float4(fa.x, fa.y, fb.x, fb.y);
}
template <> __device__ __forceinline__ float4 load4<__nv_bfloat16>(const __nv_bfloat16 *p) {
    uint2 r = *reinterpret_cast<const uint2 *>(p);
    __nv_bfloat162 a = *reinterpret_cast<__nv_bfloat162 *>(&r.x), b = *reinterpret_cast<__nv_bfloat162 *>(&r.y);
    float2 fa = __bfloat1622float2(a), fb = __bfloat1622float2(b);
    return make_float4(fa.x, fa.y, fb.x, fb.y);
}
template <typename T> __device__ __forceinline__ void store4(T *p, float4 v);
template <> __device__ __forceinline__ void store4<float>(float *p, float4 v) { *reinterpret_cast<float4 *>(p) = v; }
template <> __device__ __forceinline__ void store4<__half>(__half *p, float4 v) {
    __half2 a = __floats2half2_rn(v.x, v.y), b = __floats2half2_rn(v.z, v.w);
    uint2 r;
    r.x = *reinterpret_cast<uint32_t *>(&a);
    r.y = *reinterpret_cast<uint32_t *>(&b);
    *reinterpret_cast<uint2 *>(p) = r;
}
template <> __device__ __forceinline__ void store4<__nv_bfloat16>(__nv_bfloat16 *p, float4 v) {
    __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
    uint2 r;
    r.x = *reinterpret_cast<uint32_t *>(&a);
    r.y = *reinterpret_cast<uint32_t *>(&b);
    *reinterpret_cast<uint2 *>(p) = r;
}
template <typename T> __device__ __forceinline__ bool aligned4(const T *p) {
    return (reinterpret_cast<uintptr_t>(p) & (4 * sizeof(T) - 1)) == 0;
}

// ---------------------------------------------------------------------------------------------
// Warp-private activation tile: 32 rows (channels) x 32 scan positions, fp32, 128-byte rows with
// an XOR swizzle on the 16-byte chunk index so that both access patterns are conflict-free:
//   fill/store: 8 lanes cover one row's 8 chunks (coalesced 128 B global segments);
//   compute   : lane == row reads chunk c (4 consecutive positions) with one LDS.128.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int tile_chunk_off(int row, int c) { return row * kTile + (((c ^ (row & 7))) << 2); }
__device__ __forceinline__ float4 tile_read4(const float *tile, int row, int c) {
    return *reinterpret_cast<const float4 *>(tile + tile_chunk_off(row, c));
}
__device__ __forceinline__ void tile_write4(float *tile, int row, int c, float4 v) {
    *reinterpret_cast<float4 *>(tile + tile_chunk_off(row, c)) = v;
}

// Scan position j <-> token index t along L.
__device__ __forceinline__ int pos_to_tok(int j, int L, bool reverse) { return reverse ? L - 1 - j : j; }

// Fill a tile with scan positions [j0, j0+32) of `nrows` rows; rows >= nrows and positions >= L read 0.
// base points at (row 0, token 0); row_stride in elements.
template <typename T>
__device__ __forceinline__ void fill_tile(float *tile, const T *base, int64_t row_stride, int nrows, int j0, int L,
                                          bool reverse, int lane) {
    float4 v[8];
#pragma unroll
    for (int it = 0; it < 8; ++it) {
        const int unit = it * 32 + lane;
        const int row = unit >> 3, c = unit & 7;
        const int jl = j0 + 4 * c;               // first scan position of the chunk
        float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
        if (row < nrows && jl < L) {
            const T *rp = base + (int64_t)row * row_stride;
            if (!reverse) {
                const T *p = rp + jl;
                if (jl + 3 < L && aligned4(p)) {
                    r = load4<T>(p);
                } else {
                    r.x = to_f32<T>(p[0]);
                    if (jl + 1 < L) r.y = to_f32<T>(p[1]);
                    if (jl + 2 < L) r.z = to_f32<T>(p[2]);
                    if (jl + 3 < L) r.w = to_f32<T>(p[3]);
                }
            } else {
                const int th = L - 1 - jl;       // token of position jl (highest of the chunk)
                const T *p = rp + (th - 3);
                if (th - 3 >= 0 && aligned4(p)) {
                    float4 q = load4<T>(p);
                    r = make_float4(q.w, q.z, q.y, q.x);
                } else {
                    r.x = to_f32<T>(rp[th]);
                    if (th - 1 >= 0) r.y = to_f32<T>(rp[th - 1]);
                    if (th - 2 >= 0) r.z = to_f32<T>(rp[th - 2]);
                    if (th - 3 >= 0) r.w = to_f32<T>(rp[th - 3]);
                }
            }
        }
        v[it] = r;
    }
#pragma unroll
    for (int it = 0; it < 8; ++it) {
        const int unit = it * 32 + lane;
        tile_write4(tile, unit >> 3, unit & 7, v[it]);
    }
}

// Inverse of fill_tile: write scan positions [j0, j0+32) of `nrows` rows back to global memory.
template <typename T>
__device__ __forceinline__ void store_tile(const float *tile, T *base, int64_t row_stride, int nrows, int j0, int L,
                                           bool reverse, int lane) {
#pragma unroll
    for (int it = 0; it < 8; ++it) {
        const int unit = it * 32 + lane;
        const int row = unit >> 3, c = unit & 7;
        const int jl = j0 + 4 * c;
        if (row < nrows && jl < L) {
            const float4 r = tile_read4(tile, row, c);
            T *rp = base + (int64_t)row * row_stride;
            if (!reverse) {
                T *p = rp + jl;
                if (jl + 3 < L && aligned4(p)) {
                    store4<T>(p, r);
                } else {
                    p[0] = from_f32<T>(r.x);
                    if (jl + 1 < L) p[1] = from_f32<T>(r.y);
                    if (jl + 2 < L) p[2] = from_f32<T>(r.z);
                    if (jl + 3 < L) p[3] = from_f32<T>(r.w);
                }
            } else {
                const int th = L - 1 - jl;
                T *p = rp + (th - 3);
                if (th - 3 >= 0 && aligned4(p)) {
                    store4<T>(p, make_float4(r.w, r.z, r.y, r.x));
                } else {
                    rp[th] = from_f32<T>(r.x);
                    if (th - 1 >= 0) rp[th - 1] = from_f32<T>(r.y);
                    if (th - 2 >= 0) rp[th - 2] = from_f32<T>(r.z);
                    if (th - 3 >= 0) rp[th - 3] = from_f32<T>(r.w);
                }
            }
        }
    }
}

// In-place pre-passes over the lane's own row of a tile (lane == row == channel), vectorised and branch-free so the
// serial recurrence loop that follows contains no transcendental chains:
//   dt   <- softplus?(delta + bias), forced to 0 for positions >= nvalid (a = 1, b = 0: the scan identity)
//   gate <- z * sigmoid(z)
__device__ __forceinline__ void prepass_dt(float *tile, int lane, float bias, bool softplus, int nvalid) {
    if (nvalid >= kTile) {                               // full tile (warp-uniform): no masking
#pragma unroll
        for (int c = 0; c < kTile / 4; ++c) {
            float4 v = tile_read4(tile, lane, c);
            float x[4] = {v.x + bias, v.y + bias, v.z + bias, v.w + bias};
            if (softplus) {
#pragma unroll
                for (int e = 0; e < 4; ++e) x[e] = softplus20(x[e]);
            }
            tile_write4(tile, lane, c, make_float4(x[0], x[1], x[2], x[3]));
        }
        return;
    }
#pragma unroll
    for (int c = 0; c < kTile / 4; ++c) {
        float4 v = tile_read4(tile, lane, c);
        float x[4] = {v.x + bias, v.y + bias, v.z + bias, v.w + bias};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            if (softplus) x[e] = softplus20(x[e]);
            if (4 * c + e >= nvalid) x[e] = 0.f;
        }
        tile_write4(tile, lane, c, make_float4(x[0], x[1], x[2], x[3]));
    }
}
__device__ __forceinline__ void prepass_silu(float *tile, int lane) {
#pragma unroll
    for (int c = 0; c < kTile / 4; ++c) {
        float4 v = tile_read4(tile, lane, c);
        v.x *= sigmoidf(v.x); v.y *= sigmoidf(v.y); v.z *= sigmoidf(v.z); v.w *= sigmoidf(v.w);
        tile_write4(tile, lane, c, v);
    }
}
// g <- g * silu(z)   (both tiles are this lane's rows)
__device__ __forceinline__ void prepass_gate_grad(float *gtile, const float *ztile, int lane) {
#pragma unroll
    for (int c = 0; c < kTile / 4; ++c) {
        float4 g = tile_read4(gtile, lane, c);
        const float4 z = tile_read4(ztile, lane, c);
        g.x *= z.x * sigmoidf(z.x); g.y *= z.y * sigmoidf(z.y); g.z *= z.z * sigmoidf(z.z); g.w *= z.w * sigmoidf(z.w);
        tile_write4(gtile, lane, c, g);
    }
}

// ---------------------------------------------------------------------------------------------
// Batched fills.  The recurrence kernels are latency-sensitive (3-4 resident warps per scheduler), so the global
// loads of ALL streams of a tile are issued back to back into registers (raw, unconverted) before the first
// conversion / shared store: one DRAM/L2 latency per tile instead of one per stream.  The next tile's lines are
// pulled into L2 with prefetch.global.L2 while the current tile is being computed.
// ---------------------------------------------------------------------------------------------
template <typename T> struct Raw4 { using type = uint2; };
template <> struct Raw4<float> { using type = float4; };
template <typename T> __device__ __forceinline__ typename Raw4<T>::type ldraw4(const T *p) {
    return *reinterpret_cast<const typename Raw4<T>::type *>(p);
}
template <typename T> __device__ __forceinline__ typename Raw4<T>::type zeroraw4();
template <> __device__ __forceinline__ float4 zeroraw4<float>() { return make_float4(0.f, 0.f, 0.f, 0.f); }
template <> __device__ __forceinline__ uint2 zeroraw4<__half>() { return make_uint2(0u, 0u); }
template <> __device__ __forceinline__ uint2 zeroraw4<__nv_bfloat16>() { return make_uint2(0u, 0u); }
template <typename T> __device__ __forceinline__ float4 cvtraw4(typename Raw4<T>::type r);
template <> __device__ __forceinline__ float4 cvtraw4<float>(float4 r) { return r; }
template <> __device__ __forceinline__ float4 cvtraw4<__half>(uint2 r) {
    const float2 a = __half22float2(*reinterpret_cast<__half2 *>(&r.x)), b = __half22float2(*reinterpret_cast<__half2 *>(&r.y));
    return make_float4(a.x, a.y, b.x, b.y);
}
template <> __device__ __forceinline__ float4 cvtraw4<__nv_bfloat16>(uint2 r) {      // bf16 -> fp32 is a 16-bit shift
    return make_float4(__uint_as_float(r.x << 16), __uint_as_float(r.x & 0xffff0000u), __uint_as_float(r.y << 16),
                       __uint_as_float(r.y & 0xffff0000u));
}
#ifdef SMB_EMU
__device__ __forceinline__ void prefetch_l2(const void *) {}
__device__ __forceinline__ void red_add_v4(float *a, float x, float y, float z, float w) {
    atomicAdd(a, x); atomicAdd(a + 1, y); atomicAdd(a + 2, z); atomicAdd(a + 3, w);
}
#else
__device__ __forceinline__ void prefetch_l2(const void *p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
// one 16-byte vector reduction: 4 consecutive fp32 accumulators, address aligned to 16 bytes
__device__ __forceinline__ void red_add_v4(float *a, float x, float y, float z, float w) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(a), "f"(x), "f"(y), "f"(z), "f"(w) : "memory");
}
#endif

// true when 4-element vector accesses of a (rows, L) operand are aligned for every full tile of this walk
template <typename T> __device__ __forceinline__ bool stream_aligned(const T *base, int64_t row_stride, int L, bool reverse) {
    return aligned4(base) && (row_stride & 3) == 0 && (!reverse || (L & 3) == 0);
}

// Per-lane pointers for the fast fills / stores: lane handles chunk c = lane&7 of rows (lane>>3) + 4*it, it = 0..7.
// lp = address of (row lane>>3, chunk c) for the tile at scan position 0; a tile at j0 is lp +/- j0 and row 4*it is
// + it*rowstep, so the hot loops contain one 64-bit multiply-add per access and no selects.
template <typename T> struct LanePtr {
    const T *lp;
    int64_t rowstep;
};
template <typename T>
__device__ __forceinline__ LanePtr<T> lane_ptr(const T *base, int64_t row_stride, int L, bool reverse, int lane) {
    LanePtr<T> r;
    const int c = lane & 7;
    r.lp = base + (int64_t)(lane >> 3) * row_stride + (reverse ? (L - 4 - 4 * c) : 4 * c);
    r.rowstep = 4 * row_stride;
    return r;
}

// fill K activation tiles with scan positions [j0, j0+32); REQUIRES j0 + 32 <= L and stream_aligned() for every stream
template <typename T, int K, int KA>
__device__ __forceinline__ void fill_tiles_fast(float *const (&tiles)[KA], const LanePtr<T> (&lps)[KA], int nrows, int j0,
                                                bool reverse, int lane) {
    static_assert(K <= KA, "array too small");
    constexpr int H = sizeof(T) == 4 ? 2 : 1;            // fp32: two halves to bound the registers in flight
    constexpr int IT = 8 / H;
    const int64_t toff = reverse ? -(int64_t)j0 : (int64_t)j0;
    const int row0 = lane >> 3, c = lane & 7;
#pragma unroll
    for (int half = 0; half < H; ++half) {
        typename Raw4<T>::type r[K][IT];
#pragma unroll
        for (int i = 0; i < IT; ++i) {
            const int it = half * IT + i;
            const bool ok = row0 + 4 * it < nrows;
#pragma unroll
            for (int k = 0; k < K; ++k) r[k][i] = ok ? ldraw4<T>(lps[k].lp + toff + it * lps[k].rowstep) : zeroraw4<T>();
        }
#pragma unroll
        for (int i = 0; i < IT; ++i) {
            const int it = half * IT + i;
#pragma unroll
            for (int k = 0; k < K; ++k) {
                float4 v = cvtraw4<T>(r[k][i]);
                if (reverse) v = make_float4(v.w, v.z, v.y, v.x);
                tile_write4(tiles[k], row0 + 4 * it, c, v);
            }
        }
    }
}

// store one tile back (inverse of the fast fill); same requirements
template <typename T>
__device__ __forceinline__ void store_tile_fast(const float *tile, T *lp, int64_t rowstep, int nrows, int j0, bool reverse, int lane) {
    const int64_t toff = reverse ? -(int64_t)j0 : (int64_t)j0;
    const int row0 = lane >> 3, c = lane & 7;
#pragma unroll
    for (int it = 0; it < 8; ++it) {
        if (row0 + 4 * it < nrows) {
            float4 v = tile_read4(tile, row0 + 4 * it, c);
            if (reverse) v = make_float4(v.w, v.z, v.y, v.x);
            store4<T>(lp + toff + it * rowstep, v);
        }
    }
}

// pull the next tile's row segments into L2 (one or two lines per row and stream)
template <typename T, int K, int KA>
__device__ __forceinline__ void prefetch_tiles(const T *const (&bases)[KA], const int64_t (&strides)[KA], int nrows, int j0n, int L,
                                               bool reverse, int lane) {
    if (lane < nrows && j0n < L) {
        const int lo = reverse ? max(L - j0n - kTile, 0) : j0n;
        const int hi = reverse ? L - 1 - j0n : min(j0n + kTile, L) - 1;
#pragma unroll
        for (int k = 0; k < K; ++k) {
            const T *rp = bases[k] + (int64_t)lane * strides[k];
            prefetch_l2(rp + lo);
            if (sizeof(T) == 4) prefetch_l2(rp + hi);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Warp-private B / C tile: 32 scan positions x N states, position-major so that one position's
// states are read with broadcast LDS.128 by every lane (lane == channel).  The 16-byte chunk
// index is XOR-swizzled with (q>>1) to spread the transposing fill over 8 bank groups.
// ---------------------------------------------------------------------------------------------
template <int N> __device__ __forceinline__ int bc_off(int q, int n) {
    return q * N + ((((n >> 2) ^ ((q >> 1) & (N / 4 - 1)))) << 2) + (n & 3);
}
// same, for a position known at compile time relative to a block of 8 positions (blk = tile + 8*k*N): constant offset
template <int N, int QL, int CH> __device__ __forceinline__ float4 bc_read4_c(const float *blk) {
    return *reinterpret_cast<const float4 *>(blk + QL * N + (((CH ^ ((QL >> 1) & (N / 4 - 1)))) << 2));
}
template <int N> __device__ __forceinline__ float4 bc_read4(const float *tile, int q, int chunk) {
    return *reinterpret_cast<const float4 *>(tile + q * N + (((chunk ^ ((q >> 1) & (N / 4 - 1)))) << 2));
}
// base points at (state 0, token 0) of the (dstate, L) slab; ns / ls are the state / token strides.
template <typename T, int N>
__device__ __forceinline__ void fill_bc_tile(float *tile, const T *base, int64_t ns, int64_t ls, int j0, int L,
                                             bool reverse, int lane) {
    const int j = j0 + lane;
    const bool valid = j < L;
    const int64_t toff = (int64_t)pos_to_tok(valid ? j : 0, L, reverse) * ls;
    float v[N];
#pragma unroll
    for (int n = 0; n < N; ++n) v[n] = valid ? to_f32<T>(base[(int64_t)n * ns + toff]) : 0.f;
#pragma unroll
    for (int n = 0; n < N; ++n) tile[bc_off<N>(lane, n)] = v[n];
}

constexpr int kRun = 8;           // positions per lane in the run-per-lane kernels (bwd scan, conv1d)

// ---------------------------------------------------------------------------------------------
// per-lane runs of 8 consecutive scan positions straight from / to global memory
// ---------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ void load_run8(const T *row, int j, int L, bool reverse, float v[kRun]) {
#pragma unroll
    for (int i = 0; i < kRun; ++i) v[i] = 0.f;
    if (j >= L) return;
    if (!reverse) {
        const T *p = row + j;
        if (j + 7 < L && aligned4(p)) {
            const float4 a = load4<T>(p), b = load4<T>(p + 4);
            v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
        } else {
#pragma unroll
            for (int i = 0; i < kRun; ++i) if (j + i < L) v[i] = to_f32<T>(p[i]);
        }
    } else {
        const int th = L - 1 - j;
        const T *p = row + (th - 7);
        if (th - 7 >= 0 && aligned4(p)) {
            const float4 a = load4<T>(p), b = load4<T>(p + 4);
            v[7] = a.x; v[6] = a.y; v[5] = a.z; v[4] = a.w; v[3] = b.x; v[2] = b.y; v[1] = b.z; v[0] = b.w;
        } else {
#pragma unroll
            for (int i = 0; i < kRun; ++i) if (th - i >= 0) v[i] = to_f32<T>(row[th - i]);
        }
    }
}

template <typename T>
__device__ __forceinline__ void store_run8(T *row, int j, int L, bool reverse, const float v[kRun]) {
    if (j >= L) return;
    if (!reverse) {
        T *p = row + j;
        if (j + 7 < L && aligned4(p)) {
            store4<T>(p, make_float4(v[0], v[1], v[2], v[3]));
            store4<T>(p + 4, make_float4(v[4], v[5], v[6], v[7]));
        } else {
#pragma unroll
            for (int i = 0; i < kRun; ++i) if (j + i < L) p[i] = from_f32<T>(v[i]);
        }
    } else {
        const int th = L - 1 - j;
        T *p = row + (th - 7);
        if (th - 7 >= 0 && aligned4(p)) {
            store4<T>(p, make_float4(v[7], v[6], v[5], v[4]));
            store4<T>(p + 4, make_float4(v[3], v[2], v[1], v[0]));
        } else {
#pragma unroll
            for (int i = 0; i < kRun; ++i) if (th - i >= 0) row[th - i] = from_f32<T>(v[i]);
        }
    }
}

// K (1 or 2) B/C tiles at once: all 2*N (or N) global loads in flight before the first shared store
template <typename T, int N, int K>
__device__ __forceinline__ void fill_bc_tiles(float *const (&tiles)[K], const T *const (&bases)[K], const int64_t (&ns)[K],
                                              const int64_t (&ls)[K], int j0, int L, bool reverse, int lane) {
    const int j = j0 + lane;
    const bool valid = j < L;
    const int tok = pos_to_tok(valid ? j : 0, L, reverse);
    T v[K][N];
#pragma unroll
    for (int k = 0; k < K; ++k) {
        const T *b = bases[k] + (int64_t)tok * ls[k];
#pragma unroll
        for (int n = 0; n < N; ++n) v[k][n] = valid ? b[(int64_t)n * ns[k]] : from_f32<T>(0.f);
    }
#pragma unroll
    for (int k = 0; k < K; ++k) {
#pragma unroll
        for (int n = 0; n < N; ++n) tiles[k][bc_off<N>(lane, n)] = to_f32<T>(v[k][n]);
    }
}
template <typename T, int N, int K>
__device__ __forceinline__ void prefetch_bc(const T *const (&bases)[K], const int64_t (&ns)[K], const int64_t (&ls)[K], int j0n, int L,
                                            bool reverse, int lane) {
    if (lane < N && j0n < L) {
        const int lo = reverse ? max(L - j0n - kTile, 0) : j0n;
#pragma unroll
        for (int k = 0; k < K; ++k) prefetch_l2(bases[k] + (int64_t)lane * ns[k] + (int64_t)lo * ls[k]);
    }
}

// ---------------------------------------------------------------------------------------------
// warp reductions
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

}  // namespace smb
