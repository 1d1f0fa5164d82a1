// Per-position recurrence steps shared by the lane-per-channel kernels (forward passes, backward state recompute).
#pragma once

#include "common.cuh"

namespace smb {

// ---------------------------------------------------------------------------------------------
// one scan position for all N states of this lane's channel, states packed in pairs (FFMA2 / FMUL2):
//   a = 2^(dt A2) ; h = a h + (dt u) B          [+ y += C h in the main pass]
// A compile-time subset of the pairs evaluates the decay on the FMA pipe (decay2<M>), the rest on the MUFU.
// ---------------------------------------------------------------------------------------------
template <int N, int QL, int JN>
__device__ __forceinline__ void scan_step_agg_chunk(const float *s_B, float2 dt2, float2 du2, const float2 (&A2)[N / 2],
                                                    float2 (&h)[N / 2]) {
    const float4 b4 = bc_read4_c<N, QL, JN>(s_B);
    const float2 a0 = decay2<2 * JN>(fmul2(dt2, A2[2 * JN]));
    const float2 a1 = decay2<2 * JN + 1>(fmul2(dt2, A2[2 * JN + 1]));
    h[2 * JN] = ffma2(a0, h[2 * JN], fmul2(du2, f2(b4.x, b4.y)));
    h[2 * JN + 1] = ffma2(a1, h[2 * JN + 1], fmul2(du2, f2(b4.z, b4.w)));
}
// chunks JN .. N/4 - 1 of one position, in ascending order
template <int N, int QL, int JN = 0>
__device__ __forceinline__ void scan_step_agg(const float *s_B, float2 dt2, float2 du2, const float2 (&A2)[N / 2],
                                              float2 (&h)[N / 2]) {
    if constexpr (JN < N / 4) {
        scan_step_agg_chunk<N, QL, JN>(s_B, dt2, du2, A2, h);
        scan_step_agg<N, QL, JN + 1>(s_B, dt2, du2, A2, h);
    }
}
template <int N, int QL, int JN>
__device__ __forceinline__ void scan_step_main_chunk(const float *s_B, const float *s_C, float2 dt2, float2 du2,
                                                     const float2 (&A2)[N / 2], float2 (&h)[N / 2], float2 &y) {
    const float4 b4 = bc_read4_c<N, QL, JN>(s_B);
    const float4 c4 = bc_read4_c<N, QL, JN>(s_C);
    const float2 a0 = decay2<2 * JN>(fmul2(dt2, A2[2 * JN]));
    const float2 a1 = decay2<2 * JN + 1>(fmul2(dt2, A2[2 * JN + 1]));
    h[2 * JN] = ffma2(a0, h[2 * JN], fmul2(du2, f2(b4.x, b4.y)));
    h[2 * JN + 1] = ffma2(a1, h[2 * JN + 1], fmul2(du2, f2(b4.z, b4.w)));
    y = ffma2(f2(c4.x, c4.y), h[2 * JN], y);
    y = ffma2(f2(c4.z, c4.w), h[2 * JN + 1], y);
}
// chunks JN .. N/4 - 1 of one position; even chunks accumulate C h into ya, odd ones into yb
template <int N, int QL, int JN>
__device__ __forceinline__ void scan_step_main_from(const float *s_B, const float *s_C, float2 dt2, float2 du2,
                                                    const float2 (&A2)[N / 2], float2 (&h)[N / 2], float2 &ya, float2 &yb) {
    if constexpr (JN < N / 4) {
        scan_step_main_chunk<N, QL, JN>(s_B, s_C, dt2, du2, A2, h, (JN & 1) ? yb : ya);
        scan_step_main_from<N, QL, JN + 1>(s_B, s_C, dt2, du2, A2, h, ya, yb);
    }
}
template <int N, int QL>
__device__ __forceinline__ float scan_step_main(const float *s_B, const float *s_C, float2 dt2, float2 du2,
                                                const float2 (&A2)[N / 2], float2 (&h)[N / 2]) {
    float2 ya = f2(0.f, 0.f), yb = f2(0.f, 0.f);
    scan_step_main_from<N, QL, 0>(s_B, s_C, dt2, du2, A2, h, ya, yb);
    const float2 ys = fadd2(ya, yb);
    return ys.x + ys.y;
}

// 8 consecutive positions (compile-time local index QL = 0..7)
template <int N, int QL>
__device__ __forceinline__ void agg_block(const float *blkB, const float (&uu)[8], const float (&dd)[8], const float2 (&A2)[N / 2],
                                          float2 (&h)[N / 2], float &sumdt) {
    if constexpr (QL < 8) {
        const float dt = dd[QL], du = dt * uu[QL];
        sumdt += dt;
        scan_step_agg<N, QL>(blkB, f2(dt, dt), f2(du, du), A2, h);
        agg_block<N, QL + 1>(blkB, uu, dd, A2, h, sumdt);
    }
}
template <int N, int QL>
__device__ __forceinline__ void main_block(const float *blkB, const float *blkC, const float (&uu)[8], const float (&dd)[8], float Dv,
                                           const float2 (&A2)[N / 2], float2 (&h)[N / 2], float (&yy)[8]) {
    if constexpr (QL < 8) {
        const float dt = dd[QL], du = dt * uu[QL];
        const float ys = scan_step_main<N, QL>(blkB, blkC, f2(dt, dt), f2(du, du), A2, h);
        yy[QL] = fmaf(Dv, uu[QL], ys);
        main_block<N, QL + 1>(blkB, blkC, uu, dd, Dv, A2, h, yy);
    }
}

// ---------------------------------------------------------------------------------------------
// reverse aggregate (R1 of the backward pass)
// ---------------------------------------------------------------------------------------------
// one reverse position for all states (pairs packed):  mu = a (mu + g C)
template <int N, int QL, int JN>
__device__ __forceinline__ void ragg_step_chunk(const float *s_C, float2 dt2, float2 g2, const float2 (&A2)[N / 2],
                                                float2 (&mu)[N / 2]) {
    const float4 c4 = bc_read4_c<N, QL, JN>(s_C);
    const float2 a0 = decay2<2 * JN>(fmul2(dt2, A2[2 * JN]));
    const float2 a1 = decay2<2 * JN + 1>(fmul2(dt2, A2[2 * JN + 1]));
    mu[2 * JN] = fmul2(a0, ffma2(g2, f2(c4.x, c4.y), mu[2 * JN]));
    mu[2 * JN + 1] = fmul2(a1, ffma2(g2, f2(c4.z, c4.w), mu[2 * JN + 1]));
}
template <int N, int QL, int JN = 0>
__device__ __forceinline__ void ragg_step(const float *s_C, float2 dt2, float2 g2, const float2 (&A2)[N / 2],
                                          float2 (&mu)[N / 2]) {
    if constexpr (JN < N / 4) {
        ragg_step_chunk<N, QL, JN>(s_C, dt2, g2, A2, mu);
        ragg_step<N, QL, JN + 1>(s_C, dt2, g2, A2, mu);
    }
}
// 8 consecutive positions walked in descending order (compile-time local index QL = 7..0)
template <int N, int QL>
__device__ __forceinline__ void ragg_block(const float *blkC, const float (&gg)[8], const float (&dd)[8], const float2 (&A2)[N / 2],
                                           float2 (&mu)[N / 2], float &sumdt) {
    if constexpr (QL >= 0) {
        const float dt = dd[QL], g = gg[QL];
        sumdt += dt;
        ragg_step<N, QL>(blkC, f2(dt, dt), f2(g, g), A2, mu);
        ragg_block<N, QL - 1>(blkC, gg, dd, A2, mu, sumdt);
    }
}

}  // namespace smb
