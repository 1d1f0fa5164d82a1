// Backward selective scan, pass R3, second generation (opt-in: SMB_R3_V2=1; emulator-validated, first hardware run pending).
//
// Same algorithm, operands, outputs and launch geometry as scan_bwd_main_kernel (scan_bwd.cu: warp == channel, lane == run of
// 8 positions, CTA == 8 channels of one 256-position chunk) -- this version removes instructions, not memory
// traffic.  Per
// (state, 8 positions, lane), counted in SASS with tools/sass_loops.py: 318 -> see DESIGN.md 3.2.
//   * Kogge-Stone steps use the shuffle's own in-range predicate (shfl.sync ... d|p) on the combine, so the step is
//     2 SHFL + 1 FFMA + 1 FMUL with no ISETP / FSEL; the last step drops the span product altogether.
//   * The chunk's incoming state / adjoint is folded into lane 0's / lane 31's aggregate before the scan, so the exclusive
//     shift moves one value instead of two and needs no fix-up FFMA.
//   * A lane's span product is ex2(A * sum dt) (one FMUL + one MUFU) instead of eight FMULs.
//   * Reverse aggregate and lambda re-run are FFMA chains on a * (g C) computed packed.
//   * dA: one shared-memory partial per (lane, state) and a single 32-term column sum per warp at the end, instead of a
//     5-step shuffle reduction + atomic per state.
//   * dB / dC: two states per barrier round; the cross-channel reduction reads 16-byte vectors (4 positions) and leaves as one
//     red.global.add.v4.f32 per (tensor, state, 4 positions) per CTA: 8 LDS.128 + 7 vector adds + 1 RED per thread per two
//     states, against 2 x (16 LDS + 14 FADD + 2 RED) before, and half as many __syncthreads.
#include "scan_internal.h"

#include <cstdint>

namespace smb {
namespace {

constexpr int kW = 8;                      // channels (warps) per CTA
constexpr int kPad = kCkpt + 32;           // padded shared row: position p lives at p + (p >> 5) * 4
// sDA[warp][lane][state]: partials of up to 32 states (64 states: two passes), pitch coprime with the bank count
template <int N> constexpr int da_pitch() { return N <= 16 ? 17 : 33; }
static_assert(kRun * 32 == kCkpt, "R3 chunk must equal the checkpoint interval");

__device__ __forceinline__ int padp(int p) { return p + ((p >> 5) << 2); }

// ---- Kogge-Stone steps of the affine-map scan (A, H): value <- A * value_from_partner + H,  A <- A * A_partner ----
// up: lane combines with lane - O (forward recurrence);  down: with lane + O (adjoint recurrence).
template <int O, bool LAST>
__device__ __forceinline__ void ks_up(float &As, float &Hs, int lane) {
#ifdef SMB_EMU
    const float Au = __shfl_up_sync(0xffffffffu, As, O), Hu = __shfl_up_sync(0xffffffffu, Hs, O);
    if (lane >= O) { Hs = fmaf(As, Hu, Hs); if (!LAST) As *= Au; }
#else
    (void)lane;
    if (LAST) {
        asm volatile("{\n\t.reg .pred p;\n\t.reg .f32 hu;\n\t"
                     "shfl.sync.up.b32 hu|p, %0, %2, 0, 0xffffffff;\n\t"
                     "@p fma.rn.f32 %0, %1, hu, %0;\n\t}"
                     : "+f"(Hs) : "f"(As), "n"(O));
    } else {
        asm volatile("{\n\t.reg .pred p;\n\t.reg .f32 au, hu;\n\t"
                     "shfl.sync.up.b32 au|p, %0, %2, 0, 0xffffffff;\n\t"
                     "shfl.sync.up.b32 hu, %1, %2, 0, 0xffffffff;\n\t"
                     "@p fma.rn.f32 %1, %0, hu, %1;\n\t"
                     "@p mul.rn.f32 %0, %0, au;\n\t}"
                     : "+f"(As), "+f"(Hs) : "n"(O));
    }
#endif
}
template <int O, bool LAST>
__device__ __forceinline__ void ks_down(float &As, float &Hs, int lane) {
#ifdef SMB_EMU
    const float Ad = __shfl_down_sync(0xffffffffu, As, O), Hd = __shfl_down_sync(0xffffffffu, Hs, O);
    if (lane + O < 32) { Hs = fmaf(As, Hd, Hs); if (!LAST) As *= Ad; }
#else
    (void)lane;
    if (LAST) {
        asm volatile("{\n\t.reg .pred p;\n\t.reg .f32 hd;\n\t"
                     "shfl.sync.down.b32 hd|p, %0, %2, 0x1f, 0xffffffff;\n\t"
                     "@p fma.rn.f32 %0, %1, hd, %0;\n\t}"
                     : "+f"(Hs) : "f"(As), "n"(O));
    } else {
        asm volatile("{\n\t.reg .pred p;\n\t.reg .f32 ad, hd;\n\t"
                     "shfl.sync.down.b32 ad|p, %0, %2, 0x1f, 0xffffffff;\n\t"
                     "shfl.sync.down.b32 hd, %1, %2, 0x1f, 0xffffffff;\n\t"
                     "@p fma.rn.f32 %1, %0, hd, %1;\n\t"
                     "@p mul.rn.f32 %0, %0, ad;\n\t}"
                     : "+f"(As), "+f"(Hs) : "n"(O));
    }
#endif
}
// value of the neighbouring lane (lane - 1 / lane + 1); the edge lane keeps `edge`
__device__ __forceinline__ float from_left(float v, float edge, int lane) {
#ifdef SMB_EMU
    const float t = __shfl_up_sync(0xffffffffu, v, 1);
    return lane == 0 ? edge : t;
#else
    (void)lane;
    asm volatile("{\n\t.reg .pred p;\n\t.reg .f32 t;\n\t"
                 "shfl.sync.up.b32 t|p, %1, 1, 0, 0xffffffff;\n\t"
                 "@p mov.f32 %0, t;\n\t}"
                 : "+f"(edge) : "f"(v));
    return edge;
#endif
}
__device__ __forceinline__ float from_right(float v, float edge, int lane) {
#ifdef SMB_EMU
    const float t = __shfl_down_sync(0xffffffffu, v, 1);
    return lane == 31 ? edge : t;
#else
    (void)lane;
    asm volatile("{\n\t.reg .pred p;\n\t.reg .f32 t;\n\t"
                 "shfl.sync.down.b32 t|p, %1, 1, 0x1f, 0xffffffff;\n\t"
                 "@p mov.f32 %0, t;\n\t}"
                 : "+f"(edge) : "f"(v));
    return edge;
#endif
}

// ---- one state of one channel: everything that needs h and lambda at the same (position, state) ----
// Writes this lane's 8 dB / dC terms into the warp's slab rows and its dA partial into sda[n]; accumulates the per-position
// sums over states (lambda B, A lambda (h - b), C h) in place.
// kDense (scan-free): h_in / m_in are THIS lane's own values -- the saved state entering its run and the adjoint entering it
// from the right -- so the lane aggregates, both Kogge-Stone scans and the neighbour exchanges disappear.
template <bool kDense>
__device__ __forceinline__ void r3_state(const float *__restrict__ rowB, const float *__restrict__ rowC, float A2n, float h_in,
                                         float m_in, float sumdt, int lane, const float2 (&dt2)[kRun / 2],
                                         const float2 (&dtu2)[kRun / 2], const float2 (&g2)[kRun / 2], float2 (&sLB2)[kRun / 2],
                                         float2 (&sAq2)[kRun / 2], float2 (&yy2)[kRun / 2], float *__restrict__ myB,
                                         float *__restrict__ myC, float *__restrict__ sda_n) {
    float2 Bv2[kRun / 2], Cv2[kRun / 2];
    {
        const float4 b0 = *reinterpret_cast<const float4 *>(rowB), b1 = *reinterpret_cast<const float4 *>(rowB + 4);
        const float4 c0 = *reinterpret_cast<const float4 *>(rowC), c1 = *reinterpret_cast<const float4 *>(rowC + 4);
        Bv2[0] = f2(b0.x, b0.y); Bv2[1] = f2(b0.z, b0.w); Bv2[2] = f2(b1.x, b1.y); Bv2[3] = f2(b1.z, b1.w);
        Cv2[0] = f2(c0.x, c0.y); Cv2[1] = f2(c0.z, c0.w); Cv2[2] = f2(c1.x, c1.y); Cv2[3] = f2(c1.z, c1.w);
    }
    const float2 A2n2 = f2(A2n, A2n);
    float2 a2[kRun / 2], bb2[kRun / 2], gc2[kRun / 2], agc2[kRun / 2], hs2[kRun / 2], lam2[kRun / 2];
#pragma unroll
    for (int j = 0; j < kRun / 2; ++j) {
        a2[j] = ex2x2_mufu(fmul2(dt2[j], A2n2));
        bb2[j] = fmul2(dtu2[j], Bv2[j]);
        gc2[j] = fmul2(g2[j], Cv2[j]);
        agc2[j] = fmul2(a2[j], gc2[j]);
    }
    if constexpr (kDense) {
        float h = h_in;
#pragma unroll
        for (int j = 0; j < kRun / 2; ++j) {
            h = fmaf(a2[j].x, h, bb2[j].x); hs2[j].x = h;
            h = fmaf(a2[j].y, h, bb2[j].y); hs2[j].y = h;
        }
        float m = m_in;                                    // mu entering this run from the right
#pragma unroll
        for (int j = kRun / 2 - 1; j >= 0; --j) {
            const float my = m; m = fmaf(a2[j].y, m, agc2[j].y);
            const float mx = m; m = fmaf(a2[j].x, m, agc2[j].x);
            lam2[j] = fadd2(gc2[j], f2(mx, my));      // lambda_i = g_i C_i + mu_{i+1}
        }
    } else {
    const float Aagg = ex2(A2n * sumdt);               // product of the run's eight decays
    // ---- forward: lane aggregate, inclusive scan (h_in folded into lane 0), state entering the run, re-run ----
    float Hagg = 0.f;
#pragma unroll
    for (int j = 0; j < kRun / 2; ++j) {
        Hagg = fmaf(a2[j].x, Hagg, bb2[j].x);
        Hagg = fmaf(a2[j].y, Hagg, bb2[j].y);
    }
    if (lane == 0) Hagg = fmaf(Aagg, h_in, Hagg);
    {
        float As = Aagg, Hs = Hagg;
        ks_up<1, false>(As, Hs, lane); ks_up<2, false>(As, Hs, lane); ks_up<4, false>(As, Hs, lane);
        ks_up<8, false>(As, Hs, lane); ks_up<16, true>(As, Hs, lane);
        float h = from_left(Hs, h_in, lane);
#pragma unroll
        for (int j = 0; j < kRun / 2; ++j) {
            h = fmaf(a2[j].x, h, bb2[j].x); hs2[j].x = h;
            h = fmaf(a2[j].y, h, bb2[j].y); hs2[j].y = h;
        }
    }
    // ---- adjoint: mu_i = a_i (mu_{i+1} + g_i C_i) = a_i mu_{i+1} + (a g C)_i ; m_in folded into lane 31 ----
    float Magg = 0.f;
#pragma unroll
    for (int j = kRun / 2 - 1; j >= 0; --j) {
        Magg = fmaf(a2[j].y, Magg, agc2[j].y);
        Magg = fmaf(a2[j].x, Magg, agc2[j].x);
    }
    if (lane == 31) Magg = fmaf(Aagg, m_in, Magg);
    {
        float Ar = Aagg, Mr = Magg;
        ks_down<1, false>(Ar, Mr, lane); ks_down<2, false>(Ar, Mr, lane); ks_down<4, false>(Ar, Mr, lane);
        ks_down<8, false>(Ar, Mr, lane); ks_down<16, true>(Ar, Mr, lane);
        float m = from_right(Mr, m_in, lane);          // mu entering this run from the right
#pragma unroll
        for (int j = kRun / 2 - 1; j >= 0; --j) {
            const float my = m; m = fmaf(a2[j].y, m, agc2[j].y);
            const float mx = m; m = fmaf(a2[j].x, m, agc2[j].x);
            lam2[j] = fadd2(gc2[j], f2(mx, my));  // lambda_i = g_i C_i + mu_{i+1}
        }
    }
    }   // !kDense
    // ---- element-wise gradient terms, two positions per instruction ----
    float2 dA2 = f2(0.f, 0.f), dB2[kRun / 2], dC2[kRun / 2];
#pragma unroll
    for (int j = 0; j < kRun / 2; ++j) {
        yy2[j] = ffma2(Cv2[j], hs2[j], yy2[j]);
        dC2[j] = fmul2(g2[j], hs2[j]);
        dB2[j] = fmul2(lam2[j], dtu2[j]);
        sLB2[j] = ffma2(lam2[j], Bv2[j], sLB2[j]);
        const float2 hm = ffma2(bb2[j], f2(-1.f, -1.f), hs2[j]);     // h - b = a h_prev
        const float2 qv = fmul2(lam2[j], hm);
        dA2 = ffma2(dt2[j], qv, dA2);
        sAq2[j] = ffma2(A2n2, qv, sAq2[j]);
    }
    *sda_n = dA2.x + dA2.y;
    *reinterpret_cast<float4 *>(myB) = make_float4(dB2[0].x, dB2[0].y, dB2[1].x, dB2[1].y);
    *reinterpret_cast<float4 *>(myB + 4) = make_float4(dB2[2].x, dB2[2].y, dB2[3].x, dB2[3].y);
    *reinterpret_cast<float4 *>(myC) = make_float4(dC2[0].x, dC2[0].y, dC2[1].x, dC2[1].y);
    *reinterpret_cast<float4 *>(myC + 4) = make_float4(dC2[2].x, dC2[2].y, dC2[3].x, dC2[3].y);
}

template <int N> struct R3Smem {
    static constexpr int kBC = 2 * N * kPad;              // sB, sC
    static constexpr int kSlab = 2 * 2 * kW * kPad;       // [state of the round][tensor][warp][kPad]
    static constexpr int kDa = kW * 32 * da_pitch<N>();
    static constexpr size_t kBytes = sizeof(float) * (size_t)(kBC + kSlab + kDa);
};

template <typename T, int N, bool kHasZ, bool kDense>
__global__ void __launch_bounds__(kW * 32, scan_minb<N>(2)) scan_bwd_main2_kernel(const ScanP p) {
    extern __shared__ __align__(16) float smem[];
    float *sB = smem;                                   // [N][kPad]
    float *sC = sB + N * kPad;                          // [N][kPad]
    float *slab = sC + N * kPad;                        // [2][2][kW][kPad]
    float *sDA = slab + R3Smem<N>::kSlab;               // [kW][32][da_pitch]
    constexpr int kDaPitch = da_pitch<N>();

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int chunk = blockIdx.x, b = blockIdx.z;
    // blockIdx.y = (B/C group, run of p.opc consecutive channel octets of that group): the CTA stages the chunk's B / C tile once
    // and walks its octets one after the other, prefetching the next octet's operands into L2 while it works on the current one
    const int octs_per_group = (p.dim_per_group + kW - 1) / kW;
    const int runs_per_group = (octs_per_group + p.opc - 1) / p.opc;
    const int g = blockIdx.y / runs_per_group;
    const int oct_begin = (blockIdx.y - g * runs_per_group) * p.opc;
    const int oct_end = min(octs_per_group, oct_begin + p.opc);
    const int jc = chunk * kCkpt;
    const int jl = jc + lane * kRun;
    const bool rev = p.reverse;
    const int L = p.L;

    // ---- stage B and C for the chunk: thread t <-> position jc + t; all 2N loads in flight before the first store ----
    if constexpr (N > 32) {
        stage_bc_rounds<T, N, kPad>(sB, sC, reinterpret_cast<const T *>(p.B) + b * p.B_bs + (int64_t)g * p.B_gs,
                                    reinterpret_cast<const T *>(p.C) + b * p.C_bs + (int64_t)g * p.C_gs, p.B_ns, p.C_ns, p.B_ls, p.C_ls,
                                    jc, L, rev, threadIdx.x, padp(threadIdx.x));
    } else
    {
        const T *Bm = reinterpret_cast<const T *>(p.B) + b * p.B_bs + (int64_t)g * p.B_gs;
        const T *Cm = reinterpret_cast<const T *>(p.C) + b * p.C_bs + (int64_t)g * p.C_gs;
        const int t = threadIdx.x;
        const int j = jc + t;
        const bool valid = j < L;
        const int tok = pos_to_tok(valid ? j : 0, L, rev);
        const int so = padp(t);
        T vb[N], vc[N];
#pragma unroll
        for (int n = 0; n < N; ++n) {
            vb[n] = valid ? Bm[(int64_t)n * p.B_ns + (int64_t)tok * p.B_ls] : from_f32<T>(0.f);
            vc[n] = valid ? Cm[(int64_t)n * p.C_ns + (int64_t)tok * p.C_ls] : from_f32<T>(0.f);
        }
#pragma unroll
        for (int n = 0; n < N; ++n) {
            sB[n * kPad + so] = to_f32<T>(vb[n]);
            sC[n * kPad + so] = to_f32<T>(vc[n]);
        }
    }

    const int bo = padp(lane * kRun);                   // this lane's run inside a padded row
    float *myB0 = slab + (0 * kW + warp) * kPad + bo;   // state 0 of the round: dB row, dC row
    float *myC0 = slab + (1 * kW + warp) * kPad + bo;
    float *myB1 = slab + (2 * kW + warp) * kPad + bo;   // state 1 of the round
    float *myC1 = slab + (3 * kW + warp) * kPad + bo;
    float *sda = sDA + (warp * 32 + lane) * kDaPitch;
    // reduction role of this thread: (state of the round, tensor) x 4 consecutive positions
    const int combo = threadIdx.x >> 6, pg = threadIdx.x & 63;
    const int rpos0 = jc + 4 * pg;
    const float *rsrc = slab + (size_t)combo * kW * kPad + padp(4 * pg);
    float *const rdst0 = ((combo & 1) ? p.dC : p.dB) + (((int64_t)b * p.G + g) * N + (combo >> 1)) * (int64_t)L;
    const bool vec_ok = (L & 3) == 0 && ((reinterpret_cast<uintptr_t>(p.dB) | reinterpret_cast<uintptr_t>(p.dC)) & 15) == 0;

    // L2 prefetch of one octet's operand runs (16 bytes per lane and tensor) and dense checkpoints
    auto prefetch_octet = [&](int oct) {
        const int dd0 = g * p.dim_per_group + oct * kW;
        const int dd = dd0 + warp;
        if (dd >= (g + 1) * p.dim_per_group || jl >= L) return;
        const int tok = rev ? max(L - 1 - jl - 7, 0) : jl;
        prefetch_l2(reinterpret_cast<const T *>(p.u) + b * p.u_bs + (int64_t)dd * p.u_ds + tok);
        prefetch_l2(reinterpret_cast<const T *>(p.delta) + b * p.delta_bs + (int64_t)dd * p.delta_ds + tok);
        prefetch_l2(reinterpret_cast<const T *>(p.dout) + b * p.dout_bs + (int64_t)dd * p.dout_ds + tok);
        if (kHasZ) prefetch_l2(reinterpret_cast<const T *>(p.z) + b * p.z_bs + (int64_t)dd * p.z_ds + tok);
        if (kDense) {
            const int64_t slot = dense_slot(p, b, g, dd, chunk * 32 + lane, N);
            prefetch_l2(p.hd + slot);
            if (lane < 31) prefetch_l2(p.md + slot);
        }
    };

#pragma unroll 1
    for (int oct = oct_begin; oct < oct_end; ++oct) {
    const int d0 = g * p.dim_per_group + oct * kW;
    const int nch = min(kW, (g + 1) * p.dim_per_group - d0);
    const int d = d0 + warp;
    const bool active = warp < nch;

    // ---- per-lane runs ----
    float dt[kRun], uu[kRun], gg[kRun];
    float bias = 0.f, Dv = 0.f;
    if (active) {
        bias = p.delta_bias ? p.delta_bias[d] : 0.f;
        Dv = p.D ? p.D[d] : 0.f;
        const T *ur = reinterpret_cast<const T *>(p.u) + b * p.u_bs + (int64_t)d * p.u_ds;
        const T *dr = reinterpret_cast<const T *>(p.delta) + b * p.delta_bs + (int64_t)d * p.delta_ds;
        const T *gr = reinterpret_cast<const T *>(p.dout) + b * p.dout_bs + (int64_t)d * p.dout_ds;
        load_run8<T>(ur, jl, L, rev, uu);
        load_run8<T>(dr, jl, L, rev, dt);
        load_run8<T>(gr, jl, L, rev, gg);
        if (kHasZ) {
            float zz[kRun];
            const T *zr = reinterpret_cast<const T *>(p.z) + b * p.z_bs + (int64_t)d * p.z_ds;
            load_run8<T>(zr, jl, L, rev, zz);
#pragma unroll
            for (int i = 0; i < kRun; ++i) gg[i] *= zz[i] * sigmoidf(zz[i]);
        }
#pragma unroll
        for (int i = 0; i < kRun; ++i) {
            float v = dt[i] + bias;
            if (p.softplus) v = softplus20(v);
            dt[i] = (jl + i < L) ? v : 0.f;             // masked positions are scan identities (a=1, b=0)
        }
    } else {
#pragma unroll
        for (int i = 0; i < kRun; ++i) { dt[i] = 0.f; uu[i] = 0.f; gg[i] = 0.f; }
    }
    if (oct + 1 < oct_end) prefetch_octet(oct + 1);

    if (!active) {                                      // rows of absent channels stay zero for the whole octet
        const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
        *reinterpret_cast<float4 *>(myB0) = z4; *reinterpret_cast<float4 *>(myB0 + 4) = z4;
        *reinterpret_cast<float4 *>(myC0) = z4; *reinterpret_cast<float4 *>(myC0 + 4) = z4;
        *reinterpret_cast<float4 *>(myB1) = z4; *reinterpret_cast<float4 *>(myB1 + 4) = z4;
        *reinterpret_cast<float4 *>(myC1) = z4; *reinterpret_cast<float4 *>(myC1 + 4) = z4;
    }

    // per-state scalars of this channel, loaded once: lane n & 31 holds (A2, h_in, m_in) of state n, broadcast by shuffle
    float A2_l = 0.f, hin_l = 0.f, min_l = 0.f;
    if (active && lane < N) {
        A2_l = p.A[(int64_t)d * N + lane] * kLog2e;
        if (!kDense) hin_l = p.hs[(int64_t)b * p.hs_bs + ((int64_t)chunk * N + lane) * p.dim + d];
        min_l = p.Min[(((int64_t)b * p.nck + chunk) * N + lane) * p.dim + d];
    }
    float A2_h = 0.f, hin_h = 0.f, min_h = 0.f;         // states 32..63 (64 states only)
    if constexpr (N > 32) {
        if (active) {
            A2_h = p.A[(int64_t)d * N + 32 + lane] * kLog2e;
            if (!kDense) hin_h = p.hs[(int64_t)b * p.hs_bs + ((int64_t)chunk * N + 32 + lane) * p.dim + d];
            min_h = p.Min[(((int64_t)b * p.nck + chunk) * N + 32 + lane) * p.dim + d];
        }
    }
    float dA_lo = 0.f;                                  // 64 states: dA of state `lane`, reduced after the first 32 states
    // scan-free path: this lane's own checkpoints (state entering its run; local adjoint entering it from the right, which R1
    // computed with a zero adjoint at the chunk end -- the carried adjoint Min comes in through the decay product below)
    const float *hdp = nullptr, *mdp = nullptr;
    bool use_h = false, use_m = false;
    if (kDense) {
        const int64_t slot = dense_slot(p, b, g, active ? d : d0, chunk * 32 + lane, N);
        hdp = p.hd + slot;
        mdp = p.md + slot;
        use_h = active && jl < L;                       // blocks past the end were never written
        use_m = use_h && lane < 31 && jl + kRun < L;    // the chunk's / sequence's last block starts from Min alone
    }
    float2 dt2[kRun / 2], dtu2[kRun / 2], g2[kRun / 2], sLB2[kRun / 2], sAq2[kRun / 2], yy2[kRun / 2];
    float sumdt = 0.f;
#pragma unroll
    for (int j = 0; j < kRun / 2; ++j) {
        dt2[j] = f2(dt[2 * j], dt[2 * j + 1]);
        dtu2[j] = f2(dt[2 * j] * uu[2 * j], dt[2 * j + 1] * uu[2 * j + 1]);
        g2[j] = f2(gg[2 * j], gg[2 * j + 1]);
        sLB2[j] = f2(0.f, 0.f); sAq2[j] = f2(0.f, 0.f); yy2[j] = f2(0.f, 0.f);
        sumdt += dt[2 * j] + dt[2 * j + 1];
    }
    // sum of dt over the lanes to the right (exclusive suffix): the decay from the chunk end back to this run is ex2(A * suffix)
    float suffix = 0.f;
    if (kDense) {
        float inc = sumdt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const float t = __shfl_down_sync(0xffffffffu, inc, o);
            if (lane + o < 32) inc += t;
        }
        // the right neighbour's inclusive sum, not inc - sumdt: a non-finite dt of this run must not reach its own decay
        const float right = __shfl_down_sync(0xffffffffu, inc, 1);
        suffix = lane < 31 ? right : 0.f;
    }

    float *rdst = rdst0;
    __syncthreads();   // B/C tiles (first octet) and the zero rows are ready; the previous octet's reductions are done

    const float *rowB = sB + bo, *rowC = sC + bo;
    // dense checkpoints of the state pair one round ahead (a global load issued a round early, consumed after ~2 x 100 instructions)
    float2 hv_nx = f2(0.f, 0.f), mv_nx = f2(0.f, 0.f);
    if (kDense) {
        if (use_h) hv_nx = *reinterpret_cast<const float2 *>(hdp);
        if (use_m) mv_nx = *reinterpret_cast<const float2 *>(mdp);
    }
#pragma unroll 1
    for (int n = 0; n < N; n += 2) {
        const float A2a = state_shfl<N>(A2_l, A2_h, n), A2b = state_shfl<N>(A2_l, A2_h, n + 1);
        const float hia = state_shfl<N>(hin_l, hin_h, n), hib = state_shfl<N>(hin_l, hin_h, n + 1);
        const float mia = state_shfl<N>(min_l, min_h, n), mib = state_shfl<N>(min_l, min_h, n + 1);
        if (active && !(p.dbg & 4)) {
            if constexpr (kDense) {
                const float2 hv = hv_nx, mv = mv_nx;
                if (n + 2 < N) {
                    if (use_h) hv_nx = *reinterpret_cast<const float2 *>(hdp + n + 2);
                    if (use_m) mv_nx = *reinterpret_cast<const float2 *>(mdp + n + 2);
                }
                const float ma = fmaf(ex2(A2a * suffix), mia, mv.x), mb = fmaf(ex2(A2b * suffix), mib, mv.y);
                r3_state<true>(rowB, rowC, A2a, hv.x, ma, sumdt, lane, dt2, dtu2, g2, sLB2, sAq2, yy2, myB0, myC0, sda + (N > 32 ? (n & 31) : n));
                r3_state<true>(rowB + kPad, rowC + kPad, A2b, hv.y, mb, sumdt, lane, dt2, dtu2, g2, sLB2, sAq2, yy2, myB1, myC1, sda + (N > 32 ? (n & 31) : n) + 1);
            } else {
                r3_state<false>(rowB, rowC, A2a, hia, mia, sumdt, lane, dt2, dtu2, g2, sLB2, sAq2, yy2, myB0, myC0, sda + (N > 32 ? (n & 31) : n));
                r3_state<false>(rowB + kPad, rowC + kPad, A2b, hib, mib, sumdt, lane, dt2, dtu2, g2, sLB2, sAq2, yy2, myB1, myC1, sda + (N > 32 ? (n & 31) : n) + 1);
            }
        }
        if constexpr (N > 32) {
            if (n == 30 && active) {                    // states 0..31 complete: free the partial buffer for states 32..63
                __syncwarp();
                const float *col = sDA + (warp * 32) * kDaPitch + lane;
                float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
                for (int k = 0; k < 32; k += 4) {
                    s0 += col[(k + 0) * kDaPitch]; s1 += col[(k + 1) * kDaPitch];
                    s2 += col[(k + 2) * kDaPitch]; s3 += col[(k + 3) * kDaPitch];
                }
                dA_lo = (s0 + s1) + (s2 + s3);
                __syncwarp();
            }
        }
        rowB += 2 * kPad; rowC += 2 * kPad;
        __syncthreads();
        // ---- reduce dB / dC of the two states over the CTA's channels: 16-byte vectors, fixed trip count ----
        if (rpos0 < L && !(p.dbg & 2)) {
            float4 v[kW];
#pragma unroll
            for (int w2 = 0; w2 < kW; ++w2) v[w2] = *reinterpret_cast<const float4 *>(rsrc + w2 * kPad);
            const float2 lo = fadd2(fadd2(fadd2(f2(v[0].x, v[0].y), f2(v[1].x, v[1].y)),
                                                    fadd2(f2(v[2].x, v[2].y), f2(v[3].x, v[3].y))),
                                         fadd2(fadd2(f2(v[4].x, v[4].y), f2(v[5].x, v[5].y)),
                                                    fadd2(f2(v[6].x, v[6].y), f2(v[7].x, v[7].y))));
            const float2 hi = fadd2(fadd2(fadd2(f2(v[0].z, v[0].w), f2(v[1].z, v[1].w)),
                                                    fadd2(f2(v[2].z, v[2].w), f2(v[3].z, v[3].w))),
                                         fadd2(fadd2(f2(v[4].z, v[4].w), f2(v[5].z, v[5].w)),
                                                    fadd2(f2(v[6].z, v[6].w), f2(v[7].z, v[7].w))));
            if (p.dbg & 1) {
                if (lo.x == 1.2345e33f) rdst[0] = hi.y;      // keep the sums live
            } else if (vec_ok && rpos0 + 3 < L) {
                if (!rev) red_add_v4(rdst + rpos0, lo.x, lo.y, hi.x, hi.y);
                else red_add_v4(rdst + (L - 4 - rpos0), hi.y, hi.x, lo.y, lo.x);
            } else {
                const float rr[4] = {lo.x, lo.y, hi.x, hi.y};
#pragma unroll
                for (int e = 0; e < 4; ++e)
                    if (rpos0 + e < L) atomicAdd(rdst + pos_to_tok(rpos0 + e, L, rev), rr[e]);
            }
        }
        rdst += 2 * (int64_t)L;
        __syncthreads();
    }

    if (active) {
    // ---- dA: column sums of this warp's (lane, state) partials ----
    __syncwarp();
    if (lane < N) {
        const float *col = sDA + (warp * 32) * kDaPitch + lane;
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
        for (int k = 0; k < 32; k += 4) {
            s0 += col[(k + 0) * kDaPitch]; s1 += col[(k + 1) * kDaPitch];
            s2 += col[(k + 2) * kDaPitch]; s3 += col[(k + 3) * kDaPitch];
        }
        if constexpr (N > 32) {
            atomicAdd(p.dA + (int64_t)d * N + lane, dA_lo);
            atomicAdd(p.dA + (int64_t)d * N + 32 + lane, (s0 + s1) + (s2 + s3));
        } else {
            atomicAdd(p.dA + (int64_t)d * N + lane, (s0 + s1) + (s2 + s3));
        }
    }
    __syncwarp();                                        // the next octet's partials overwrite these rows
    float sLB[kRun], sAq[kRun], yy[kRun];
#pragma unroll
    for (int j = 0; j < kRun / 2; ++j) {
        sLB[2 * j] = sLB2[j].x; sLB[2 * j + 1] = sLB2[j].y;
        sAq[2 * j] = sAq2[j].x; sAq[2 * j + 1] = sAq2[j].y;
        yy[2 * j] = yy2[j].x; yy[2 * j + 1] = yy2[j].y;
    }
    // ---- epilogue: du, ddelta, dz, (out_z), dD, ddelta_bias ----
    float duv[kRun], ddv[kRun];
    float dDacc = 0.f, dbacc = 0.f;
#pragma unroll
    for (int i = 0; i < kRun; ++i) {
        duv[i] = fmaf(dt[i], sLB[i], Dv * gg[i]);
        float ddt = fmaf(uu[i], sLB[i], kLn2 * sAq[i]);
        if (p.softplus) ddt *= one_minus_exp_neg(dt[i]); // sigmoid(raw) == 1 - exp(-softplus(raw))
        if (jl + i >= L) ddt = 0.f;
        ddv[i] = ddt;
        dDacc = fmaf(gg[i], uu[i], dDacc);
        dbacc += ddt;
    }
    {
        T *dur = reinterpret_cast<T *>(p.du) + b * p.du_bs + (int64_t)d * p.du_ds;
        T *ddr = reinterpret_cast<T *>(p.ddelta) + b * p.ddelta_bs + (int64_t)d * p.ddelta_ds;
        store_run8<T>(dur, jl, L, rev, duv);
        store_run8<T>(ddr, jl, L, rev, ddv);
    }
    if (kHasZ) {
        float zz[kRun], go[kRun], dzv[kRun], ozv[kRun];
        const T *zr = reinterpret_cast<const T *>(p.z) + b * p.z_bs + (int64_t)d * p.z_ds;
        const T *gr = reinterpret_cast<const T *>(p.dout) + b * p.dout_bs + (int64_t)d * p.dout_ds;
        load_run8<T>(zr, jl, L, rev, zz);
        load_run8<T>(gr, jl, L, rev, go);
#pragma unroll
        for (int i = 0; i < kRun; ++i) {
            const float y = fmaf(Dv, uu[i], yy[i]);
            const float sg = sigmoidf(zz[i]);
            dzv[i] = go[i] * y * sg * (1.f + zz[i] * (1.f - sg));
            ozv[i] = y * zz[i] * sg;
        }
        T *dzr = reinterpret_cast<T *>(p.dz) + b * p.dz_bs + (int64_t)d * p.dz_ds;
        store_run8<T>(dzr, jl, L, rev, dzv);
        if (p.out_z) {
            T *ozr = reinterpret_cast<T *>(p.out_z) + b * p.out_z_bs + (int64_t)d * p.out_z_ds;
            store_run8<T>(ozr, jl, L, rev, ozv);
        }
    }
    dDacc = warp_sum(dDacc);
    dbacc = warp_sum(dbacc);
    if (lane == 0) {
        if (p.dD) atomicAdd(p.dD + d, dDacc);
        if (p.ddelta_bias) atomicAdd(p.ddelta_bias + d, dbacc);
    }
    }   // active
    }   // octets
}

template <typename T, int N, bool kHasZ>
cudaError_t launch_main2(const ScanP &p, cudaStream_t st) {
    const size_t sm = R3Smem<N>::kBytes;
    cudaError_t e;
    // octets per CTA: as many as keeps >= ~4 CTAs per resident slot (8 x 132 SMs) in the grid
    const int opg = (p.dim_per_group + kW - 1) / kW;
    ScanP q = p;
    {
        const long total = (long)p.nck * opg * p.G * p.batch;
        long opc = total / 1056;
        if (opc < 1) opc = 1;
        if (opc > opg) opc = opg;
        const char *e = getenv("SMB_R3_OPC");            // A/B switch: octets per CTA (1 = one CTA per octet, as in round 1)
        if (e && atoi(e) > 0) opc = atoi(e) > opg ? opg : atoi(e);
        q.opc = (int)opc;
    }
    const int runs = ((opg + q.opc - 1) / q.opc) * p.G;
    dim3 grid(p.nck, runs, p.batch);
    if (p.hd && p.md) {
        SMB_SET_SMEM_ONCE((scan_bwd_main2_kernel<T, N, kHasZ, true>), sm);
        scan_bwd_main2_kernel<T, N, kHasZ, true><<<grid, kW * 32, sm, st>>>(q); count_launch();
    } else {
        SMB_SET_SMEM_ONCE((scan_bwd_main2_kernel<T, N, kHasZ, false>), sm);
        scan_bwd_main2_kernel<T, N, kHasZ, false><<<grid, kW * 32, sm, st>>>(q); count_launch();
    }
    return cudaGetLastError();
}
template <typename T>
cudaError_t launch_main2_t(const ScanP &p, int N, bool has_z, cudaStream_t st) {
    switch (N) {
        case 64: return has_z ? launch_main2<T, 64, true>(p, st) : launch_main2<T, 64, false>(p, st);
        case 32: return has_z ? launch_main2<T, 32, true>(p, st) : launch_main2<T, 32, false>(p, st);
        case 16: return has_z ? launch_main2<T, 16, true>(p, st) : launch_main2<T, 16, false>(p, st);
        default: return has_z ? launch_main2<T, 8, true>(p, st) : launch_main2<T, 8, false>(p, st);
    }
}

}  // namespace

cudaError_t scan_bwd_main_v2_dispatch(const ScanP &p, int dtype, int N, bool has_z, cudaStream_t st) {
    switch (dtype) {
        case 0: return launch_main2_t<float>(p, N, has_z, st);
        case 1: return launch_main2_t<__half>(p, N, has_z, st);
        default: return launch_main2_t<__nv_bfloat16>(p, N, has_z, st);
    }
}

}  // namespace smb
