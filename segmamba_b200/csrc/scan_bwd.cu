// Backward selective scan for sm_90a: chunk-parallel, three passes over 256-position chunks.
//
//   R1  scan_bwd_ragg_kernel  lane-per-channel reverse walk of each chunk with zero incoming adjoint:
//                             (P = prod a, Mloc = adjoint at the chunk start)                     [1 ex2 / update]
//   R2  carry_kernel          reverse exclusive scan of (P, Mloc) over chunks -> Min per chunk    [tiny]
//   R3  scan_bwd_main_kernel  warp-per-channel, 8 positions per lane in registers: forward state recompute
//                             seeded from the saved chunk state, reverse adjoint scan seeded from Min, all
//                             gradients; dB/dC are reduced over the CTA's channels in shared memory before
//                             ONE fp32 atomic per (state, position) per CTA (the reference issues one per
//                             channel, selective_scan_bwd_kernel.cuh:297-316)                      [1 ex2 / update]
//
// Adjoint recurrence in "mu" form (mu_t = a_t lambda_t, the gradient w.r.t. h_{t-1}), which needs no
// a_{t+1} look-ahead across lanes/chunks (the reference fetches it through smem_delta_a, :244-262):
//     lambda_t = g_t C_t + mu_{t+1},      mu_t = a_t lambda_t
// Gradients (SURVEY.md Appendix D / selective_scan_bwd_kernel.cuh:276-294,439-453):
//     du  = dt * sum_n lambda B + D g            ddt = u * sum_n lambda B + sum_n lambda A (h - b)
//     dA  = sum_t lambda dt (h - b)              dB  = sum_d lambda dt u        dC = sum_d g h
//     ddelta = ddt * sigmoid(delta + bias) (softplus)     dz = dout y sigmoid(z)(1 + z(1 - sigmoid(z)))
#include "scan_internal.h"
#include "scan_steps.cuh"

#include <type_traits>

namespace smb {

constexpr int kBwdWarps = 8;               // channels per CTA in R3
constexpr int kRowPad = kCkpt + 32;        // padded smem row: position p lives at p + (p>>5)*4
static_assert(kRun * 32 == kCkpt, "R3 chunk must equal the checkpoint interval");

__device__ __forceinline__ int pad_pos(int p) { return p + ((p >> 5) << 2); }

// ---------------------------------------------------------------------------------------------
// R1: reverse aggregate per chunk (lane == channel)
// ---------------------------------------------------------------------------------------------
template <typename T, int N, bool kHasZ>
__global__ void __launch_bounds__(kWarpsPerCta * 32) scan_bwd_ragg_kernel(const ScanP p) {
    extern __shared__ __align__(16) float smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int w = blockIdx.x * kWarpsPerCta + warp;
    if (w >= p.n_work) return;
    const WorkItem wi = decode_work(p, w);          // here S == kCkpt, n_seg == nck
    const int d = wi.d0 + lane;
    const bool active = lane < wi.nrows;

    float *s_dt = smem + warp * (3 * kTile * kTile + kTile * N);
    float *s_g = s_dt + kTile * kTile;
    float *s_z = s_g + kTile * kTile;
    float *s_C = s_z + kTile * kTile;

    float2 A2[N / 2], mu[N / 2];                      // state pairs packed for FFMA2
#pragma unroll
    for (int m = 0; m < N / 2; ++m) {
        A2[m] = active ? f2(p.A[(int64_t)d * N + 2 * m] * kLog2e, p.A[(int64_t)d * N + 2 * m + 1] * kLog2e) : f2(0.f, 0.f);
        mu[m] = f2(0.f, 0.f);
    }
    const float bias = (active && p.delta_bias) ? p.delta_bias[d] : 0.f;
    float sumdt = 0.f;

    const T *dl = reinterpret_cast<const T *>(p.delta) + wi.b * p.delta_bs + (int64_t)wi.d0 * p.delta_ds;
    const T *go = reinterpret_cast<const T *>(p.dout) + wi.b * p.dout_bs + (int64_t)wi.d0 * p.dout_ds;
    const T *z = kHasZ ? reinterpret_cast<const T *>(p.z) + wi.b * p.z_bs + (int64_t)wi.d0 * p.z_ds : nullptr;
    const T *Cm = reinterpret_cast<const T *>(p.C) + wi.b * p.C_bs + (int64_t)wi.g * p.C_gs;

    const int j_begin = wi.seg * kCkpt;
    const int j_end = min(p.L, j_begin + kCkpt);
    const int last_tile = j_begin + ((j_end - j_begin - 1) / kTile) * kTile;
    const bool fast = stream_aligned(dl, p.delta_ds, p.L, p.reverse) && stream_aligned(go, p.dout_ds, p.L, p.reverse) &&
                      (!kHasZ || stream_aligned(z, p.z_ds, p.L, p.reverse));
    const LanePtr<T> lps[3] = {lane_ptr(dl, p.delta_ds, p.L, p.reverse, lane), lane_ptr(go, p.dout_ds, p.L, p.reverse, lane),
                               lane_ptr(kHasZ ? z : dl, kHasZ ? p.z_ds : p.delta_ds, p.L, p.reverse, lane)};
    for (int j0 = last_tile; j0 >= j_begin; j0 -= kTile) {
        {
            constexpr int K = kHasZ ? 3 : 2;
            const T *const bases[3] = {dl, go, kHasZ ? z : dl};
            const int64_t strides[3] = {p.delta_ds, p.dout_ds, kHasZ ? p.z_ds : p.delta_ds};
            if (fast && j0 + kTile <= p.L) {
                float *const tiles[3] = {s_dt, s_g, s_z};
                fill_tiles_fast<T, K, 3>(tiles, lps, wi.nrows, j0, p.reverse, lane);
            } else {
                fill_tile<T>(s_dt, dl, p.delta_ds, wi.nrows, j0, p.L, p.reverse, lane);
                fill_tile<T>(s_g, go, p.dout_ds, wi.nrows, j0, p.L, p.reverse, lane);
                if (kHasZ) fill_tile<T>(s_z, z, p.z_ds, wi.nrows, j0, p.L, p.reverse, lane);
            }
            float *const bt[1] = {s_C};
            const T *const bb[1] = {Cm};
            const int64_t bns[1] = {p.C_ns}, bls[1] = {p.C_ls};
            fill_bc_tiles<T, N, 1>(bt, bb, bns, bls, j0, p.L, p.reverse, lane);
            if (j0 - kTile >= j_begin) {
                prefetch_tiles<T, K, 3>(bases, strides, wi.nrows, j0 - kTile, p.L, p.reverse, lane);
                prefetch_bc<T, N, 1>(bb, bns, bls, j0 - kTile, p.L, p.reverse, lane);
            }
        }
        __syncwarp();
        prepass_dt(s_dt, lane, bias, p.softplus, j_end - j0);      // masked positions: a = 1, and g == 0 there
        if (kHasZ) prepass_gate_grad(s_g, s_z, lane);
#pragma unroll 1
        for (int c0 = kTile / 4 - 2; c0 >= 0; c0 -= 2) {  // blocks of 8 positions, descending
            const float *blkC = s_C + 4 * c0 * N;
            const float4 da = tile_read4(s_dt, lane, c0), db = tile_read4(s_dt, lane, c0 + 1);
            const float4 ga = tile_read4(s_g, lane, c0), gb = tile_read4(s_g, lane, c0 + 1);
            const float dd[8] = {da.x, da.y, da.z, da.w, db.x, db.y, db.z, db.w};
            const float gg[8] = {ga.x, ga.y, ga.z, ga.w, gb.x, gb.y, gb.z, gb.w};
            ragg_block<N, 7>(blkC, gg, dd, A2, mu, sumdt);
            const int blk = (j0 + 4 * c0) >> 3;            // block just finished; its left neighbour starts its adjoint from mu
            if (p.md && active && (blk & 31)) dense_store<N>(p.md + dense_slot(p, wi.b, wi.g, d, blk - 1, N), mu);
        }
        __syncwarp();
    }
    if (active) {
        const int64_t o = (((int64_t)wi.b * p.n_seg + wi.seg) * N) * p.dim + d;
#pragma unroll
        for (int m = 0; m < N / 2; ++m) {
            p.Pb[o + (int64_t)(2 * m) * p.dim] = ex2(A2[m].x * sumdt);
            p.Pb[o + (int64_t)(2 * m + 1) * p.dim] = ex2(A2[m].y * sumdt);
            p.Mloc[o + (int64_t)(2 * m) * p.dim] = mu[m].x;
            p.Mloc[o + (int64_t)(2 * m + 1) * p.dim] = mu[m].y;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// R3: main backward kernel (warp == channel, lane == run of 8 positions, CTA == 8 channels)
// grid = (chunks, channel octets (group-aligned), batch)
// ---------------------------------------------------------------------------------------------
template <typename T, int N, bool kHasZ>
#ifdef SMB_R3_MINB
__global__ void __launch_bounds__(kBwdWarps * 32, SMB_R3_MINB) scan_bwd_main_kernel(const ScanP p) {
#else
__global__ void __launch_bounds__(kBwdWarps * 32) scan_bwd_main_kernel(const ScanP p) {
#endif
    extern __shared__ __align__(16) float smem[];
    float *sB = smem;                                  // [N][kRowPad]
    float *sC = sB + N * kRowPad;                      // [N][kRowPad]
    float *slabB = sC + N * kRowPad;                   // [kBwdWarps][kRowPad]
    float *slabC = slabB + kBwdWarps * kRowPad;        // [kBwdWarps][kRowPad]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int chunk = blockIdx.x, b = blockIdx.z;
    const int octs_per_group = (p.dim_per_group + kBwdWarps - 1) / kBwdWarps;
    const int g = blockIdx.y / octs_per_group;
    const int d0 = g * p.dim_per_group + (blockIdx.y - g * octs_per_group) * kBwdWarps;
    const int nch = min(kBwdWarps, (g + 1) * p.dim_per_group - d0);   // active channels (warps) in this CTA
    const int d = d0 + warp;
    const bool active = warp < nch;
    const int jc = chunk * kCkpt;                      // first scan position of the chunk
    const int jl = jc + lane * kRun;                   // first scan position of this lane's run
    const bool rev = p.reverse;
    const int L = p.L;

    // ---- stage B and C for the chunk: thread t <-> position jc + t; all 2N loads in flight before the first store ----
    if constexpr (N > 32) {
        stage_bc_rounds<T, N, kRowPad>(sB, sC, reinterpret_cast<const T *>(p.B) + b * p.B_bs + (int64_t)g * p.B_gs,
                                       reinterpret_cast<const T *>(p.C) + b * p.C_bs + (int64_t)g * p.C_gs, p.B_ns, p.C_ns, p.B_ls,
                                       p.C_ls, jc, L, rev, threadIdx.x, pad_pos(threadIdx.x));
    } else
    {
        const T *Bm = reinterpret_cast<const T *>(p.B) + b * p.B_bs + (int64_t)g * p.B_gs;
        const T *Cm = reinterpret_cast<const T *>(p.C) + b * p.C_bs + (int64_t)g * p.C_gs;
        const int t = threadIdx.x;
        const int j = jc + t;
        const bool valid = j < L;
        const int tok = pos_to_tok(valid ? j : 0, L, rev);
        const int so = pad_pos(t);
        T vb[N], vc[N];
#pragma unroll
        for (int n = 0; n < N; ++n) {
            vb[n] = valid ? Bm[(int64_t)n * p.B_ns + (int64_t)tok * p.B_ls] : from_f32<T>(0.f);
            vc[n] = valid ? Cm[(int64_t)n * p.C_ns + (int64_t)tok * p.C_ls] : from_f32<T>(0.f);
        }
#pragma unroll
        for (int n = 0; n < N; ++n) {
            sB[n * kRowPad + so] = to_f32<T>(vb[n]);
            sC[n * kRowPad + so] = to_f32<T>(vc[n]);
        }
    }

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
    __syncthreads();   // B/C tiles ready

    const int bo = pad_pos(lane * kRun);               // this lane's run inside a padded row
    float *myB = slabB + warp * kRowPad + bo;
    float *myC = slabC + warp * kRowPad + bo;

    // per-state scalars of this channel, loaded once: lane n & 31 holds (A2, h_in, m_in) of state n, broadcast by shuffle
    float A2_l = 0.f, hin_l = 0.f, min_l = 0.f;
    if (active && lane < N) {
        A2_l = p.A[(int64_t)d * N + lane] * kLog2e;
        hin_l = p.hs[(int64_t)b * p.hs_bs + ((int64_t)chunk * N + lane) * p.dim + d];
        min_l = p.Min[(((int64_t)b * p.nck + chunk) * N + lane) * p.dim + d];
    }
    float A2_h = 0.f, hin_h = 0.f, min_h = 0.f;         // states 32..63 (64 states only)
    if constexpr (N > 32) {
        if (active) {
            A2_h = p.A[(int64_t)d * N + 32 + lane] * kLog2e;
            hin_h = p.hs[(int64_t)b * p.hs_bs + ((int64_t)chunk * N + 32 + lane) * p.dim + d];
            min_h = p.Min[(((int64_t)b * p.nck + chunk) * N + 32 + lane) * p.dim + d];
        }
    }
    // item pairs (2j, 2j+1) packed for FFMA2
    float2 dt2[kRun / 2], dtu2[kRun / 2], g2[kRun / 2], sLB2[kRun / 2], sAq2[kRun / 2], yy2[kRun / 2];
#pragma unroll
    for (int j = 0; j < kRun / 2; ++j) {
        dt2[j] = f2(dt[2 * j], dt[2 * j + 1]);
        dtu2[j] = f2(dt[2 * j] * uu[2 * j], dt[2 * j + 1] * uu[2 * j + 1]);
        g2[j] = f2(gg[2 * j], gg[2 * j + 1]);
        sLB2[j] = f2(0.f, 0.f); sAq2[j] = f2(0.f, 0.f); yy2[j] = f2(0.f, 0.f);
    }

#pragma unroll 1
    for (int n = 0; n < N; ++n) {
        float2 dB2[kRun / 2], dC2[kRun / 2];
        const float A2n = state_shfl<N>(A2_l, A2_h, n);
        const float h_in = state_shfl<N>(hin_l, hin_h, n);
        const float m_in = state_shfl<N>(min_l, min_h, n);
        if (active) {
            float2 Bv2[kRun / 2], Cv2[kRun / 2];
            {
                const float4 b0 = *reinterpret_cast<const float4 *>(sB + n * kRowPad + bo);
                const float4 b1 = *reinterpret_cast<const float4 *>(sB + n * kRowPad + bo + 4);
                const float4 c0 = *reinterpret_cast<const float4 *>(sC + n * kRowPad + bo);
                const float4 c1 = *reinterpret_cast<const float4 *>(sC + n * kRowPad + bo + 4);
                Bv2[0] = f2(b0.x, b0.y); Bv2[1] = f2(b0.z, b0.w); Bv2[2] = f2(b1.x, b1.y); Bv2[3] = f2(b1.z, b1.w);
                Cv2[0] = f2(c0.x, c0.y); Cv2[1] = f2(c0.z, c0.w); Cv2[2] = f2(c1.x, c1.y); Cv2[3] = f2(c1.z, c1.w);
            }
            const float2 A2n2 = f2(A2n, A2n);
            float2 a2[kRun / 2], bb2[kRun / 2], gc2[kRun / 2], hs2[kRun / 2], lam2[kRun / 2];
#pragma unroll
            for (int j = 0; j < kRun / 2; ++j) {
                a2[j] = ex2x2_mufu(fmul2(dt2[j], A2n2));
                bb2[j] = fmul2(dtu2[j], Bv2[j]);
                gc2[j] = fmul2(g2[j], Cv2[j]);
            }
            // lane aggregates of the forward recurrence (sequential over the 8 positions)
            float Aagg = 1.f, Hagg = 0.f;
#pragma unroll
            for (int j = 0; j < kRun / 2; ++j) {
                Hagg = fmaf(a2[j].x, Hagg, bb2[j].x); Aagg *= a2[j].x;
                Hagg = fmaf(a2[j].y, Hagg, bb2[j].y); Aagg *= a2[j].y;
            }
            // exclusive forward warp scan -> state entering this lane's run
            float As = Aagg, Hs = Hagg;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const float Au = __shfl_up_sync(0xffffffffu, As, o), Hu = __shfl_up_sync(0xffffffffu, Hs, o);
                if (lane >= o) { Hs = fmaf(As, Hu, Hs); As *= Au; }
            }
            float Ae = __shfl_up_sync(0xffffffffu, As, 1), He = __shfl_up_sync(0xffffffffu, Hs, 1);
            if (lane == 0) { Ae = 1.f; He = 0.f; }
            float h = fmaf(Ae, h_in, He);
#pragma unroll
            for (int j = 0; j < kRun / 2; ++j) {
                h = fmaf(a2[j].x, h, bb2[j].x); hs2[j].x = h;
                h = fmaf(a2[j].y, h, bb2[j].y); hs2[j].y = h;
            }
            // lane aggregates of the reverse (adjoint) recurrence  mu_i = a_i (mu_{i+1} + g_i C_i)
            float Magg = 0.f;
#pragma unroll
            for (int j = kRun / 2 - 1; j >= 0; --j) {
                Magg = a2[j].y * (Magg + gc2[j].y);
                Magg = a2[j].x * (Magg + gc2[j].x);
            }
            float Ar = Aagg, Mr = Magg;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const float Ad = __shfl_down_sync(0xffffffffu, Ar, o), Md = __shfl_down_sync(0xffffffffu, Mr, o);
                if (lane + o < 32) { Mr = fmaf(Ar, Md, Mr); Ar *= Ad; }
            }
            float Ax = __shfl_down_sync(0xffffffffu, Ar, 1), Mx = __shfl_down_sync(0xffffffffu, Mr, 1);
            if (lane == 31) { Ax = 1.f; Mx = 0.f; }
            float m = fmaf(Ax, m_in, Mx);                // mu entering this run from the right
#pragma unroll
            for (int j = kRun / 2 - 1; j >= 0; --j) {
                lam2[j].y = gc2[j].y + m; m = a2[j].y * lam2[j].y;
                lam2[j].x = gc2[j].x + m; m = a2[j].x * lam2[j].x;
            }
            // element-wise gradient terms, two positions per instruction
            float2 dA2 = f2(0.f, 0.f);
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
            const float dAacc = warp_sum(dA2.x + dA2.y);          // dA_n = sum_t lambda dt (h - b)
            if (lane == 0) atomicAdd(p.dA + (int64_t)d * N + n, dAacc);
        } else {
#pragma unroll
            for (int j = 0; j < kRun / 2; ++j) { dB2[j] = f2(0.f, 0.f); dC2[j] = f2(0.f, 0.f); }
        }
        float dBv[kRun], dCv[kRun];
#pragma unroll
        for (int j = 0; j < kRun / 2; ++j) {
            dBv[2 * j] = dB2[j].x; dBv[2 * j + 1] = dB2[j].y;
            dCv[2 * j] = dC2[j].x; dCv[2 * j + 1] = dC2[j].y;
        }
        // ---- reduce dB / dC over the CTA's channels ----
        *reinterpret_cast<float4 *>(myB) = make_float4(dBv[0], dBv[1], dBv[2], dBv[3]);
        *reinterpret_cast<float4 *>(myB + 4) = make_float4(dBv[4], dBv[5], dBv[6], dBv[7]);
        *reinterpret_cast<float4 *>(myC) = make_float4(dCv[0], dCv[1], dCv[2], dCv[3]);
        *reinterpret_cast<float4 *>(myC + 4) = make_float4(dCv[4], dCv[5], dCv[6], dCv[7]);
        __syncthreads();
        {
            const int t = threadIdx.x;
            const int j = jc + t;
            if (j < L) {
                const int so = pad_pos(t);
                float vb[kBwdWarps], vc[kBwdWarps];   // inactive warps wrote zeros: fixed trip count, loads first
#pragma unroll
                for (int w2 = 0; w2 < kBwdWarps; ++w2) {
                    vb[w2] = slabB[w2 * kRowPad + so];
                    vc[w2] = slabC[w2 * kRowPad + so];
                }
                const float sb = ((vb[0] + vb[1]) + (vb[2] + vb[3])) + ((vb[4] + vb[5]) + (vb[6] + vb[7]));
                const float sc = ((vc[0] + vc[1]) + (vc[2] + vc[3])) + ((vc[4] + vc[5]) + (vc[6] + vc[7]));
                const int tok = pos_to_tok(j, L, rev);
                const int64_t o = (((int64_t)b * p.G + g) * N + n) * (int64_t)L + tok;
                atomicAdd(p.dB + o, sb);
                atomicAdd(p.dC + o, sc);
            }
        }
        __syncthreads();
    }

    if (!active) return;
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
        if (p.softplus) ddt *= -expm1f(-dt[i]);          // sigmoid(raw) == 1 - exp(-softplus(raw))
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
}

// =============================================================================================
// State-stash backward (default): lane == channel for every pass, no warp scans.
//   K_F  scan_bwd_stash_kernel   forward recompute from the saved 256-position states, writing every state pair
//                                h[t, 2m..2m+1] to a workspace stash (bf16x2 for 16-bit I/O, float2 for fp32 I/O)
//   R1   scan_bwd_ragg_kernel + carry (as above)
//   K_R  scan_bwd_sweep_kernel   reverse sweep: lambda_t = g_t C_t + mu_{t+1}, mu_t = a_t lambda_t, and every gradient from
//                                (lambda_t, mu_t, h_t, h_{t-1}); dB / dC are reduced over the warp's 32 channels with a
//                                shared-memory transpose and leave as one 16-byte vector atomic per (tensor, state) per
//                                4 positions per warp (red.global.add.v4.f32).
// dA / ddelta use  lambda_t a_t h_{t-1} = mu_t h_{t-1}  (no h - b cancellation).
// =============================================================================================
template <typename T> struct StashT { using type = __nv_bfloat162; };
template <> struct StashT<float> { using type = float2; };
__device__ __forceinline__ void stash_store(float2 *p, float2 v) { *p = v; }
__device__ __forceinline__ void stash_store(__nv_bfloat162 *p, float2 v) { *p = __floats2bfloat162_rn(v.x, v.y); }
__device__ __forceinline__ float2 stash_cvt(float2 v) { return v; }
__device__ __forceinline__ float2 stash_cvt(__nv_bfloat162 v) { return __bfloat1622float2(v); }
template <typename S> __device__ __forceinline__ S stash_zero();
template <> __device__ __forceinline__ float2 stash_zero<float2>() { return make_float2(0.f, 0.f); }
template <> __device__ __forceinline__ __nv_bfloat162 stash_zero<__nv_bfloat162>() { return __floats2bfloat162_rn(0.f, 0.f); }

template <int N, int QL, typename S>
__device__ __forceinline__ void stash_block(const float *blkB, const float (&uu)[8], const float (&dd)[8], const float2 (&A2)[N / 2],
                                            float2 (&h)[N / 2], S *sp, int64_t pos_stride, int64_t m_stride, bool active) {
    if constexpr (QL < 8) {
        const float dt = dd[QL], du = dt * uu[QL];
        scan_step_agg<N, QL>(blkB, f2(dt, dt), f2(du, du), A2, h);
        if (active) {
#pragma unroll
            for (int m = 0; m < N / 2; ++m) stash_store(sp + QL * pos_stride + m * m_stride, h[m]);
        }
        stash_block<N, QL + 1, S>(blkB, uu, dd, A2, h, sp, pos_stride, m_stride, active);
    }
}

template <typename T, int N>
__global__ void __launch_bounds__(kWarpsPerCta * 32) scan_bwd_stash_kernel(const ScanP p) {
    using S = typename StashT<T>::type;
    extern __shared__ __align__(16) float smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int w = blockIdx.x * kWarpsPerCta + warp;
    if (w >= p.n_work) return;
    const WorkItem wi = decode_work(p, w);          // S == kCkpt, n_seg == nck
    const int d = wi.d0 + lane;
    const bool active = lane < wi.nrows;
    float *s_u = smem + warp * (2 * kTile * kTile + kTile * N);
    float *s_dt = s_u + kTile * kTile;
    float *s_B = s_dt + kTile * kTile;
    float2 A2[N / 2], h[N / 2];
#pragma unroll
    for (int m = 0; m < N / 2; ++m) {
        A2[m] = active ? f2(p.A[(int64_t)d * N + 2 * m] * kLog2e, p.A[(int64_t)d * N + 2 * m + 1] * kLog2e) : f2(0.f, 0.f);
        const int64_t o = (int64_t)wi.b * p.hs_bs + ((int64_t)wi.seg * N + 2 * m) * p.dim + d;
        h[m] = active ? f2(p.hs[o], p.hs[o + p.dim]) : f2(0.f, 0.f);
    }
    const float bias = (active && p.delta_bias) ? p.delta_bias[d] : 0.f;
    const T *u = reinterpret_cast<const T *>(p.u) + wi.b * p.u_bs + (int64_t)wi.d0 * p.u_ds;
    const T *dl = reinterpret_cast<const T *>(p.delta) + wi.b * p.delta_bs + (int64_t)wi.d0 * p.delta_ds;
    const T *Bm = reinterpret_cast<const T *>(p.B) + wi.b * p.B_bs + (int64_t)wi.g * p.B_gs;
    const int64_t m_stride = p.dim, pos_stride = (int64_t)(N / 2) * p.dim;
    S *stash = reinterpret_cast<S *>(p.stash) + (int64_t)wi.b * p.Lpad * pos_stride + d;

    const int j_begin = wi.seg * kCkpt;
    const int j_end = min(p.L, j_begin + kCkpt);
    const bool fast = stream_aligned(u, p.u_ds, p.L, p.reverse) && stream_aligned(dl, p.delta_ds, p.L, p.reverse);
    const LanePtr<T> lps[2] = {lane_ptr(u, p.u_ds, p.L, p.reverse, lane), lane_ptr(dl, p.delta_ds, p.L, p.reverse, lane)};
    for (int j0 = j_begin; j0 < j_end; j0 += kTile) {
        {
            float *const tiles[2] = {s_u, s_dt};
            const T *const bases[2] = {u, dl};
            const int64_t strides[2] = {p.u_ds, p.delta_ds};
            if (fast && j0 + kTile <= p.L) {
                fill_tiles_fast<T, 2, 2>(tiles, lps, wi.nrows, j0, p.reverse, lane);
            } else {
                fill_tile<T>(s_u, u, p.u_ds, wi.nrows, j0, p.L, p.reverse, lane);
                fill_tile<T>(s_dt, dl, p.delta_ds, wi.nrows, j0, p.L, p.reverse, lane);
            }
            float *const bt[1] = {s_B};
            const T *const bb[1] = {Bm};
            const int64_t bns[1] = {p.B_ns}, bls[1] = {p.B_ls};
            fill_bc_tiles<T, N, 1>(bt, bb, bns, bls, j0, p.L, p.reverse, lane);
            if (j0 + kTile < j_end) {
                prefetch_tiles<T, 2, 2>(bases, strides, wi.nrows, j0 + kTile, p.L, p.reverse, lane);
                prefetch_bc<T, N, 1>(bb, bns, bls, j0 + kTile, p.L, p.reverse, lane);
            }
        }
        __syncwarp();
        prepass_dt(s_dt, lane, bias, p.softplus, j_end - j0);      // masked positions are identities: h is simply repeated
#pragma unroll 1
        for (int c0 = 0; c0 < kTile / 4; c0 += 2) {
            const float *blkB = s_B + 4 * c0 * N;
            const float4 ua = tile_read4(s_u, lane, c0), ub = tile_read4(s_u, lane, c0 + 1);
            const float4 da = tile_read4(s_dt, lane, c0), db = tile_read4(s_dt, lane, c0 + 1);
            const float uu[8] = {ua.x, ua.y, ua.z, ua.w, ub.x, ub.y, ub.z, ub.w};
            const float dd[8] = {da.x, da.y, da.z, da.w, db.x, db.y, db.z, db.w};
            stash_block<N, 0, S>(blkB, uu, dd, A2, h, stash + (int64_t)(j0 + 4 * c0) * pos_stride, pos_stride, m_stride, active);
        }
        __syncwarp();
    }
}

__device__ __forceinline__ float sigmoid_of_softplus_inv(float dt) {   // sigmoid(raw) where dt = softplus(raw):  1 - exp(-dt)
    const float r = 1.f - __expf(-dt);
    const float s = dt * (1.f - dt * (0.5f - dt * (1.f / 6.f - dt * (1.f / 24.f))));
    return dt < 0.1f ? s : r;
}

constexpr int kTrPitch = 36;                    // transpose buffer row pitch (floats): conflict-free STS.128 rows / LDS columns

template <typename T, int N, bool kHasZ>
__global__ void __launch_bounds__(kWarpsPerCta * 32, 2) scan_bwd_sweep_kernel(const ScanP p) {
    using S = typename StashT<T>::type;
    static_assert(N == 16 || N == 8, "dstate");
    extern __shared__ __align__(16) float smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int w = blockIdx.x * kWarpsPerCta + warp;
    if (w >= p.n_work) return;
    const WorkItem wi = decode_work(p, w);          // S == kCkpt, n_seg == nck
    const int d = wi.d0 + lane;
    const bool active = lane < wi.nrows;
    constexpr int kWarpFloats = 4 * kTile * kTile + 2 * kTile * N + 32 * kTrPitch;
    float *s_dt = smem + warp * kWarpFloats;
    float *s_u = s_dt + kTile * kTile;
    float *s_g = s_u + kTile * kTile;
    float *s_z = s_g + kTile * kTile;
    float *s_B = s_z + kTile * kTile;
    float *s_C = s_B + kTile * N;
    float *s_tr = s_C + kTile * N;

    float2 A2[N / 2], mu[N / 2], dA2[N / 2], hcur[N / 2];
#pragma unroll
    for (int m = 0; m < N / 2; ++m) {
        A2[m] = active ? f2(p.A[(int64_t)d * N + 2 * m] * kLog2e, p.A[(int64_t)d * N + 2 * m + 1] * kLog2e) : f2(0.f, 0.f);
        const int64_t o = (((int64_t)wi.b * p.nck + wi.seg) * N + 2 * m) * p.dim + d;
        mu[m] = active ? f2(p.Min[o], p.Min[o + p.dim]) : f2(0.f, 0.f);
        dA2[m] = f2(0.f, 0.f);
    }
    const float bias = (active && p.delta_bias) ? p.delta_bias[d] : 0.f;
    const float Dv = (active && p.D) ? p.D[d] : 0.f;
    float dDacc = 0.f, dbacc = 0.f;

    const T *u = reinterpret_cast<const T *>(p.u) + wi.b * p.u_bs + (int64_t)wi.d0 * p.u_ds;
    const T *dl = reinterpret_cast<const T *>(p.delta) + wi.b * p.delta_bs + (int64_t)wi.d0 * p.delta_ds;
    const T *go = reinterpret_cast<const T *>(p.dout) + wi.b * p.dout_bs + (int64_t)wi.d0 * p.dout_ds;
    const T *z = kHasZ ? reinterpret_cast<const T *>(p.z) + wi.b * p.z_bs + (int64_t)wi.d0 * p.z_ds : nullptr;
    const T *Bm = reinterpret_cast<const T *>(p.B) + wi.b * p.B_bs + (int64_t)wi.g * p.B_gs;
    const T *Cm = reinterpret_cast<const T *>(p.C) + wi.b * p.C_bs + (int64_t)wi.g * p.C_gs;
    T *du = reinterpret_cast<T *>(p.du) + wi.b * p.du_bs + (int64_t)wi.d0 * p.du_ds;
    T *dde = reinterpret_cast<T *>(p.ddelta) + wi.b * p.ddelta_bs + (int64_t)wi.d0 * p.ddelta_ds;
    T *dz = kHasZ ? reinterpret_cast<T *>(p.dz) + wi.b * p.dz_bs + (int64_t)wi.d0 * p.dz_ds : nullptr;
    T *oz = (kHasZ && p.out_z) ? reinterpret_cast<T *>(p.out_z) + wi.b * p.out_z_bs + (int64_t)wi.d0 * p.out_z_ds : nullptr;
    const int64_t m_stride = p.dim, pos_stride = (int64_t)(N / 2) * p.dim;
    const S *stash = reinterpret_cast<const S *>(p.stash) + (int64_t)wi.b * p.Lpad * pos_stride + d;
    // this lane's slot of the cross-channel reduction: lanes 0..15 -> dB state (lane), lanes 16..31 -> dC state (lane-16)
    float *dBC = ((lane < 16) ? p.dB : p.dC) + (((int64_t)wi.b * p.G + wi.g) * N + (lane & 15)) * (int64_t)p.L;
    const bool red_slot = (lane & 15) < N;
    const bool vec_ok = (p.L & 3) == 0 && ((reinterpret_cast<uintptr_t>(p.dB) | reinterpret_cast<uintptr_t>(p.dC)) & 15) == 0;

    const int j_begin = wi.seg * kCkpt;
    const int j_end = min(p.L, j_begin + kCkpt);
    const int last_tile = j_begin + ((j_end - j_begin - 1) / kTile) * kTile;
    const bool fast = stream_aligned(u, p.u_ds, p.L, p.reverse) && stream_aligned(dl, p.delta_ds, p.L, p.reverse) &&
                      stream_aligned(go, p.dout_ds, p.L, p.reverse) && (!kHasZ || stream_aligned(z, p.z_ds, p.L, p.reverse));
    const LanePtr<T> lps[4] = {lane_ptr(dl, p.delta_ds, p.L, p.reverse, lane), lane_ptr(u, p.u_ds, p.L, p.reverse, lane),
                               lane_ptr(go, p.dout_ds, p.L, p.reverse, lane),
                               lane_ptr(kHasZ ? z : dl, kHasZ ? p.z_ds : p.delta_ds, p.L, p.reverse, lane)};
    // state at the last position of the walk
    {
        const S *sp = stash + (int64_t)(last_tile + kTile - 1) * pos_stride;
#pragma unroll
        for (int m = 0; m < N / 2; ++m) hcur[m] = active ? stash_cvt(sp[m * m_stride]) : f2(0.f, 0.f);
    }
    for (int j0 = last_tile; j0 >= j_begin; j0 -= kTile) {
        {
            constexpr int K = kHasZ ? 4 : 3;
            float *const tiles[4] = {s_dt, s_u, s_g, s_z};
            const T *const bases[4] = {dl, u, go, kHasZ ? z : dl};
            const int64_t strides[4] = {p.delta_ds, p.u_ds, p.dout_ds, kHasZ ? p.z_ds : p.delta_ds};
            if (fast && j0 + kTile <= p.L) {
                fill_tiles_fast<T, K, 4>(tiles, lps, wi.nrows, j0, p.reverse, lane);
            } else {
                fill_tile<T>(s_dt, dl, p.delta_ds, wi.nrows, j0, p.L, p.reverse, lane);
                fill_tile<T>(s_u, u, p.u_ds, wi.nrows, j0, p.L, p.reverse, lane);
                fill_tile<T>(s_g, go, p.dout_ds, wi.nrows, j0, p.L, p.reverse, lane);
                if (kHasZ) fill_tile<T>(s_z, z, p.z_ds, wi.nrows, j0, p.L, p.reverse, lane);
            }
            float *const bt[2] = {s_B, s_C};
            const T *const bb[2] = {Bm, Cm};
            const int64_t bns[2] = {p.B_ns, p.C_ns}, bls[2] = {p.B_ls, p.C_ls};
            fill_bc_tiles<T, N, 2>(bt, bb, bns, bls, j0, p.L, p.reverse, lane);
            if (j0 - kTile >= j_begin) {
                prefetch_tiles<T, K, 4>(bases, strides, wi.nrows, j0 - kTile, p.L, p.reverse, lane);
                prefetch_bc<T, N, 2>(bb, bns, bls, j0 - kTile, p.L, p.reverse, lane);
            }
        }
        __syncwarp();
        prepass_dt(s_dt, lane, bias, p.softplus, j_end - j0);
        if (kHasZ) {
            // g <- dout * silu(z) ;  z-slot <- dout * d silu(z)/dz  (then dz = slot * y);  if out_z is wanted keep silu(z) instead
#pragma unroll
            for (int c = 0; c < kTile / 4; ++c) {
                const float4 g4 = tile_read4(s_g, lane, c), z4 = tile_read4(s_z, lane, c);
                const float gg[4] = {g4.x, g4.y, g4.z, g4.w}, zz[4] = {z4.x, z4.y, z4.z, z4.w};
                float gn[4], zc[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float sg = sigmoidf(zz[e]);
                    gn[e] = gg[e] * zz[e] * sg;
                    zc[e] = gg[e] * sg * (1.f + zz[e] * (1.f - sg));
                }
                tile_write4(s_g, lane, c, make_float4(gn[0], gn[1], gn[2], gn[3]));
                tile_write4(s_z, lane, c, make_float4(zc[0], zc[1], zc[2], zc[3]));
            }
        }
        // pull the stash lines of the next (lower) tile into L2 while this one is processed: 8 lines (one per state pair) per
        // position, lane l covers position l of that tile
        if (j0 - kTile >= 0 && active) {
            const S *sp = stash + (int64_t)(j0 - kTile + lane) * pos_stride - lane;      // line start: channel d0
#pragma unroll
            for (int m = 0; m < N / 2; ++m) prefetch_l2(sp + m * m_stride);
        }
#pragma unroll 1
        for (int c = kTile / 4 - 1; c >= 0; --c) {            // blocks of 4 positions, descending
            const float4 d4 = tile_read4(s_dt, lane, c), u4 = tile_read4(s_u, lane, c), g4 = tile_read4(s_g, lane, c);
            float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
            if (kHasZ) z4 = tile_read4(s_z, lane, c);
            float4 duv = make_float4(0.f, 0.f, 0.f, 0.f), ddv = duv, dzv = duv, red = duv;
            const int q0 = 4 * c;
            const float *blkB = s_B + q0 * N, *blkC = s_C + q0 * N;
#pragma unroll 1
            for (int e = 3; e >= 0; --e) {
                const int pos = j0 + q0 + e;
                const bool valid = pos < j_end;
                // h_{t-1}: issue the loads first, consume them at the end of this position
                S hp[N / 2];
                {
                    const S *sp = stash + (int64_t)(pos - 1) * pos_stride;
#pragma unroll
                    for (int m = 0; m < N / 2; ++m) hp[m] = (active && pos > 0) ? sp[m * m_stride] : stash_zero<S>();
                }
                const float dt = e == 3 ? d4.w : e == 2 ? d4.z : e == 1 ? d4.y : d4.x;
                const float uv = e == 3 ? u4.w : e == 2 ? u4.z : e == 1 ? u4.y : u4.x;
                const float g = e == 3 ? g4.w : e == 2 ? g4.z : e == 1 ? g4.y : g4.x;
                const float zc = e == 3 ? z4.w : e == 2 ? z4.z : e == 1 ? z4.y : z4.x;
                const float2 dt2 = f2(dt, dt), g2 = f2(g, g), dtu2 = f2(dt * uv, dt * uv);
                float2 yacc = f2(0.f, 0.f), slb = f2(0.f, 0.f), saq = f2(0.f, 0.f);
                float2 vB[N / 2], vC[N / 2];
                const int sw = ((q0 + e) >> 1) & (N / 4 - 1);      // B/C tile swizzle of this position
                const float *rowB = blkB + e * N, *rowC = blkC + e * N;
#pragma unroll
                for (int jn = 0; jn < N / 4; ++jn) {
                    const float4 b4 = *reinterpret_cast<const float4 *>(rowB + ((jn ^ sw) << 2));
                    const float4 c4 = *reinterpret_cast<const float4 *>(rowC + ((jn ^ sw) << 2));
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        const int m = 2 * jn + hh;
                        const float2 Bp = hh ? f2(b4.z, b4.w) : f2(b4.x, b4.y);
                        const float2 Cp = hh ? f2(c4.z, c4.w) : f2(c4.x, c4.y);
                        const float2 a = ex2x2_mufu(fmul2(dt2, A2[m]));
                        const float2 lam = ffma2(g2, Cp, mu[m]);
                        mu[m] = fmul2(a, lam);
                        yacc = ffma2(Cp, hcur[m], yacc);
                        vC[m] = fmul2(g2, hcur[m]);
                        vB[m] = fmul2(lam, dtu2);
                        slb = ffma2(lam, Bp, slb);
                    }
                }
                // ---- reduce vB / vC over the 32 channels of this warp: transpose through shared memory ----
                float *row = s_tr + lane * kTrPitch;
#pragma unroll
                for (int m = 0; m < N / 2; m += 2) {
                    *reinterpret_cast<float4 *>(row + 2 * m) = make_float4(vB[m].x, vB[m].y, vB[m + 1].x, vB[m + 1].y);
                    *reinterpret_cast<float4 *>(row + 16 + 2 * m) = make_float4(vC[m].x, vC[m].y, vC[m + 1].x, vC[m + 1].y);
                }
                __syncwarp();
#pragma unroll
                for (int m = 0; m < N / 2; ++m) {
                    const float2 hpv = stash_cvt(hp[m]);
                    const float2 qm = fmul2(mu[m], hpv);                // lambda_t a_t h_{t-1}
                    dA2[m] = ffma2(dt2, qm, dA2[m]);
                    saq = ffma2(A2[m], qm, saq);
                    hcur[m] = hpv;
                }
                const float y = fmaf(Dv, uv, yacc.x + yacc.y);
                const float lb = slb.x + slb.y;
                float ddt = fmaf(uv, lb, kLn2 * (saq.x + saq.y));
                if (p.softplus) ddt *= sigmoid_of_softplus_inv(dt);
                ddt = valid ? ddt : 0.f;
                const float duo = fmaf(dt, lb, Dv * g), dzo = zc * y;
                dDacc = fmaf(g, uv, dDacc);
                dbacc += ddt;
                float rsum;
                {
                    const int col = (lane < 16) ? (lane & 15) : 16 + (lane & 15);
                    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
                    for (int r = 0; r < 32; r += 4) {
                        s0 += s_tr[(r + 0) * kTrPitch + col];
                        s1 += s_tr[(r + 1) * kTrPitch + col];
                        s2 += s_tr[(r + 2) * kTrPitch + col];
                        s3 += s_tr[(r + 3) * kTrPitch + col];
                    }
                    rsum = (s0 + s1) + (s2 + s3);
                }
                __syncwarp();
                if (e == 3) { duv.w = duo; ddv.w = ddt; dzv.w = dzo; red.w = rsum; }
                else if (e == 2) { duv.z = duo; ddv.z = ddt; dzv.z = dzo; red.z = rsum; }
                else if (e == 1) { duv.y = duo; ddv.y = ddt; dzv.y = dzo; red.y = rsum; }
                else { duv.x = duo; ddv.x = ddt; dzv.x = dzo; red.x = rsum; }
            }
            // in place: u-slot <- du, dt-slot <- ddelta, z-slot <- dz
            tile_write4(s_u, lane, c, duv);
            tile_write4(s_dt, lane, c, ddv);
            if (kHasZ) tile_write4(s_z, lane, c, dzv);
            // dB / dC: 4 consecutive positions of this lane's (tensor, state) row
            if (red_slot) {
                const int pos0 = j0 + q0;
                if (pos0 + 3 < p.L && vec_ok) {
                    float *a = dBC + (p.reverse ? (p.L - 4 - pos0) : pos0);
                    if (!p.reverse) red_add_v4(a, red.x, red.y, red.z, red.w);
                    else red_add_v4(a, red.w, red.z, red.y, red.x);
                } else {
                    const float rr[4] = {red.x, red.y, red.z, red.w};
#pragma unroll
                    for (int e = 0; e < 4; ++e)
                        if (pos0 + e < p.L) atomicAdd(dBC + pos_to_tok(pos0 + e, p.L, p.reverse), rr[e]);
                }
            }
        }
        __syncwarp();
        store_tile<T>(s_u, du, p.du_ds, wi.nrows, j0, p.L, p.reverse, lane);
        store_tile<T>(s_dt, dde, p.ddelta_ds, wi.nrows, j0, p.L, p.reverse, lane);
        if (kHasZ) store_tile<T>(s_z, dz, p.dz_ds, wi.nrows, j0, p.L, p.reverse, lane);
        __syncwarp();
    }
    if (active) {
#pragma unroll
        for (int m = 0; m < N / 2; ++m) {
            atomicAdd(p.dA + (int64_t)d * N + 2 * m, dA2[m].x);
            atomicAdd(p.dA + (int64_t)d * N + 2 * m + 1, dA2[m].y);
        }
        if (p.dD) atomicAdd(p.dD + d, dDacc);
        if (p.ddelta_bias) atomicAdd(p.ddelta_bias + d, dbacc);
    }
    (void)oz;
}

// More than 16 states (32, 64): the same reverse sweep with the dB / dC transpose in rounds of 16 states per tensor.  Each
// 4-state chunk is written to the transpose buffer as soon as it is computed and every round is reduced before the next one,
// so no dB / dC terms stay in registers across rounds; the reduced values leave as one vector atomic per (tensor, state,
// 4 positions) as above.
template <typename T, int N, bool kHasZ>
__global__ void __launch_bounds__(kWarpsPerCta * 32, 2) scan_bwd_sweep_wide_kernel(const ScanP p) {
    using S = typename StashT<T>::type;
    static_assert(N % 16 == 0 && N > 16, "dstate");
    constexpr int kRed = (N + 15) / 16;             // rounds of the dB / dC transpose: 16 states of each tensor per round
    extern __shared__ __align__(16) float smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int w = blockIdx.x * kWarpsPerCta + warp;
    if (w >= p.n_work) return;
    const WorkItem wi = decode_work(p, w);          // S == kCkpt, n_seg == nck
    const int d = wi.d0 + lane;
    const bool active = lane < wi.nrows;
    constexpr int kWarpFloats = 4 * kTile * kTile + 2 * kTile * N + 32 * kTrPitch;
    float *s_dt = smem + warp * kWarpFloats;
    float *s_u = s_dt + kTile * kTile;
    float *s_g = s_u + kTile * kTile;
    float *s_z = s_g + kTile * kTile;
    float *s_B = s_z + kTile * kTile;
    float *s_C = s_B + kTile * N;
    float *s_tr = s_C + kTile * N;

    float2 A2[N / 2], mu[N / 2], dA2[N / 2], hcur[N / 2];
#pragma unroll
    for (int m = 0; m < N / 2; ++m) {
        A2[m] = active ? f2(p.A[(int64_t)d * N + 2 * m] * kLog2e, p.A[(int64_t)d * N + 2 * m + 1] * kLog2e) : f2(0.f, 0.f);
        const int64_t o = (((int64_t)wi.b * p.nck + wi.seg) * N + 2 * m) * p.dim + d;
        mu[m] = active ? f2(p.Min[o], p.Min[o + p.dim]) : f2(0.f, 0.f);
        dA2[m] = f2(0.f, 0.f);
    }
    const float bias = (active && p.delta_bias) ? p.delta_bias[d] : 0.f;
    const float Dv = (active && p.D) ? p.D[d] : 0.f;
    float dDacc = 0.f, dbacc = 0.f;

    const T *u = reinterpret_cast<const T *>(p.u) + wi.b * p.u_bs + (int64_t)wi.d0 * p.u_ds;
    const T *dl = reinterpret_cast<const T *>(p.delta) + wi.b * p.delta_bs + (int64_t)wi.d0 * p.delta_ds;
    const T *go = reinterpret_cast<const T *>(p.dout) + wi.b * p.dout_bs + (int64_t)wi.d0 * p.dout_ds;
    const T *z = kHasZ ? reinterpret_cast<const T *>(p.z) + wi.b * p.z_bs + (int64_t)wi.d0 * p.z_ds : nullptr;
    const T *Bm = reinterpret_cast<const T *>(p.B) + wi.b * p.B_bs + (int64_t)wi.g * p.B_gs;
    const T *Cm = reinterpret_cast<const T *>(p.C) + wi.b * p.C_bs + (int64_t)wi.g * p.C_gs;
    T *du = reinterpret_cast<T *>(p.du) + wi.b * p.du_bs + (int64_t)wi.d0 * p.du_ds;
    T *dde = reinterpret_cast<T *>(p.ddelta) + wi.b * p.ddelta_bs + (int64_t)wi.d0 * p.ddelta_ds;
    T *dz = kHasZ ? reinterpret_cast<T *>(p.dz) + wi.b * p.dz_bs + (int64_t)wi.d0 * p.dz_ds : nullptr;
    T *oz = (kHasZ && p.out_z) ? reinterpret_cast<T *>(p.out_z) + wi.b * p.out_z_bs + (int64_t)wi.d0 * p.out_z_ds : nullptr;
    const int64_t m_stride = p.dim, pos_stride = (int64_t)(N / 2) * p.dim;
    const S *stash = reinterpret_cast<const S *>(p.stash) + (int64_t)wi.b * p.Lpad * pos_stride + d;
    // this lane's slot of the cross-channel reduction in round r: lanes 0..15 -> dB state 16 r + lane, lanes 16..31 -> dC state
    // 16 r + lane - 16
    float *dBC = ((lane < 16) ? p.dB : p.dC) + (((int64_t)wi.b * p.G + wi.g) * N + (lane & 15)) * (int64_t)p.L;
    const bool red_slot = (lane & 15) < N;
    const bool vec_ok = (p.L & 3) == 0 && ((reinterpret_cast<uintptr_t>(p.dB) | reinterpret_cast<uintptr_t>(p.dC)) & 15) == 0;

    const int j_begin = wi.seg * kCkpt;
    const int j_end = min(p.L, j_begin + kCkpt);
    const int last_tile = j_begin + ((j_end - j_begin - 1) / kTile) * kTile;
    const bool fast = stream_aligned(u, p.u_ds, p.L, p.reverse) && stream_aligned(dl, p.delta_ds, p.L, p.reverse) &&
                      stream_aligned(go, p.dout_ds, p.L, p.reverse) && (!kHasZ || stream_aligned(z, p.z_ds, p.L, p.reverse));
    const LanePtr<T> lps[4] = {lane_ptr(dl, p.delta_ds, p.L, p.reverse, lane), lane_ptr(u, p.u_ds, p.L, p.reverse, lane),
                               lane_ptr(go, p.dout_ds, p.L, p.reverse, lane),
                               lane_ptr(kHasZ ? z : dl, kHasZ ? p.z_ds : p.delta_ds, p.L, p.reverse, lane)};
    // state at the last position of the walk
    {
        const S *sp = stash + (int64_t)(last_tile + kTile - 1) * pos_stride;
#pragma unroll
        for (int m = 0; m < N / 2; ++m) hcur[m] = active ? stash_cvt(sp[m * m_stride]) : f2(0.f, 0.f);
    }
    for (int j0 = last_tile; j0 >= j_begin; j0 -= kTile) {
        {
            constexpr int K = kHasZ ? 4 : 3;
            float *const tiles[4] = {s_dt, s_u, s_g, s_z};
            const T *const bases[4] = {dl, u, go, kHasZ ? z : dl};
            const int64_t strides[4] = {p.delta_ds, p.u_ds, p.dout_ds, kHasZ ? p.z_ds : p.delta_ds};
            if (fast && j0 + kTile <= p.L) {
                fill_tiles_fast<T, K, 4>(tiles, lps, wi.nrows, j0, p.reverse, lane);
            } else {
                fill_tile<T>(s_dt, dl, p.delta_ds, wi.nrows, j0, p.L, p.reverse, lane);
                fill_tile<T>(s_u, u, p.u_ds, wi.nrows, j0, p.L, p.reverse, lane);
                fill_tile<T>(s_g, go, p.dout_ds, wi.nrows, j0, p.L, p.reverse, lane);
                if (kHasZ) fill_tile<T>(s_z, z, p.z_ds, wi.nrows, j0, p.L, p.reverse, lane);
            }
            float *const bt[2] = {s_B, s_C};
            const T *const bb[2] = {Bm, Cm};
            const int64_t bns[2] = {p.B_ns, p.C_ns}, bls[2] = {p.B_ls, p.C_ls};
            fill_bc_tiles<T, N, 2>(bt, bb, bns, bls, j0, p.L, p.reverse, lane);
            if (j0 - kTile >= j_begin) {
                prefetch_tiles<T, K, 4>(bases, strides, wi.nrows, j0 - kTile, p.L, p.reverse, lane);
                prefetch_bc<T, N, 2>(bb, bns, bls, j0 - kTile, p.L, p.reverse, lane);
            }
        }
        __syncwarp();
        prepass_dt(s_dt, lane, bias, p.softplus, j_end - j0);
        if (kHasZ) {
            // g <- dout * silu(z) ;  z-slot <- dout * d silu(z)/dz  (then dz = slot * y);  if out_z is wanted keep silu(z) instead
#pragma unroll
            for (int c = 0; c < kTile / 4; ++c) {
                const float4 g4 = tile_read4(s_g, lane, c), z4 = tile_read4(s_z, lane, c);
                const float gg[4] = {g4.x, g4.y, g4.z, g4.w}, zz[4] = {z4.x, z4.y, z4.z, z4.w};
                float gn[4], zc[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float sg = sigmoidf(zz[e]);
                    gn[e] = gg[e] * zz[e] * sg;
                    zc[e] = gg[e] * sg * (1.f + zz[e] * (1.f - sg));
                }
                tile_write4(s_g, lane, c, make_float4(gn[0], gn[1], gn[2], gn[3]));
                tile_write4(s_z, lane, c, make_float4(zc[0], zc[1], zc[2], zc[3]));
            }
        }
        // pull the stash lines of the next (lower) tile into L2 while this one is processed: 8 lines (one per state pair) per
        // position, lane l covers position l of that tile
        if (j0 - kTile >= 0 && active) {
            const S *sp = stash + (int64_t)(j0 - kTile + lane) * pos_stride - lane;      // line start: channel d0
#pragma unroll
            for (int m = 0; m < N / 2; ++m) prefetch_l2(sp + m * m_stride);
        }
#pragma unroll 1
        for (int c = kTile / 4 - 1; c >= 0; --c) {            // blocks of 4 positions, descending
            const float4 d4 = tile_read4(s_dt, lane, c), u4 = tile_read4(s_u, lane, c), g4 = tile_read4(s_g, lane, c);
            float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
            if (kHasZ) z4 = tile_read4(s_z, lane, c);
            float4 duv = make_float4(0.f, 0.f, 0.f, 0.f), ddv = duv, dzv = duv, red[kRed];
#pragma unroll
            for (int r = 0; r < kRed; ++r) red[r] = duv;
            const int q0 = 4 * c;
            const float *blkB = s_B + q0 * N, *blkC = s_C + q0 * N;
#pragma unroll 1
            for (int e = 3; e >= 0; --e) {
                const int pos = j0 + q0 + e;
                const bool valid = pos < j_end;
                // h_{t-1}: issue the loads first, consume them at the end of this position
                S hp[N / 2];
                {
                    const S *sp = stash + (int64_t)(pos - 1) * pos_stride;
#pragma unroll
                    for (int m = 0; m < N / 2; ++m) hp[m] = (active && pos > 0) ? sp[m * m_stride] : stash_zero<S>();
                }
                const float dt = e == 3 ? d4.w : e == 2 ? d4.z : e == 1 ? d4.y : d4.x;
                const float uv = e == 3 ? u4.w : e == 2 ? u4.z : e == 1 ? u4.y : u4.x;
                const float g = e == 3 ? g4.w : e == 2 ? g4.z : e == 1 ? g4.y : g4.x;
                const float zc = e == 3 ? z4.w : e == 2 ? z4.z : e == 1 ? z4.y : z4.x;
                const float2 dt2 = f2(dt, dt), g2 = f2(g, g), dtu2 = f2(dt * uv, dt * uv);
                float2 yacc = f2(0.f, 0.f), slb = f2(0.f, 0.f), saq = f2(0.f, 0.f);
                const int sw = ((q0 + e) >> 1) & bc_swz<N>();      // B/C tile swizzle of this position
                const float *rowB = blkB + e * N, *rowC = blkC + e * N;
                float rs[kRed];                                    // this lane's reduced dB / dC of each round
                // more than 16 states: one transpose round per 16 states, each 4-state chunk goes to shared memory as soon as
                // it is computed, so no dB / dC terms stay in registers across chunks
                float *row = s_tr + lane * kTrPitch;
#pragma unroll
                for (int r = 0; r < kRed; ++r) {
#pragma unroll
                    for (int jr = 0; jr < 4; ++jr) {
                        const int jn = 4 * r + jr;
                        const float4 b4 = *reinterpret_cast<const float4 *>(rowB + ((jn ^ sw) << 2));
                        const float4 c4 = *reinterpret_cast<const float4 *>(rowC + ((jn ^ sw) << 2));
                        float2 vB[2], vC[2];
#pragma unroll
                        for (int hh = 0; hh < 2; ++hh) {
                            const int m = 2 * jn + hh;
                            const float2 Bp = hh ? f2(b4.z, b4.w) : f2(b4.x, b4.y);
                            const float2 Cp = hh ? f2(c4.z, c4.w) : f2(c4.x, c4.y);
                            const float2 a = ex2x2_mufu(fmul2(dt2, A2[m]));
                            const float2 lam = ffma2(g2, Cp, mu[m]);
                            mu[m] = fmul2(a, lam);
                            yacc = ffma2(Cp, hcur[m], yacc);
                            vC[hh] = fmul2(g2, hcur[m]);
                            vB[hh] = fmul2(lam, dtu2);
                            slb = ffma2(lam, Bp, slb);
                        }
                        *reinterpret_cast<float4 *>(row + 4 * jr) = make_float4(vB[0].x, vB[0].y, vB[1].x, vB[1].y);
                        *reinterpret_cast<float4 *>(row + 16 + 4 * jr) = make_float4(vC[0].x, vC[0].y, vC[1].x, vC[1].y);
                    }
                    __syncwarp();
                    const int col = (lane < 16) ? (lane & 15) : 16 + (lane & 15);
                    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
                    for (int k = 0; k < 32; k += 4) {
                        s0 += s_tr[(k + 0) * kTrPitch + col];
                        s1 += s_tr[(k + 1) * kTrPitch + col];
                        s2 += s_tr[(k + 2) * kTrPitch + col];
                        s3 += s_tr[(k + 3) * kTrPitch + col];
                    }
                    rs[r] = (s0 + s1) + (s2 + s3);
                    __syncwarp();
                }
#pragma unroll
                for (int m = 0; m < N / 2; ++m) {
                    const float2 hpv = stash_cvt(hp[m]);
                    const float2 qm = fmul2(mu[m], hpv);                // lambda_t a_t h_{t-1}
                    dA2[m] = ffma2(dt2, qm, dA2[m]);
                    saq = ffma2(A2[m], qm, saq);
                    hcur[m] = hpv;
                }
                const float y = fmaf(Dv, uv, yacc.x + yacc.y);
                const float lb = slb.x + slb.y;
                float ddt = fmaf(uv, lb, kLn2 * (saq.x + saq.y));
                if (p.softplus) ddt *= sigmoid_of_softplus_inv(dt);
                ddt = valid ? ddt : 0.f;
                const float duo = fmaf(dt, lb, Dv * g), dzo = zc * y;
                dDacc = fmaf(g, uv, dDacc);
                dbacc += ddt;
                if (e == 3) { duv.w = duo; ddv.w = ddt; dzv.w = dzo; for (int r = 0; r < kRed; ++r) red[r].w = rs[r]; }
                else if (e == 2) { duv.z = duo; ddv.z = ddt; dzv.z = dzo; for (int r = 0; r < kRed; ++r) red[r].z = rs[r]; }
                else if (e == 1) { duv.y = duo; ddv.y = ddt; dzv.y = dzo; for (int r = 0; r < kRed; ++r) red[r].y = rs[r]; }
                else { duv.x = duo; ddv.x = ddt; dzv.x = dzo; for (int r = 0; r < kRed; ++r) red[r].x = rs[r]; }
            }
            // in place: u-slot <- du, dt-slot <- ddelta, z-slot <- dz
            tile_write4(s_u, lane, c, duv);
            tile_write4(s_dt, lane, c, ddv);
            if (kHasZ) tile_write4(s_z, lane, c, dzv);
            // dB / dC: 4 consecutive positions of this lane's (tensor, state) row
#pragma unroll
            for (int r = 0; r < kRed; ++r) {
            if (red_slot) {
                const int pos0 = j0 + q0;
                float *dBCr = dBC + (int64_t)(16 * r) * p.L;
                if (pos0 + 3 < p.L && vec_ok) {
                    float *a = dBCr + (p.reverse ? (p.L - 4 - pos0) : pos0);
                    if (!p.reverse) red_add_v4(a, red[r].x, red[r].y, red[r].z, red[r].w);
                    else red_add_v4(a, red[r].w, red[r].z, red[r].y, red[r].x);
                } else {
                    const float rr[4] = {red[r].x, red[r].y, red[r].z, red[r].w};
#pragma unroll
                    for (int e = 0; e < 4; ++e)
                        if (pos0 + e < p.L) atomicAdd(dBCr + pos_to_tok(pos0 + e, p.L, p.reverse), rr[e]);
                }
            }
            }
        }
        __syncwarp();
        store_tile<T>(s_u, du, p.du_ds, wi.nrows, j0, p.L, p.reverse, lane);
        store_tile<T>(s_dt, dde, p.ddelta_ds, wi.nrows, j0, p.L, p.reverse, lane);
        if (kHasZ) store_tile<T>(s_z, dz, p.dz_ds, wi.nrows, j0, p.L, p.reverse, lane);
        __syncwarp();
    }
    if (active) {
#pragma unroll
        for (int m = 0; m < N / 2; ++m) {
            atomicAdd(p.dA + (int64_t)d * N + 2 * m, dA2[m].x);
            atomicAdd(p.dA + (int64_t)d * N + 2 * m + 1, dA2[m].y);
        }
        if (p.dD) atomicAdd(p.dD + d, dDacc);
        if (p.ddelta_bias) atomicAdd(p.ddelta_bias + d, dbacc);
    }
    (void)oz;
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
template <typename T, int N, bool kHasZ>
static cudaError_t launch_bwd(const ScanP &p, cudaStream_t st) {
    cudaError_t e;
    // R1
    const int ctas = (p.n_work + kWarpsPerCta - 1) / kWarpsPerCta;
    const size_t sm1 = (size_t)kWarpsPerCta * (3 * kTile * kTile + kTile * N) * sizeof(float);
    const char *r1v2 = getenv("SMB_RAGG_V2");                 // software-pipelined R1 for 16-bit activations (scan_bwd_v2.cu); =0: A/B
    if (sizeof(T) == 2 && !(r1v2 && r1v2[0] == '0')) {
        if ((e = scan_bwd_ragg_v2_dispatch(p, sizeof(T) == 2 && std::is_same<T, __half>::value ? 1 : 2, N, kHasZ, st)) != cudaSuccess) return e;
    } else {
        SMB_SET_SMEM_ONCE((scan_bwd_ragg_kernel<T, N, kHasZ>), sm1);
        scan_bwd_ragg_kernel<T, N, kHasZ><<<ctas, kWarpsPerCta * 32, sm1, st>>>(p); count_launch();
    }
    // R2
    if ((e = carry_launch(p.Pb, p.Mloc, p.Min, nullptr, p.batch, p.nck, N, p.dim, 1, st)) != cudaSuccess) return e;
    if (p.stash && !(kHasZ && p.out_z)) {
        // K_F: forward recompute into the stash, then K_R: lane-per-channel reverse sweep
        const size_t smf = (size_t)kWarpsPerCta * (2 * kTile * kTile + kTile * N) * sizeof(float);
        SMB_SET_SMEM_ONCE((scan_bwd_stash_kernel<T, N>), smf);
        scan_bwd_stash_kernel<T, N><<<ctas, kWarpsPerCta * 32, smf, st>>>(p); count_launch();
        const size_t smr = (size_t)kWarpsPerCta * (4 * kTile * kTile + 2 * kTile * N + 32 * kTrPitch) * sizeof(float);
        if constexpr (N > 16) {
            SMB_SET_SMEM_ONCE((scan_bwd_sweep_wide_kernel<T, N, kHasZ>), smr);
            scan_bwd_sweep_wide_kernel<T, N, kHasZ><<<ctas, kWarpsPerCta * 32, smr, st>>>(p); count_launch();
        } else {
            SMB_SET_SMEM_ONCE((scan_bwd_sweep_kernel<T, N, kHasZ>), smr);
            scan_bwd_sweep_kernel<T, N, kHasZ><<<ctas, kWarpsPerCta * 32, smr, st>>>(p); count_launch();
        }
        return cudaGetLastError();
    }
    // R3 (low-memory path; also used when the caller wants out_z recomputed)
    {   // second-generation R3 (scan_bwd_r3v2.cu): same results, fewer instructions per update; SMB_R3_V2=0 keeps the first one (A/B)
        const char *r3v2 = getenv("SMB_R3_V2");
        if (!(r3v2 && r3v2[0] == '0'))
            return scan_bwd_main_v2_dispatch(p, std::is_same<T, float>::value ? 0 : (std::is_same<T, __half>::value ? 1 : 2), N, kHasZ, st);
    }
    const size_t sm3 = (size_t)(2 * N + 2 * kBwdWarps) * kRowPad * sizeof(float);
    SMB_SET_SMEM_ONCE((scan_bwd_main_kernel<T, N, kHasZ>), sm3);
    const int octs = ((p.dim_per_group + kBwdWarps - 1) / kBwdWarps) * p.G;
    dim3 grid(p.nck, octs, p.batch);
    scan_bwd_main_kernel<T, N, kHasZ><<<grid, kBwdWarps * 32, sm3, st>>>(p); count_launch();
    return cudaGetLastError();
}

template <typename T>
static cudaError_t launch_bwd_t(const ScanP &p, int N, bool has_z, cudaStream_t st) {
    switch (N) {
        case 64: return has_z ? launch_bwd<T, 64, true>(p, st) : launch_bwd<T, 64, false>(p, st);
        case 32: return has_z ? launch_bwd<T, 32, true>(p, st) : launch_bwd<T, 32, false>(p, st);
        case 16: return has_z ? launch_bwd<T, 16, true>(p, st) : launch_bwd<T, 16, false>(p, st);
        default: return has_z ? launch_bwd<T, 8, true>(p, st) : launch_bwd<T, 8, false>(p, st);
    }
}

cudaError_t scan_bwd_dispatch(const ScanP &p, int dtype, int N, bool has_z, cudaStream_t st) {
    switch (dtype) {
        case 0: return launch_bwd_t<float>(p, N, has_z, st);
        case 1: return launch_bwd_t<__half>(p, N, has_z, st);
        default: return launch_bwd_t<__nv_bfloat16>(p, N, has_z, st);
    }
}

}  // namespace smb
