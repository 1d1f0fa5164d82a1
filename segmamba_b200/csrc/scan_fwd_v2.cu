// Forward selective scan, software-pipelined variant for 16-bit activations (opt-in: SMB_FWD_V2=1; see DESIGN.md 3.1).
//
// Same three passes, mapping and arithmetic as scan_fwd.cu (lane == channel, all N states in registers, B/C broadcast from a
// warp-private tile).  What changes is how a tile reaches the SM.  In scan_fwd.cu every warp alternates between a fill phase
// (global loads -> convert -> shared) and a compute phase (16 ex2 per position); the warps of a CTA run in lockstep, so the
// MUFU pipe idles while they all fill (ncu: XU 64 % / 46 % busy in the two passes, top stall long_scoreboard).  Here the
// NEXT tile is copied global -> shared with cp.async while the current one is computed:
//   * u / delta / z tiles stay in their 16-bit storage type in two alternating stages (2 KB each: 32 rows x 64 bytes, the
//     16-byte units of a row XOR-swizzled with (row >> 1) & 3 so that the per-lane LDS.128 of the compute phase and the
//     8-byte cp.async / store accesses are both conflict-free); conversion, softplus and SiLU happen in registers when a lane
//     reads its 8 positions, and y / out_z are written back in place over the consumed u / z units for the coalesced store;
//   * B / C rows land in a raw staging buffer and are transposed into the position-major fp32 broadcast tile at the top of
//     the iteration, before the staging buffer is handed to the next cp.async.
// Shared memory per warp: 11 KB (pass 1) / 18 KB (pass 3), against 10 / 16 KB in scan_fwd.cu.  Tiles that are ragged or not
// 8-byte aligned take a synchronous fill into the same stage layout, so there is one compute path.
#include "raw_tiles.cuh"
#include "scan_internal.h"
#include "scan_steps.cuh"
#include "tma.cuh"

namespace smb {

// Tensor maps of one forward call (TMA mode, SMB_FWD_V2=2).  Activations: rank 3 (L, a1, a2) where (a1, a2) = (channel, batch)
// ordered by increasing stride (swap = 1 when the batch stride is the smaller one, as in the mixer's channel-major layout);
// box = 32 tokens x 32 channels x 1 batch, SWIZZLE_64B.  B / C: rank 3 (L, state | batch), box = 32 tokens x N states, no swizzle.
struct ScanTmaps {
    CUtensorMap u, d, z, B, C;
    int swap_u, swap_d, swap_z, swap_B, swap_C;
};
template <bool kIsBC>
__device__ __forceinline__ void tma_tile(void *smem, const CUtensorMap *m, int swap, int tok0, int row0, int b, uint64_t *bar) {
    if (swap) tma_load_3d(smem, m, tok0, b, row0, bar);
    else tma_load_3d(smem, m, tok0, row0, b, bar);
}

// ---------------------------------------------------------------------------------------------
// pass 1
// ---------------------------------------------------------------------------------------------
template <int N> struct AggSmem { static constexpr int kWarpBytes = 4 * kRawTileBytes + kTile * N * 4 + N * kTile * 2; };

template <typename T, int N, bool kRev, bool kTma>
__global__ void __launch_bounds__(kWarpsPerCta * 32, scan_minb<N>(4)) scan_fwd_agg2_kernel(const ScanP p, const __grid_constant__ ScanTmaps tm) {
    static_assert(sizeof(T) == 2, "the pipelined variant is for 16-bit activations");
    extern __shared__ __align__(1024) float smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int w = blockIdx.x * kWarpsPerCta + warp;
    if (w >= p.n_work) return;
    const WorkItem wi = decode_work(p, w);
    const int d = wi.d0 + lane;
    const bool active = lane < wi.nrows;

    unsigned char *wb = reinterpret_cast<unsigned char *>(smem) + (size_t)warp * AggSmem<N>::kWarpBytes;
    constexpr int kStageBytes = 2 * kRawTileBytes;           // stage s: u at wb + s * kStageBytes, delta one tile further
    float *s_B = reinterpret_cast<float *>(wb + 4 * kRawTileBytes);
    T *rawB = reinterpret_cast<T *>(wb + 4 * kRawTileBytes + kTile * N * 4);
    uint64_t *bar = reinterpret_cast<uint64_t *>(reinterpret_cast<unsigned char *>(smem) + (size_t)kWarpsPerCta * AggSmem<N>::kWarpBytes) + warp;
    constexpr unsigned kTmaBytes = 2 * kRawTileBytes + N * kTile * 2;
    unsigned phase = 0;
    if (kTma) {
        if (lane == 0) mbar_init(bar, 1);
        __syncwarp();
    }

    float2 A2[N / 2], h[N / 2];
#pragma unroll
    for (int m = 0; m < N / 2; ++m) {
        A2[m] = active ? f2(p.A[(int64_t)d * N + 2 * m] * kLog2e, p.A[(int64_t)d * N + 2 * m + 1] * kLog2e) : f2(0.f, 0.f);
        h[m] = f2(0.f, 0.f);
    }
    const float bias = (active && p.delta_bias) ? p.delta_bias[d] : 0.f;
    float sumdt = 0.f;

    const T *u = reinterpret_cast<const T *>(p.u) + wi.b * p.u_bs + (int64_t)wi.d0 * p.u_ds;
    const T *dl = reinterpret_cast<const T *>(p.delta) + wi.b * p.delta_bs + (int64_t)wi.d0 * p.delta_ds;
    const T *Bm = reinterpret_cast<const T *>(p.B) + wi.b * p.B_bs + (int64_t)wi.g * p.B_gs;

    const int j_begin = wi.seg * p.S;
    const int j_end = min(p.L, j_begin + p.S);
    const bool fast = stream_aligned(u, p.u_ds, p.L, kRev) && stream_aligned(dl, p.delta_ds, p.L, kRev) && bc_aligned(Bm, p.B_ns, p.L, kRev);
    const LanePtr<T> lpu = lane_ptr(u, p.u_ds, p.L, kRev, lane), lpd = lane_ptr(dl, p.delta_ds, p.L, kRev, lane);

    int stage = 0;
    bool pending = false;
    auto tma_issue = [&](unsigned char *du, unsigned char *dd, int jt) {      // one elected lane; every tile, ragged ones included
        if (lane == 0) {
            const int tok0 = kRev ? p.L - kTile - jt : jt;
            fence_proxy_async();
            mbar_expect_tx(bar, kTmaBytes);
            tma_tile<false>(du, &tm.u, tm.swap_u, tok0, wi.d0, wi.b, bar);
            tma_tile<false>(dd, &tm.d, tm.swap_d, tok0, wi.d0, wi.b, bar);
            tma_tile<true>(rawB, &tm.B, tm.swap_B, tok0, 0, wi.b, bar);
        }
    };
    if (kTma) {
        if (j_begin < j_end) {
            tma_issue(wb, wb + kRawTileBytes, j_begin);
            pending = true;
        }
    } else if (j_begin < j_end && fast && j_begin + kTile <= p.L) {
        issue_tile<T>(wb, lpu, wi.nrows, j_begin, kRev, lane);
        issue_tile<T>(wb + kRawTileBytes, lpd, wi.nrows, j_begin, kRev, lane);
        issue_bc<T, N>(rawB, Bm, p.B_ns, j_begin, p.L, kRev, lane);
        cp_async_commit();
        pending = true;
    }
    for (int j0 = j_begin; j0 < j_end; j0 += kTile) {
        unsigned char *t_u = wb + stage * kStageBytes, *t_d = t_u + kRawTileBytes;
        unsigned char *n_u = wb + (stage ^ 1) * kStageBytes, *n_d = n_u + kRawTileBytes;
        if (kTma) {
            mbar_wait(bar, phase);
            phase ^= 1;
            convert_bc<T, N, kRev>(s_B, rawB, lane);
        } else if (pending) {
            cp_async_wait_all();
            __syncwarp();
            convert_bc<T, N, kRev>(s_B, rawB, lane);
        } else {
            fill_raw_sync<T, kRev>(t_u, u, p.u_ds, wi.nrows, j0, p.L, lane);
            fill_raw_sync<T, kRev>(t_d, dl, p.delta_ds, wi.nrows, j0, p.L, lane);
            float *const bt[1] = {s_B};
            const T *const bb[1] = {Bm};
            const int64_t bns[1] = {p.B_ns}, bls[1] = {p.B_ls};
            fill_bc_tiles<T, N, 1>(bt, bb, bns, bls, j0, p.L, kRev, lane);
        }
        __syncwarp();
        const int jn = j0 + kTile;
        const bool next_async = kTma ? jn < j_end : (jn < j_end && fast && jn + kTile <= p.L);
        if (kTma) {
            if (next_async) tma_issue(n_u, n_d, jn);
        } else if (next_async) {                            // in flight during the compute below
            issue_tile<T>(n_u, lpu, wi.nrows, jn, kRev, lane);
            issue_tile<T>(n_d, lpd, wi.nrows, jn, kRev, lane);
            issue_bc<T, N>(rawB, Bm, p.B_ns, jn, p.L, kRev, lane);
            cp_async_commit();
        }
        const int nvalid = j_end - j0;
#pragma unroll 1
        for (int u8 = 0; u8 < kTile / 8; ++u8) {
            float uu[8], dd[8];
            if (kTma) {
                read_unit_asc<T, kRev>(t_u, lane, u8, uu);
                read_unit_asc<T, kRev>(t_d, lane, u8, dd);
            } else {
                read_unit<T, kRev>(t_u, lane, u8, uu);
                read_unit<T, kRev>(t_d, lane, u8, dd);
            }
            unit_dt(dd, bias, p.softplus, 8 * u8, nvalid);
            agg_block<N, 0>(s_B + 8 * u8 * N, uu, dd, A2, h, sumdt);
        }
        __syncwarp();                                       // s_B and this stage are free for the next iteration's writers
        pending = next_async;
        stage ^= 1;
    }
    if (active) {
        const int64_t o = (((int64_t)wi.b * p.n_seg + wi.seg) * N) * p.dim + d;
#pragma unroll
        for (int m = 0; m < N / 2; ++m) {
            p.P[o + (int64_t)(2 * m) * p.dim] = ex2(A2[m].x * sumdt);
            p.P[o + (int64_t)(2 * m + 1) * p.dim] = ex2(A2[m].y * sumdt);
            p.H[o + (int64_t)(2 * m) * p.dim] = h[m].x;
            p.H[o + (int64_t)(2 * m + 1) * p.dim] = h[m].y;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// pass 3
// ---------------------------------------------------------------------------------------------
template <int N> struct MainSmem { static constexpr int kWarpBytes = 6 * kRawTileBytes + 2 * kTile * N * 4 + 2 * N * kTile * 2; };

template <typename T, int N, bool kHasZ, bool kRev, bool kTma>
__global__ void __launch_bounds__(kWarpsPerCta * 32, scan_minb<N>(3)) scan_fwd_main2_kernel(const ScanP p, const __grid_constant__ ScanTmaps tm) {
    static_assert(sizeof(T) == 2, "the pipelined variant is for 16-bit activations");
    extern __shared__ __align__(1024) float smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int w = blockIdx.x * kWarpsPerCta + warp;
    if (w >= p.n_work) return;
    const WorkItem wi = decode_work(p, w);
    const int d = wi.d0 + lane;
    const bool active = lane < wi.nrows;

    unsigned char *wb = reinterpret_cast<unsigned char *>(smem) + (size_t)warp * MainSmem<N>::kWarpBytes;
    constexpr int kStageBytes = 3 * kRawTileBytes;           // stage s: u, delta, z tiles at wb + s * kStageBytes
    float *s_B = reinterpret_cast<float *>(wb + 6 * kRawTileBytes);
    float *s_C = s_B + kTile * N;
    T *rawB = reinterpret_cast<T *>(wb + 6 * kRawTileBytes + 2 * kTile * N * 4);
    T *rawC = rawB + N * kTile;
    uint64_t *bar = reinterpret_cast<uint64_t *>(reinterpret_cast<unsigned char *>(smem) + (size_t)kWarpsPerCta * MainSmem<N>::kWarpBytes) + warp;
    constexpr unsigned kTmaBytes = (kHasZ ? 3 : 2) * kRawTileBytes + 2 * N * kTile * 2;
    unsigned phase = 0;
    if (kTma) {
        if (lane == 0) mbar_init(bar, 1);
        __syncwarp();
    }

    float2 A2[N / 2], h[N / 2];
    {
        const int64_t o = (((int64_t)wi.b * p.n_seg + wi.seg) * N) * p.dim + d;
#pragma unroll
        for (int m = 0; m < N / 2; ++m) {
            A2[m] = active ? f2(p.A[(int64_t)d * N + 2 * m] * kLog2e, p.A[(int64_t)d * N + 2 * m + 1] * kLog2e) : f2(0.f, 0.f);
            h[m] = active ? f2(p.hin[o + (int64_t)(2 * m) * p.dim], p.hin[o + (int64_t)(2 * m + 1) * p.dim]) : f2(0.f, 0.f);
        }
    }
    const float bias = (active && p.delta_bias) ? p.delta_bias[d] : 0.f;
    const float Dv = (active && p.D) ? p.D[d] : 0.f;

    const T *u = reinterpret_cast<const T *>(p.u) + wi.b * p.u_bs + (int64_t)wi.d0 * p.u_ds;
    const T *dl = reinterpret_cast<const T *>(p.delta) + wi.b * p.delta_bs + (int64_t)wi.d0 * p.delta_ds;
    const T *z = kHasZ ? reinterpret_cast<const T *>(p.z) + wi.b * p.z_bs + (int64_t)wi.d0 * p.z_ds : nullptr;
    const T *Bm = reinterpret_cast<const T *>(p.B) + wi.b * p.B_bs + (int64_t)wi.g * p.B_gs;
    const T *Cm = reinterpret_cast<const T *>(p.C) + wi.b * p.C_bs + (int64_t)wi.g * p.C_gs;
    T *out = p.out ? reinterpret_cast<T *>(p.out) + wi.b * p.out_bs + (int64_t)wi.d0 * p.out_ds : nullptr;
    T *out_z = kHasZ ? reinterpret_cast<T *>(p.out_z) + wi.b * p.out_z_bs + (int64_t)wi.d0 * p.out_z_ds : nullptr;

    const int j_begin = wi.seg * p.S;
    const int j_end = min(p.L, j_begin + p.S);
    const bool fast = stream_aligned(u, p.u_ds, p.L, kRev) && stream_aligned(dl, p.delta_ds, p.L, kRev) &&
                      (!kHasZ || stream_aligned(z, p.z_ds, p.L, kRev)) && bc_aligned(Bm, p.B_ns, p.L, kRev) &&
                      bc_aligned(Cm, p.C_ns, p.L, kRev);
    const LanePtr<T> lpu = lane_ptr(u, p.u_ds, p.L, kRev, lane), lpd = lane_ptr(dl, p.delta_ds, p.L, kRev, lane);
    const LanePtr<T> lpzi = lane_ptr(kHasZ ? z : u, kHasZ ? p.z_ds : p.u_ds, p.L, kRev, lane);
    const bool fast_out = out ? stream_aligned(out, p.out_ds, p.L, kRev) : true;
    const bool fast_oz = kHasZ ? stream_aligned(out_z, p.out_z_ds, p.L, kRev) : true;
    const LanePtr<T> lpo = lane_ptr(out ? (const T *)out : u, out ? p.out_ds : p.u_ds, p.L, kRev, lane);
    const LanePtr<T> lpz = lane_ptr(kHasZ ? (const T *)out_z : u, kHasZ ? p.out_z_ds : p.u_ds, p.L, kRev, lane);

    int stage = 0;
    bool pending = false;
    auto tma_issue = [&](unsigned char *du, unsigned char *dd, unsigned char *dz, int jt) {
        if (lane == 0) {
            const int tok0 = kRev ? p.L - kTile - jt : jt;
            fence_proxy_async();                               // the stage was last touched through the generic proxy
            mbar_expect_tx(bar, kTmaBytes);
            tma_tile<false>(du, &tm.u, tm.swap_u, tok0, wi.d0, wi.b, bar);
            tma_tile<false>(dd, &tm.d, tm.swap_d, tok0, wi.d0, wi.b, bar);
            if (kHasZ) tma_tile<false>(dz, &tm.z, tm.swap_z, tok0, wi.d0, wi.b, bar);
            tma_tile<true>(rawB, &tm.B, tm.swap_B, tok0, 0, wi.b, bar);
            tma_tile<true>(rawC, &tm.C, tm.swap_C, tok0, 0, wi.b, bar);
        }
    };
    if (kTma) {
        if (j_begin < j_end) {
            tma_issue(wb, wb + kRawTileBytes, wb + 2 * kRawTileBytes, j_begin);
            pending = true;
        }
    } else if (j_begin < j_end && fast && j_begin + kTile <= p.L) {
        issue_tile<T>(wb, lpu, wi.nrows, j_begin, kRev, lane);
        issue_tile<T>(wb + kRawTileBytes, lpd, wi.nrows, j_begin, kRev, lane);
        if (kHasZ) issue_tile<T>(wb + 2 * kRawTileBytes, lpzi, wi.nrows, j_begin, kRev, lane);
        issue_bc<T, N>(rawB, Bm, p.B_ns, j_begin, p.L, kRev, lane);
        issue_bc<T, N>(rawC, Cm, p.C_ns, j_begin, p.L, kRev, lane);
        cp_async_commit();
        pending = true;
    }
    for (int j0 = j_begin; j0 < j_end; j0 += kTile) {
        unsigned char *t_u = wb + stage * kStageBytes, *t_d = t_u + kRawTileBytes, *t_z = t_u + 2 * kRawTileBytes;
        unsigned char *n_u = wb + (stage ^ 1) * kStageBytes, *n_d = n_u + kRawTileBytes, *n_z = n_u + 2 * kRawTileBytes;
        if (p.hstates && (j0 % kCkpt) == 0 && active) {
            const int64_t o = (((int64_t)wi.b * (p.nck + 1) + j0 / kCkpt) * N) * p.dim + d;
#pragma unroll
            for (int m = 0; m < N / 2; ++m) {
                p.hstates[o + (int64_t)(2 * m) * p.dim] = h[m].x;
                p.hstates[o + (int64_t)(2 * m + 1) * p.dim] = h[m].y;
            }
        }
        if (kTma) {
            mbar_wait(bar, phase);
            phase ^= 1;
            convert_bc<T, N, kRev>(s_B, rawB, lane);
            convert_bc<T, N, kRev>(s_C, rawC, lane);
        } else if (pending) {
            cp_async_wait_all();
            __syncwarp();
            convert_bc<T, N, kRev>(s_B, rawB, lane);
            convert_bc<T, N, kRev>(s_C, rawC, lane);
        } else {
            fill_raw_sync<T, kRev>(t_u, u, p.u_ds, wi.nrows, j0, p.L, lane);
            fill_raw_sync<T, kRev>(t_d, dl, p.delta_ds, wi.nrows, j0, p.L, lane);
            if (kHasZ) fill_raw_sync<T, kRev>(t_z, z, p.z_ds, wi.nrows, j0, p.L, lane);
            float *const bt[2] = {s_B, s_C};
            const T *const bb[2] = {Bm, Cm};
            const int64_t bns[2] = {p.B_ns, p.C_ns}, bls[2] = {p.B_ls, p.C_ls};
            fill_bc_tiles<T, N, 2>(bt, bb, bns, bls, j0, p.L, kRev, lane);
        }
        __syncwarp();
        const int jn = j0 + kTile;
        const bool next_async = kTma ? jn < j_end : (jn < j_end && fast && jn + kTile <= p.L);
        if (kTma) {
            if (next_async) tma_issue(n_u, n_d, n_z, jn);
        } else if (next_async) {
            issue_tile<T>(n_u, lpu, wi.nrows, jn, kRev, lane);
            issue_tile<T>(n_d, lpd, wi.nrows, jn, kRev, lane);
            if (kHasZ) issue_tile<T>(n_z, lpzi, wi.nrows, jn, kRev, lane);
            issue_bc<T, N>(rawB, Bm, p.B_ns, jn, p.L, kRev, lane);
            issue_bc<T, N>(rawC, Cm, p.C_ns, jn, p.L, kRev, lane);
            cp_async_commit();
        }
        const int nvalid = j_end - j0;
#pragma unroll 1
        for (int u8 = 0; u8 < kTile / 8; ++u8) {
            float uu[8], dd[8], yy[8];
            if (kTma) {
                read_unit_asc<T, kRev>(t_u, lane, u8, uu);
                read_unit_asc<T, kRev>(t_d, lane, u8, dd);
            } else {
                read_unit<T, kRev>(t_u, lane, u8, uu);
                read_unit<T, kRev>(t_d, lane, u8, dd);
            }
            unit_dt(dd, bias, p.softplus, 8 * u8, nvalid);
            if (p.hd && active) dense_store<N>(p.hd + dense_slot(p, wi.b, wi.g, d, (j0 >> 3) + u8, N), h);
            main_block<N, 0>(s_B + 8 * u8 * N, s_C + 8 * u8 * N, uu, dd, Dv, A2, h, yy);
            if (kHasZ) {
                float zz[8];
                if (kTma) read_unit_asc<T, kRev>(t_z, lane, u8, zz);
                else read_unit<T, kRev>(t_z, lane, u8, zz);
#pragma unroll
                for (int e = 0; e < 8; ++e) zz[e] = yy[e] * zz[e] * sigmoidf(zz[e]);
                if (kTma) write_unit_asc<T, kRev>(t_z, lane, u8, zz);   // in place: this lane consumed the unit
                else write_unit<T, kRev>(t_z, lane, u8, zz);
            }
            if (out) {
                if (kTma) write_unit_asc<T, kRev>(t_u, lane, u8, yy);
                else write_unit<T, kRev>(t_u, lane, u8, yy);
            }
        }
        __syncwarp();
        const bool full = j0 + kTile <= p.L;
        if (kTma) {
            const int tok0 = kRev ? p.L - kTile - j0 : j0;      // >= 0 and 4-aligned whenever `full` and the fast flags hold
            if (out) {
                if (full && fast_out) store_asc_fast<T>(t_u, out + tok0, p.out_ds, wi.nrows, lane);
                else store_asc_sync<T, kRev>(t_u, out, p.out_ds, wi.nrows, j0, p.L, lane);
            }
            if (kHasZ) {
                if (full && fast_oz) store_asc_fast<T>(t_z, out_z + tok0, p.out_z_ds, wi.nrows, lane);
                else store_asc_sync<T, kRev>(t_z, out_z, p.out_z_ds, wi.nrows, j0, p.L, lane);
            }
        } else {
            if (out) {
                if (full && fast_out) store_raw_fast<T>(t_u, const_cast<T *>(lpo.lp), lpo.rowstep, wi.nrows, j0, kRev, lane);
                else store_raw_sync<T, kRev>(t_u, out, p.out_ds, wi.nrows, j0, p.L, lane);
            }
            if (kHasZ) {
                if (full && fast_oz) store_raw_fast<T>(t_z, const_cast<T *>(lpz.lp), lpz.rowstep, wi.nrows, j0, kRev, lane);
                else store_raw_sync<T, kRev>(t_z, out_z, p.out_z_ds, wi.nrows, j0, p.L, lane);
            }
        }
        __syncwarp();
        pending = next_async;
        stage ^= 1;
    }
    if (p.hstates && j_end == p.L && active) {
        const int64_t o = (((int64_t)wi.b * (p.nck + 1) + p.nck) * N) * p.dim + d;
#pragma unroll
        for (int m = 0; m < N / 2; ++m) {
            p.hstates[o + (int64_t)(2 * m) * p.dim] = h[m].x;
            p.hstates[o + (int64_t)(2 * m + 1) * p.dim] = h[m].y;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// host side (same orchestration as launch_fwd in scan_fwd.cu)
// ---------------------------------------------------------------------------------------------
// ---- tensor maps (TMA mode) ----
// rank-3 map over (L, a1, a2) with the two outer axes ordered by increasing stride; *swap = 1 when axis 1 is `second`
static bool make_map3(CUtensorMap *m, int *swap, const void *base, int L, int first_n, int64_t first_stride, int first_box, int second_n,
                      int64_t second_stride, int second_box, bool swizzle64, int dtype) {
    // size-1 axes carry no meaningful stride: give them one that keeps the strides increasing
    if (first_n == 1) first_stride = second_stride * second_n;
    if (second_n == 1) second_stride = first_stride * first_n;
    if (((uintptr_t)base & 15) || ((first_stride * 2) & 15) || ((second_stride * 2) & 15) || first_stride <= 0 || second_stride <= 0) return false;
    TmapDesc d;
    memset(&d, 0, sizeof(d));
    d.base = base; d.rank = 3; d.elem_bytes = 2; d.swizzle64 = swizzle64 ? 1 : 0;
    d.dims[0] = (uint64_t)L; d.box[0] = kTile;
    const bool sw = second_stride < first_stride;
    d.dims[1] = sw ? second_n : first_n;   d.strides[0] = (uint64_t)(sw ? second_stride : first_stride) * 2;   d.box[1] = sw ? second_box : first_box;
    d.dims[2] = sw ? first_n : second_n;   d.strides[1] = (uint64_t)(sw ? first_stride : second_stride) * 2;   d.box[2] = sw ? first_box : second_box;
    *swap = sw ? 1 : 0;
    return tmap_encode(m, d, dtype) == cudaSuccess;
}
static bool make_tmaps(ScanTmaps &tm, const ScanP &p, int N, bool has_z, int dtype) {
    if (p.G != 1 || p.B_ls != 1 || p.C_ls != 1) return false;
    // activations: (L, channel, batch), box 32 x 32 x 1, 64-byte swizzle;  B / C: (L, state, batch), box 32 x N x 1
    if (!make_map3(&tm.u, &tm.swap_u, p.u, p.L, p.dim, p.u_ds, kTile, p.batch, p.u_bs, 1, true, dtype)) return false;
    if (!make_map3(&tm.d, &tm.swap_d, p.delta, p.L, p.dim, p.delta_ds, kTile, p.batch, p.delta_bs, 1, true, dtype)) return false;
    if (has_z && !make_map3(&tm.z, &tm.swap_z, p.z, p.L, p.dim, p.z_ds, kTile, p.batch, p.z_bs, 1, true, dtype)) return false;
    if (!make_map3(&tm.B, &tm.swap_B, p.B, p.L, N, p.B_ns, N, p.batch, p.B_bs, 1, false, dtype)) return false;
    if (!make_map3(&tm.C, &tm.swap_C, p.C, p.L, N, p.C_ns, N, p.batch, p.C_bs, 1, false, dtype)) return false;
    return true;
}

template <typename T, int N, bool kRev, bool kTma>
static cudaError_t launch_fwd2(const ScanP &p, const ScanTmaps &tm, bool has_z, float *x, cudaStream_t st) {
    const int ctas = (p.n_work + kWarpsPerCta - 1) / kWarpsPerCta;
    const size_t sm1 = (size_t)kWarpsPerCta * AggSmem<N>::kWarpBytes + 64;      // + one mbarrier per warp (TMA mode)
    const size_t sm3 = (size_t)kWarpsPerCta * MainSmem<N>::kWarpBytes + 64;
    cudaError_t e;
    SMB_SET_SMEM_ONCE((scan_fwd_agg2_kernel<T, N, kRev, kTma>), sm1);
    if (p.n_seg > 1) {
        scan_fwd_agg2_kernel<T, N, kRev, kTma><<<ctas, kWarpsPerCta * 32, sm1, st>>>(p, tm); count_launch();
        if ((e = carry_launch(p.P, p.H, p.hin, x ? p.cumP : nullptr, p.batch, p.n_seg, N, p.dim, 0, st)) != cudaSuccess) return e;
    } else {
        if ((e = cudaMemsetAsync(p.hin, 0, sizeof(float) * (size_t)p.batch * N * p.dim, st)) != cudaSuccess) return e;
        if (x) {
            scan_fwd_agg2_kernel<T, N, kRev, kTma><<<ctas, kWarpsPerCta * 32, sm1, st>>>(p, tm); count_launch();
            if ((e = cudaMemcpyAsync(p.cumP, p.P, sizeof(float) * (size_t)p.batch * N * p.dim, cudaMemcpyDeviceToDevice, st)) != cudaSuccess) return e;
        }
    }
    if (has_z) {
        SMB_SET_SMEM_ONCE((scan_fwd_main2_kernel<T, N, true, kRev, kTma>), sm3);
        scan_fwd_main2_kernel<T, N, true, kRev, kTma><<<ctas, kWarpsPerCta * 32, sm3, st>>>(p, tm); count_launch();
    } else {
        SMB_SET_SMEM_ONCE((scan_fwd_main2_kernel<T, N, false, kRev, kTma>), sm3);
        scan_fwd_main2_kernel<T, N, false, kRev, kTma><<<ctas, kWarpsPerCta * 32, sm3, st>>>(p, tm); count_launch();
    }
    if (x) return x_finalize_launch(p, N, x, st);
    return cudaGetLastError();
}

template <typename T, int N>
static cudaError_t launch_fwd2_n(const ScanP &p, int dtype, int mode, bool has_z, float *x, cudaStream_t st) {
    static ScanTmaps tm_static;                                   // zeroed: what the cp.async instantiations receive
    ScanTmaps tm = tm_static;
    const bool tma = mode == 2 && make_tmaps(tm, p, N, has_z, dtype);   // falls back to cp.async when a map cannot be built
    if (tma) return p.reverse ? launch_fwd2<T, N, true, true>(p, tm, has_z, x, st) : launch_fwd2<T, N, false, true>(p, tm, has_z, x, st);
    return p.reverse ? launch_fwd2<T, N, true, false>(p, tm, has_z, x, st) : launch_fwd2<T, N, false, false>(p, tm, has_z, x, st);
}

template <typename T>
static cudaError_t launch_fwd2_t(const ScanP &p, int dtype, int N, int mode, bool has_z, float *x, cudaStream_t st) {
    switch (N) {
        case 64: return launch_fwd2_n<T, 64>(p, dtype, mode, has_z, x, st);
        case 32: return launch_fwd2_n<T, 32>(p, dtype, mode, has_z, x, st);
        case 16: return launch_fwd2_n<T, 16>(p, dtype, mode, has_z, x, st);
        default: return launch_fwd2_n<T, 8>(p, dtype, mode, has_z, x, st);
    }
}

cudaError_t scan_fwd_v2_dispatch(const ScanP &p, int dtype, int N, bool has_z, float *x, int mode, cudaStream_t st) {
    if (dtype == 1) return launch_fwd2_t<__half>(p, dtype, N, mode, has_z, x, st);
    return launch_fwd2_t<__nv_bfloat16>(p, dtype, N, mode, has_z, x, st);
}

}  // namespace smb
