// R1 of the backward selective scan (reverse aggregate per 256-position chunk), software-pipelined variant for 16-bit
// activations (opt-in: SMB_RAGG_V2=1).  Same arithmetic as scan_bwd_ragg_kernel in scan_bwd.cu; the tiles reach the SM the
// way scan_fwd_v2.cu does it: delta / dout / z stay in their storage type in two alternating cp.async stages and are
// converted (softplus, gate gradient) in registers when a lane reads its 8 positions, C goes through a raw staging row buffer
// into the broadcast tile.  The walk is descending, so the tile prefetched during the compute of tile j0 is j0 - 32.
#include "raw_tiles.cuh"
#include "scan_internal.h"
#include "scan_steps.cuh"

namespace smb {

template <int N> struct RaggSmem { static constexpr int kWarpBytes = 6 * kRawTileBytes + kTile * N * 4 + N * kTile * 2; };

template <typename T, int N, bool kHasZ, bool kRev>
__global__ void __launch_bounds__(kWarpsPerCta * 32, scan_minb<N>(3)) scan_bwd_ragg2_kernel(const ScanP p) {
    static_assert(sizeof(T) == 2, "the pipelined variant is for 16-bit activations");
    extern __shared__ __align__(16) float smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int w = blockIdx.x * kWarpsPerCta + warp;
    if (w >= p.n_work) return;
    const WorkItem wi = decode_work(p, w);          // S == kCkpt, n_seg == nck
    const int d = wi.d0 + lane;
    const bool active = lane < wi.nrows;

    unsigned char *wb = reinterpret_cast<unsigned char *>(smem) + (size_t)warp * RaggSmem<N>::kWarpBytes;
    constexpr int kStageBytes = 3 * kRawTileBytes;           // stage s: delta, dout, z tiles at wb + s * kStageBytes
    float *s_C = reinterpret_cast<float *>(wb + 6 * kRawTileBytes);
    T *rawC = reinterpret_cast<T *>(wb + 6 * kRawTileBytes + kTile * N * 4);

    float2 A2[N / 2], mu[N / 2];
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
    const bool fast = stream_aligned(dl, p.delta_ds, p.L, kRev) && stream_aligned(go, p.dout_ds, p.L, kRev) &&
                      (!kHasZ || stream_aligned(z, p.z_ds, p.L, kRev)) && bc_aligned(Cm, p.C_ns, p.L, kRev);
    const LanePtr<T> lpd = lane_ptr(dl, p.delta_ds, p.L, kRev, lane), lpg = lane_ptr(go, p.dout_ds, p.L, kRev, lane);
    const LanePtr<T> lpz = lane_ptr(kHasZ ? z : dl, kHasZ ? p.z_ds : p.delta_ds, p.L, kRev, lane);

    int stage = 0;
    bool pending = false;
    if (fast && last_tile + kTile <= p.L) {
        issue_tile<T>(wb, lpd, wi.nrows, last_tile, kRev, lane);
        issue_tile<T>(wb + kRawTileBytes, lpg, wi.nrows, last_tile, kRev, lane);
        if (kHasZ) issue_tile<T>(wb + 2 * kRawTileBytes, lpz, wi.nrows, last_tile, kRev, lane);
        issue_bc<T, N>(rawC, Cm, p.C_ns, last_tile, p.L, kRev, lane);
        cp_async_commit();
        pending = true;
    }
    for (int j0 = last_tile; j0 >= j_begin; j0 -= kTile) {
        unsigned char *t_d = wb + stage * kStageBytes, *t_g = t_d + kRawTileBytes, *t_z = t_d + 2 * kRawTileBytes;
        unsigned char *n_d = wb + (stage ^ 1) * kStageBytes, *n_g = n_d + kRawTileBytes, *n_z = n_d + 2 * kRawTileBytes;
        if (pending) {
            cp_async_wait_all();
            __syncwarp();
            convert_bc<T, N, kRev>(s_C, rawC, lane);
        } else {
            fill_raw_sync<T, kRev>(t_d, dl, p.delta_ds, wi.nrows, j0, p.L, lane);
            fill_raw_sync<T, kRev>(t_g, go, p.dout_ds, wi.nrows, j0, p.L, lane);
            if (kHasZ) fill_raw_sync<T, kRev>(t_z, z, p.z_ds, wi.nrows, j0, p.L, lane);
            float *const bt[1] = {s_C};
            const T *const bb[1] = {Cm};
            const int64_t bns[1] = {p.C_ns}, bls[1] = {p.C_ls};
            fill_bc_tiles<T, N, 1>(bt, bb, bns, bls, j0, p.L, kRev, lane);
        }
        __syncwarp();
        const int jn = j0 - kTile;
        const bool next_async = jn >= j_begin && fast;          // every tile below the last one is full
        if (next_async) {
            issue_tile<T>(n_d, lpd, wi.nrows, jn, kRev, lane);
            issue_tile<T>(n_g, lpg, wi.nrows, jn, kRev, lane);
            if (kHasZ) issue_tile<T>(n_z, lpz, wi.nrows, jn, kRev, lane);
            issue_bc<T, N>(rawC, Cm, p.C_ns, jn, p.L, kRev, lane);
            cp_async_commit();
        }
        const int nvalid = j_end - j0;
#pragma unroll 1
        for (int u8 = kTile / 8 - 1; u8 >= 0; --u8) {            // units of 8 positions, descending
            float dd[8], gg[8];
            read_unit<T, kRev>(t_d, lane, u8, dd);
            read_unit<T, kRev>(t_g, lane, u8, gg);
            unit_dt(dd, bias, p.softplus, 8 * u8, nvalid);       // masked positions: a = 1, and g == 0 there (zero fill)
            if (kHasZ) {
                float zz[8];
                read_unit<T, kRev>(t_z, lane, u8, zz);
#pragma unroll
                for (int e = 0; e < 8; ++e) gg[e] *= zz[e] * sigmoidf(zz[e]);
            }
            ragg_block<N, 7>(s_C + 8 * u8 * N, gg, dd, A2, mu, sumdt);
            const int blk = (j0 >> 3) + u8;                      // block just finished; its left neighbour starts from mu
            if (p.md && active && (blk & 31)) dense_store<N>(p.md + dense_slot(p, wi.b, wi.g, d, blk - 1, N), mu);
        }
        __syncwarp();
        pending = next_async;
        stage ^= 1;
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

template <typename T, int N, bool kHasZ, bool kRev>
static cudaError_t launch_ragg2(const ScanP &p, cudaStream_t st) {
    const int ctas = (p.n_work + kWarpsPerCta - 1) / kWarpsPerCta;
    const size_t sm = (size_t)kWarpsPerCta * RaggSmem<N>::kWarpBytes;
    cudaError_t e;
    SMB_SET_SMEM_ONCE((scan_bwd_ragg2_kernel<T, N, kHasZ, kRev>), sm);
    scan_bwd_ragg2_kernel<T, N, kHasZ, kRev><<<ctas, kWarpsPerCta * 32, sm, st>>>(p); count_launch();
    return cudaGetLastError();
}
template <typename T, int N>
static cudaError_t launch_ragg2_n(const ScanP &p, bool has_z, cudaStream_t st) {
    if (has_z) return p.reverse ? launch_ragg2<T, N, true, true>(p, st) : launch_ragg2<T, N, true, false>(p, st);
    return p.reverse ? launch_ragg2<T, N, false, true>(p, st) : launch_ragg2<T, N, false, false>(p, st);
}

template <typename T>
static cudaError_t launch_ragg2_t(const ScanP &p, int N, bool has_z, cudaStream_t st) {
    switch (N) {
        case 64: return launch_ragg2_n<T, 64>(p, has_z, st);
        case 32: return launch_ragg2_n<T, 32>(p, has_z, st);
        case 16: return launch_ragg2_n<T, 16>(p, has_z, st);
        default: return launch_ragg2_n<T, 8>(p, has_z, st);
    }
}

cudaError_t scan_bwd_ragg_v2_dispatch(const ScanP &p, int dtype, int N, bool has_z, cudaStream_t st) {
    if (dtype == 1) return launch_ragg2_t<__half>(p, N, has_z, st);
    return launch_ragg2_t<__nv_bfloat16>(p, N, has_z, st);
}

}  // namespace smb
