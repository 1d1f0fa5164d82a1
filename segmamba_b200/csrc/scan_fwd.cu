// Forward selective scan for sm_90a: lane-per-channel, three passes.
//
//   pass 1  scan_fwd_agg_kernel   per (batch, 32-channel tile, segment): zero-initialised recurrence over the
//                                 segment -> aggregate (P = prod a, H = state) per state          [1 ex2 / update]
//   pass 2  carry_kernel          per (batch, state, channel): exclusive scan of the (P, H) monoid over segments
//                                 (the SSMScanOp monoid of selective_scan_common.h:110-115)      [tiny]
//   pass 3  scan_fwd_main_kernel  same walk, seeded with the carried state, fused softplus, B.dt.u input
//                                 projection, C contraction, D skip and SiLU(z) gate             [1 ex2 / update]
//
// Mapping: one warp owns 32 channels (lane == channel) x one segment of S scan positions and keeps all
// `N` states of its channel in registers; B/C for a position are broadcast-read from a warp-private
// shared-memory tile, so B and C are fetched once per 32 channels instead of once per channel
// (the reference re-reads them per channel CTA, selective_scan_fwd_kernel.cuh:182-194).
// Restates selective_scan_fwd_kernel (selective_scan_fwd_kernel.cuh:67-303); see DESIGN.md.
#include "scan_internal.h"
#include "scan_steps.cuh"

namespace smb {

// ---------------------------------------------------------------------------------------------
// pass 1
// ---------------------------------------------------------------------------------------------
template <typename T, int N>
__global__ void __launch_bounds__(kWarpsPerCta * 32) scan_fwd_agg_kernel(const ScanP p) {
    extern __shared__ __align__(16) float smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int w = blockIdx.x * kWarpsPerCta + warp;
    if (w >= p.n_work) return;
    const WorkItem wi = decode_work(p, w);
    const int d = wi.d0 + lane;
    const bool active = lane < wi.nrows;

    float *s_u = smem + warp * (2 * kTile * kTile + kTile * N);
    float *s_dt = s_u + kTile * kTile;
    float *s_B = s_dt + kTile * kTile;

    float2 A2[N / 2], h[N / 2];                       // state pairs (2m, 2m+1) packed for FFMA2
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
        prepass_dt(s_dt, lane, bias, p.softplus, j_end - j0);      // masked positions become scan identities
#pragma unroll 1
        for (int c0 = 0; c0 < kTile / 4; c0 += 2) {      // blocks of 8 positions: all shared offsets are constants
            const float *blkB = s_B + 4 * c0 * N;
            const float4 ua = tile_read4(s_u, lane, c0), ub = tile_read4(s_u, lane, c0 + 1);
            const float4 da = tile_read4(s_dt, lane, c0), db = tile_read4(s_dt, lane, c0 + 1);
            const float uu[8] = {ua.x, ua.y, ua.z, ua.w, ub.x, ub.y, ub.z, ub.w};
            const float dd[8] = {da.x, da.y, da.z, da.w, db.x, db.y, db.z, db.w};
            agg_block<N, 0>(blkB, uu, dd, A2, h, sumdt);
        }
        __syncwarp();
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
// pass 2: exclusive scan over segments of (P, H) under (P2,H2) o (P1,H1) = (P1 P2, P2 H1 + H2).
// Block = (32 channels) x (32 segment groups); each thread first reduces its group of segments,
// a 32-step shared-memory prefix links the groups, then the thread re-walks its group writing the
// incoming state of every segment.  `reverse_carry` scans from the last segment down (backward pass).
// Layout of P, H, hin, cumP: (batch, n_seg, N, dim), dim fastest.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) carry_kernel(const float *__restrict__ P, const float *__restrict__ H,
                                                     float *__restrict__ hin, float *__restrict__ cumP, int n_seg,
                                                     int N, int dim, int reverse_carry) {
    __shared__ float sP[32][33], sH[32][33];
    const int dl = threadIdx.x & 31, grp = threadIdx.x >> 5;
    const int d = blockIdx.x * 32 + dl;
    const int n = blockIdx.y, b = blockIdx.z;
    const int per = (n_seg + 31) / 32;
    const int s_lo = grp * per, s_hi = min(n_seg, s_lo + per);
    const bool active = d < dim;
    const int64_t base = ((int64_t)b * n_seg * N + n) * dim + d;
    const int64_t sstride = (int64_t)N * dim;
    // phase A: group aggregate
    float gp = 1.f, gh = 0.f;
    if (active) {
        if (!reverse_carry) {
            for (int s = s_lo; s < s_hi; ++s) {
                const float ps = P[base + s * sstride], hs = H[base + s * sstride];
                gh = fmaf(ps, gh, hs);
                gp *= ps;
            }
        } else {
            for (int s = s_hi - 1; s >= s_lo; --s) {
                const float ps = P[base + s * sstride], hs = H[base + s * sstride];
                gh = fmaf(ps, gh, hs);
                gp *= ps;
            }
        }
    }
    sP[grp][dl] = gp;
    sH[grp][dl] = gh;
    __syncthreads();
    // phase B: incoming state of this group = combination of all earlier (later, if reverse) groups
    float hcar = 0.f, pcar = 1.f;
    if (!reverse_carry) {
        for (int g2 = 0; g2 < grp; ++g2) {
            hcar = fmaf(sP[g2][dl], hcar, sH[g2][dl]);
            pcar *= sP[g2][dl];
        }
    } else {
        for (int g2 = 31; g2 > grp; --g2) {
            hcar = fmaf(sP[g2][dl], hcar, sH[g2][dl]);
            pcar *= sP[g2][dl];
        }
    }
    // phase C: write the incoming state of each segment (and the running product, forward only)
    if (active) {
        if (!reverse_carry) {
            for (int s = s_lo; s < s_hi; ++s) {
                const float ps = P[base + s * sstride], hs = H[base + s * sstride];
                hin[base + s * sstride] = hcar;
                hcar = fmaf(ps, hcar, hs);
                pcar *= ps;
                if (cumP) cumP[base + s * sstride] = pcar;
            }
        } else {
            for (int s = s_hi - 1; s >= s_lo; --s) {
                const float ps = P[base + s * sstride], hs = H[base + s * sstride];
                hin[base + s * sstride] = hcar;
                hcar = fmaf(ps, hcar, hs);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// pass 3
// ---------------------------------------------------------------------------------------------
template <typename T, int N, bool kHasZ>
__global__ void __launch_bounds__(kWarpsPerCta * 32, SMB_FWD_MAIN_MINB) scan_fwd_main_kernel(const ScanP p) {
    extern __shared__ __align__(16) float smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int w = blockIdx.x * kWarpsPerCta + warp;
    if (w >= p.n_work) return;
    const WorkItem wi = decode_work(p, w);
    const int d = wi.d0 + lane;
    const bool active = lane < wi.nrows;

    float *s_u = smem + warp * (3 * kTile * kTile + 2 * kTile * N);
    float *s_dt = s_u + kTile * kTile;
    float *s_z = s_dt + kTile * kTile;
    float *s_B = s_z + kTile * kTile;
    float *s_C = s_B + kTile * N;

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
    const bool fast = stream_aligned(u, p.u_ds, p.L, p.reverse) && stream_aligned(dl, p.delta_ds, p.L, p.reverse) &&
                      (!kHasZ || stream_aligned(z, p.z_ds, p.L, p.reverse));
    const LanePtr<T> lps[3] = {lane_ptr(u, p.u_ds, p.L, p.reverse, lane), lane_ptr(dl, p.delta_ds, p.L, p.reverse, lane),
                               lane_ptr(kHasZ ? z : u, kHasZ ? p.z_ds : p.u_ds, p.L, p.reverse, lane)};
    const bool fast_out = out ? stream_aligned(out, p.out_ds, p.L, p.reverse) : true;
    const bool fast_oz = kHasZ ? stream_aligned(out_z, p.out_z_ds, p.L, p.reverse) : true;
    const LanePtr<T> lpo = lane_ptr(out ? (const T *)out : u, out ? p.out_ds : p.u_ds, p.L, p.reverse, lane);
    const LanePtr<T> lpz = lane_ptr(kHasZ ? (const T *)out_z : u, kHasZ ? p.out_z_ds : p.u_ds, p.L, p.reverse, lane);
    for (int j0 = j_begin; j0 < j_end; j0 += kTile) {
        if (p.hstates && (j0 % kCkpt) == 0 && active) {
            const int64_t o = (((int64_t)wi.b * (p.nck + 1) + j0 / kCkpt) * N) * p.dim + d;
#pragma unroll
            for (int m = 0; m < N / 2; ++m) {
                p.hstates[o + (int64_t)(2 * m) * p.dim] = h[m].x;
                p.hstates[o + (int64_t)(2 * m + 1) * p.dim] = h[m].y;
            }
        }
        {
            constexpr int K = kHasZ ? 3 : 2;
            float *const tiles[3] = {s_u, s_dt, s_z};
            const T *const bases[3] = {u, dl, kHasZ ? z : u};
            const int64_t strides[3] = {p.u_ds, p.delta_ds, kHasZ ? p.z_ds : p.u_ds};
            if (fast && j0 + kTile <= p.L) {
                fill_tiles_fast<T, K, 3>(tiles, lps, wi.nrows, j0, p.reverse, lane);
            } else {
                fill_tile<T>(s_u, u, p.u_ds, wi.nrows, j0, p.L, p.reverse, lane);
                fill_tile<T>(s_dt, dl, p.delta_ds, wi.nrows, j0, p.L, p.reverse, lane);
                if (kHasZ) fill_tile<T>(s_z, z, p.z_ds, wi.nrows, j0, p.L, p.reverse, lane);
            }
            float *const bt[2] = {s_B, s_C};
            const T *const bb[2] = {Bm, Cm};
            const int64_t bns[2] = {p.B_ns, p.C_ns}, bls[2] = {p.B_ls, p.C_ls};
            fill_bc_tiles<T, N, 2>(bt, bb, bns, bls, j0, p.L, p.reverse, lane);
            if (j0 + kTile < j_end) {
                prefetch_tiles<T, K, 3>(bases, strides, wi.nrows, j0 + kTile, p.L, p.reverse, lane);
                prefetch_bc<T, N, 2>(bb, bns, bls, j0 + kTile, p.L, p.reverse, lane);
            }
        }
        __syncwarp();
        prepass_dt(s_dt, lane, bias, p.softplus, j_end - j0);      // masked positions become scan identities
        if (kHasZ) prepass_silu(s_z, lane);
#pragma unroll 1
        for (int c0 = 0; c0 < kTile / 4; c0 += 2) {      // blocks of 8 positions: all shared offsets are constants
            const float *blkB = s_B + 4 * c0 * N, *blkC = s_C + 4 * c0 * N;
            const float4 ua = tile_read4(s_u, lane, c0), ub = tile_read4(s_u, lane, c0 + 1);
            const float4 da = tile_read4(s_dt, lane, c0), db = tile_read4(s_dt, lane, c0 + 1);
            const float uu[8] = {ua.x, ua.y, ua.z, ua.w, ub.x, ub.y, ub.z, ub.w};
            const float dd[8] = {da.x, da.y, da.z, da.w, db.x, db.y, db.z, db.w};
            float yy[8];
            if (p.hd && active) dense_store<N>(p.hd + dense_slot(p, wi.b, wi.g, d, (j0 + 4 * c0) >> 3, N), h);
            main_block<N, 0>(blkB, blkC, uu, dd, Dv, A2, h, yy);
            if (kHasZ) {
                const float4 za = tile_read4(s_z, lane, c0), zb = tile_read4(s_z, lane, c0 + 1);   // already silu(z)
                tile_write4(s_z, lane, c0, make_float4(yy[0] * za.x, yy[1] * za.y, yy[2] * za.z, yy[3] * za.w));
                tile_write4(s_z, lane, c0 + 1, make_float4(yy[4] * zb.x, yy[5] * zb.y, yy[6] * zb.z, yy[7] * zb.w));
            }
            // in-place: the same lane that consumed (row, c) overwrites it
            tile_write4(s_u, lane, c0, make_float4(yy[0], yy[1], yy[2], yy[3]));
            tile_write4(s_u, lane, c0 + 1, make_float4(yy[4], yy[5], yy[6], yy[7]));
        }
        __syncwarp();
        const bool full = j0 + kTile <= p.L;
        if (out) {
            if (full && fast_out) store_tile_fast<T>(s_u, const_cast<T *>(lpo.lp), lpo.rowstep, wi.nrows, j0, p.reverse, lane);
            else store_tile<T>(s_u, out, p.out_ds, wi.nrows, j0, p.L, p.reverse, lane);
        }
        if (kHasZ) {
            if (full && fast_oz) store_tile_fast<T>(s_z, const_cast<T *>(lpz.lp), lpz.rowstep, wi.nrows, j0, p.reverse, lane);
            else store_tile<T>(s_z, out_z, p.out_z_ds, wi.nrows, j0, p.L, p.reverse, lane);
        }
        __syncwarp();
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
// x = the reference's per-2048-chunk running state (selective_scan_fwd_kernel.cuh:251-254):
// x[b,d,c,2n] = prod of exp(dt A) from position 0 to the chunk end, x[b,d,c,2n+1] = h at the chunk end.
// ---------------------------------------------------------------------------------------------
__global__ void x_finalize_kernel(const float *__restrict__ hstates, const float *__restrict__ cumP, float *__restrict__ x,
                                  int batch, int dim, int N, int L, int S, int n_seg, int nck, int n_chunks) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t total = (int64_t)batch * dim * n_chunks * N;
    if (idx >= total) return;
    const int n = idx % N;
    const int c = (idx / N) % n_chunks;
    const int d = (idx / ((int64_t)N * n_chunks)) % dim;
    const int b = idx / ((int64_t)N * n_chunks * dim);
    const int end = min(L, (c + 1) * 2048);                 // scan positions covered up to here
    const int ck = (end == L) ? nck : end / kCkpt;
    const int se = (end + S - 1) / S - 1;
    const float hv = hstates[(((int64_t)b * (nck + 1) + ck) * N + n) * dim + d];
    const float pv = cumP[(((int64_t)b * n_seg + se) * N + n) * dim + d];
    float *xo = x + (((int64_t)b * dim + d) * n_chunks + c) * 2 * N;
    xo[2 * n] = pv;
    xo[2 * n + 1] = hv;
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
template <typename T, int N>
static cudaError_t launch_fwd(const ScanP &p, bool has_z, float *x, cudaStream_t st) {
    const int ctas = (p.n_work + kWarpsPerCta - 1) / kWarpsPerCta;
    const size_t sm1 = (size_t)kWarpsPerCta * (2 * kTile * kTile + kTile * N) * sizeof(float);
    const size_t sm3 = (size_t)kWarpsPerCta * (3 * kTile * kTile + 2 * kTile * N) * sizeof(float);
    cudaError_t e;
    SMB_SET_SMEM_ONCE((scan_fwd_agg_kernel<T, N>), sm1);
    if (p.n_seg > 1) {
        scan_fwd_agg_kernel<T, N><<<ctas, kWarpsPerCta * 32, sm1, st>>>(p); count_launch();
        dim3 cg((p.dim + 31) / 32, N, p.batch);
        carry_kernel<<<cg, 1024, 0, st>>>(p.P, p.H, p.hin, x ? p.cumP : nullptr, p.n_seg, N, p.dim, 0); count_launch();
    } else {
        // single segment: incoming state is zero; cumP (only for x) still needs pass 1
        if ((e = cudaMemsetAsync(p.hin, 0, sizeof(float) * (size_t)p.batch * N * p.dim, st)) != cudaSuccess) return e;
        if (x) {
            scan_fwd_agg_kernel<T, N><<<ctas, kWarpsPerCta * 32, sm1, st>>>(p); count_launch();
            if ((e = cudaMemcpyAsync(p.cumP, p.P, sizeof(float) * (size_t)p.batch * N * p.dim, cudaMemcpyDeviceToDevice, st)) != cudaSuccess) return e;
        }
    }
    if (has_z) {
        SMB_SET_SMEM_ONCE((scan_fwd_main_kernel<T, N, true>), sm3);
        scan_fwd_main_kernel<T, N, true><<<ctas, kWarpsPerCta * 32, sm3, st>>>(p); count_launch();
    } else {
        SMB_SET_SMEM_ONCE((scan_fwd_main_kernel<T, N, false>), sm3);
        scan_fwd_main_kernel<T, N, false><<<ctas, kWarpsPerCta * 32, sm3, st>>>(p); count_launch();
    }
    if (x) {
        const int n_chunks = (p.L + 2047) / 2048;
        const int64_t total = (int64_t)p.batch * p.dim * n_chunks * N;
        x_finalize_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(p.hstates, p.cumP, x, p.batch, p.dim, N, p.L, p.S,
                                                                          p.n_seg, p.nck, n_chunks); count_launch();
    }
    return cudaGetLastError();
}

template <typename T>
static cudaError_t launch_fwd_n(const ScanP &p, int N, bool has_z, float *x, cudaStream_t st) {
    if (N == 16) return launch_fwd<T, 16>(p, has_z, x, st);
    return launch_fwd<T, 8>(p, has_z, x, st);
}

cudaError_t x_finalize_launch(const ScanP &p, int N, float *x, cudaStream_t st) {
    const int n_chunks = (p.L + 2047) / 2048;
    const int64_t total = (int64_t)p.batch * p.dim * n_chunks * N;
    x_finalize_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(p.hstates, p.cumP, x, p.batch, p.dim, N, p.L, p.S, p.n_seg, p.nck,
                                                                      n_chunks); count_launch();
    return cudaGetLastError();
}

cudaError_t scan_fwd_dispatch(const ScanP &p, int dtype, int N, bool has_z, float *x, cudaStream_t st) {
    {   // 16-bit activations: software-pipelined kernels, tiles staged by TMA (mode 2; falls back to cp.async staging, mode 1,
        // when no tensor map can describe the operands).  SMB_FWD_V2=0 selects the single-buffered kernels below, =1 the
        // cp.async staging -- A/B switches, read per call.
        const char *v2 = getenv("SMB_FWD_V2");
        const int mode = (v2 && v2[0] >= '0' && v2[0] <= '2') ? v2[0] - '0' : 2;
        if (dtype != 0 && mode) return scan_fwd_v2_dispatch(p, dtype, N, has_z, x, mode, st);
    }
    switch (dtype) {
        case 0: return launch_fwd_n<float>(p, N, has_z, x, st);
        case 1: return launch_fwd_n<__half>(p, N, has_z, x, st);
        default: return launch_fwd_n<__nv_bfloat16>(p, N, has_z, x, st);
    }
}

// exposed for the backward pass (forward-state recompute) and tests
template <typename T, int N>
static cudaError_t launch_agg_only(const ScanP &p, cudaStream_t st) {
    const int ctas = (p.n_work + kWarpsPerCta - 1) / kWarpsPerCta;
    const size_t sm1 = (size_t)kWarpsPerCta * (2 * kTile * kTile + kTile * N) * sizeof(float);
    cudaError_t e;
    SMB_SET_SMEM_ONCE((scan_fwd_agg_kernel<T, N>), sm1);
    scan_fwd_agg_kernel<T, N><<<ctas, kWarpsPerCta * 32, sm1, st>>>(p); count_launch();
    return cudaGetLastError();
}

cudaError_t scan_fwd_agg_dispatch(const ScanP &p, int dtype, int N, cudaStream_t st) {
#define SMB_AGG(T) (N == 16 ? launch_agg_only<T, 16>(p, st) : launch_agg_only<T, 8>(p, st))
    switch (dtype) {
        case 0: return SMB_AGG(float);
        case 1: return SMB_AGG(__half);
        default: return SMB_AGG(__nv_bfloat16);
    }
#undef SMB_AGG
}

cudaError_t carry_launch(const float *P, const float *H, float *hin, float *cumP, int batch, int n_seg, int N, int dim,
                         int reverse_carry, cudaStream_t st) {
    dim3 cg((dim + 31) / 32, N, batch);
    carry_kernel<<<cg, 1024, 0, st>>>(P, H, hin, cumP, n_seg, N, dim, reverse_carry); count_launch();
    return cudaGetLastError();
}

}  // namespace smb
