// Internal parameter block shared by the scan kernels (device + host).
#pragma once

#include <cstdlib>

#include "common.cuh"

namespace smb {

// Build-time tuning knobs (tools/build_variants.py builds alternative libraries with -D overrides; the defaults are the
// hardware-verified configuration and leave the generated code unchanged).
#ifndef SMB_WARPS_PER_CTA
#define SMB_WARPS_PER_CTA 4
#endif
#ifndef SMB_FWD_MAIN_MINB
#define SMB_FWD_MAIN_MINB 3
#endif
constexpr int kWarpsPerCta = SMB_WARPS_PER_CTA;   // independent warps per CTA in the lane-per-channel kernels
// Minimum resident CTAs per SM asked of ptxas (it sets the register cap).  8 and 16 states keep the tuned value; at 32 / 64 states a
// lane holds 2-4x the state, and the per-warp shared tiles grow with N so that they bound the residency before registers do.
template <int N> constexpr int scan_minb(int tuned) { return N <= 16 ? tuned : (N == 32 && tuned > 2 ? 2 : 1); }

struct ScanP {
    int batch, dim, L, G;
    int dim_per_group, tiles_per_group, n_tiles;   // 32-channel tiles never straddle a B/C group
    int S, n_seg, n_work, nck;                     // segment length, #segments, #warp work items, #checkpoints
    bool reverse, softplus;
    const void *u, *delta, *z, *B, *C, *dout;
    const float *A, *D, *delta_bias;
    void *out, *out_z;
    float *hstates;
    int64_t u_bs, u_ds, delta_bs, delta_ds, z_bs, z_ds, out_bs, out_ds, out_z_bs, out_z_ds, dout_bs, dout_ds;
    int64_t B_bs, B_gs, B_ns, B_ls, C_bs, C_gs, C_ns, C_ls;
    float *P, *H, *hin, *cumP;                     // (batch, n_seg, N, dim) workspaces
    // ---- backward only ----
    void *du, *ddelta, *dz;
    float *dA, *dB, *dC, *dD, *ddelta_bias;        // fp32 accumulators (zero-initialised by the caller)
    int64_t du_bs, du_ds, ddelta_bs, ddelta_ds, dz_bs, dz_ds;
    const float *hs;                               // forward states at every kCkpt-th position: (batch, *, N, dim)
    int64_t hs_bs;                                 // batch stride of hs in floats
    float *Pb, *Mloc, *Min;                        // (batch, nck, N, dim) reverse aggregates / carried adjoints
    void *stash;                                   // (batch, Lpad, N/2, dim) state pairs (bf16x2 or float2), or nullptr
    int Lpad;
    // dense checkpoints (every 8th scan position), see dense_slot(): hd = forward state entering a block (written by the
    // forward main pass, read by R3), md = local adjoint entering a block from the right (written by R1, read by R3)
    float *hd, *md;
    int opc;                                       // R3: channel octets handled by one CTA (scan_bwd_r3v2.cu)
    int dbg;                                       // timing experiments only (SMB_R3_DBG, results are wrong when set): see scan_bwd_r3v2.cu
};

// Dense checkpoint layout, chosen for the reader: R3's CTA = (256-position chunk, channel octet) finds its 32 blocks x 8
// channels x N states in one contiguous run; the writers (lane == channel) store N consecutive floats per lane.
//   slot(b, octet, blk, w) = (((b * n_oct + octet) * (nck * 32) + blk) * 8 + w) * N,   octet / w from the channel's index in its group
__host__ __device__ __forceinline__ int dense_octs(int dim_per_group, int G) { return ((dim_per_group + 7) >> 3) * G; }
__device__ __forceinline__ int64_t dense_slot(const ScanP &p, int b, int g, int d, int blk, int N) {
    const int dg = d - g * p.dim_per_group;
    const int opg = (p.dim_per_group + 7) >> 3;
    return ((((int64_t)b * (opg * p.G) + g * opg + (dg >> 3)) * ((int64_t)p.nck * 32) + blk) * 8 + (dg & 7)) * N;
}
template <int N>
__device__ __forceinline__ void dense_store(float *dst, const float2 (&v)[N / 2]) {
#pragma unroll
    for (int k = 0; k < N / 4; ++k) *reinterpret_cast<float4 *>(dst + 4 * k) = make_float4(v[2 * k].x, v[2 * k].y, v[2 * k + 1].x, v[2 * k + 1].y);
}

// Per-state scalar of one channel held across a warp: state n lives in lane n & 31 of `lo` (n < 32) or `hi` (64 states)
template <int N> __device__ __forceinline__ float state_shfl(float lo, float hi, int n) {
    if constexpr (N > 32) return __shfl_sync(0xffffffffu, n < 32 ? lo : hi, n & 31);
    else return __shfl_sync(0xffffffffu, lo, n);
}
// B / C staging of the warp-per-channel R3 kernels for more than 32 states: thread t <-> position jc + t, states in rounds of 32 so
// that at most 2 x 32 loads are in flight (32 states and fewer stage in one round, inline in the kernels)
template <typename T, int N, int kPitch>
__device__ __forceinline__ void stage_bc_rounds(float *sB, float *sC, const T *Bm, const T *Cm, int64_t B_ns, int64_t C_ns, int64_t B_ls,
                                                int64_t C_ls, int jc, int L, bool rev, int t, int so) {
    const int j = jc + t;
    const bool valid = j < L;
    const int tok = pos_to_tok(valid ? j : 0, L, rev);
#pragma unroll
    for (int n0 = 0; n0 < N; n0 += 32) {
        T vb[32], vc[32];
#pragma unroll
        for (int n = 0; n < 32; ++n) {
            vb[n] = valid ? Bm[(int64_t)(n0 + n) * B_ns + (int64_t)tok * B_ls] : from_f32<T>(0.f);
            vc[n] = valid ? Cm[(int64_t)(n0 + n) * C_ns + (int64_t)tok * C_ls] : from_f32<T>(0.f);
        }
#pragma unroll
        for (int n = 0; n < 32; ++n) {
            sB[(n0 + n) * kPitch + so] = to_f32<T>(vb[n]);
            sC[(n0 + n) * kPitch + so] = to_f32<T>(vc[n]);
        }
    }
}

struct WorkItem {
    int b, seg, g, d0, nrows;
};

// work item w -> (batch, segment, channel tile); tiles vary fastest so that warps working on the same
// (batch, segment) -- and therefore the same B/C slab -- are co-scheduled.
__device__ __forceinline__ WorkItem decode_work(const ScanP &p, int w) {
    WorkItem wi;
    const int tile = w % p.n_tiles;
    const int rest = w / p.n_tiles;
    wi.seg = rest % p.n_seg;
    wi.b = rest / p.n_seg;
    wi.g = tile / p.tiles_per_group;
    const int tg = tile - wi.g * p.tiles_per_group;
    wi.d0 = wi.g * p.dim_per_group + tg * 32;
    wi.nrows = min(32, (wi.g + 1) * p.dim_per_group - wi.d0);
    return wi;
}

// Segment length heuristic (host): largest S in {seg_min .. 2048} that still yields >= 24 warps per SM (two waves at the
// 12-warp residency the kernels reach) on the 132 SMs of an H100; S divides 2048 so the reference's 2048-position chunk states fall on
// segment ends, and divides or is a multiple of kCkpt so checkpoints fall on tile boundaries of exactly one segment.
// Shortest segment: one 32-position tile, so that the small late-stage problems (L = 4096 / 512) still spread over the chip.
// SMB_SEG_MIN = 64 / 128 / 256 is the A/B switch (read per call).
inline int seg_min() {
    const char *e = getenv("SMB_SEG_MIN");
    const int v = e ? atoi(e) : 32;
    return (v == 64 || v == 128 || v == 256) ? v : 32;
}
inline int plan_segment(int batch, int n_tiles, int L) {
    const long target = 132L * 24;
    const int smin = seg_min();
    int S = 2048;
    while (S > smin && (long)batch * n_tiles * ((L + S - 1) / S) < target) S >>= 1;
    return S;
}

cudaError_t scan_fwd_dispatch(const ScanP &p, int dtype, int N, bool has_z, float *x, cudaStream_t st);
// software-pipelined variant for 16-bit activations, scan_fwd_v2.cu; chosen by scan_fwd_dispatch when SMB_FWD_V2 = 1 (tiles
// staged with cp.async) or 2 (tiles staged with TMA bulk tensor copies + mbarrier; falls back to 1 if a tensor map cannot be built)
cudaError_t scan_fwd_v2_dispatch(const ScanP &p, int dtype, int N, bool has_z, float *x, int mode, cudaStream_t st);
cudaError_t x_finalize_launch(const ScanP &p, int N, float *x, cudaStream_t st);
cudaError_t scan_fwd_agg_dispatch(const ScanP &p, int dtype, int N, cudaStream_t st);
// software-pipelined R1 (reverse aggregate) for 16-bit activations, scan_bwd_v2.cu; chosen by launch_bwd when SMB_RAGG_V2=1
cudaError_t scan_bwd_ragg_v2_dispatch(const ScanP &p, int dtype, int N, bool has_z, cudaStream_t st);
// second-generation R3 (main backward pass), scan_bwd_r3v2.cu; chosen by launch_bwd when SMB_R3_V2=1
cudaError_t scan_bwd_main_v2_dispatch(const ScanP &p, int dtype, int N, bool has_z, cudaStream_t st);
cudaError_t scan_bwd_dispatch(const ScanP &p, int dtype, int N, bool has_z, cudaStream_t st);
cudaError_t carry_launch(const float *P, const float *H, float *hin, float *cumP, int batch, int n_seg, int N, int dim,
                         int reverse_carry, cudaStream_t st);

}  // namespace smb
