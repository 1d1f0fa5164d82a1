// Implicit-GEMM 3x3x3 convolution (stride 1, padding 1, no bias) on channels-last activations, sm_90a: TMA -> shared memory
// -> wgmma.mma_async -> staged epilogue, on the pipeline of wgmma_pipe.cuh (the one the GEMM of gemm_tc.cu runs).
//
//   forward   Y[t, co] = sum_tap sum_ci X[t + off(tap), ci] . Wt[co, tap, ci]          M = tokens, N = C_out, K = 27 x C_in
//             The data gradient is the same product on dY with the weight flipped in all three axes and C_in / C_out
//             swapped (the caller re-lays the 27 C_in C_out weights).
//   wgrad     dW[co, tap, ci] += sum_t dY[t - off(tap), co] . X[t, ci]                  M = co, N = C_in, K = tokens, per tap
//
// X and dY are read through 5-D tensor maps (C, W, H, D, batch).  The A operand of one tap is a brick of voxels shifted by
// off(tap) = (kw - 1, kh - 1, kd - 1); the TMA unit zero-fills whatever part of the box lies outside the volume, which is the
// padding.  Batch stays its own axis, so a shift past d = 0 reads zeros and never the previous sample.  No im2col is stored.
//
// Forward tile: 128 output voxels = one brick x BN output channels.  With BN <= 128 the brick is 16 x 8 x 1 (8 x 16 x 1 for
// W <= 8) and one K block covers the three kh taps of a (kd, kw) pair from one box of bh + 2 rows (see kFoldABytes); wider
// tiles take a brick of powers of two, w first, and one tap per K block.  Input channels come in boxes of 64 (C = 48 or 96
// leaves the last box a quarter or half zero-filled: 25 % of the MMA work of those passes is spent on zeros).
// Weight gradient: see conv3d_wgrad_kernel.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>

#include "conv3d_internal.h"
#include "gemm_internal.h"
#include "wgmma_pipe.cuh"

namespace smb {
void count_launch();

namespace {

constexpr int kTaps = 27;
// Folded forward: the output brick is bw x bh x 1 with bw = 8 or 16 and bw x bh = 128, so one A box of bw x (bh + 2) rows
// serves the three kh taps of a (kd, kw) pair -- tap kh starts kh x bw rows (kh x bw x 128 bytes, a multiple of 1024) into
// it -- and the B tiles of those three taps sit side by side in the stage.  Per 128 output voxels the A traffic falls from
// 27 boxes of 128 rows to 9 of at most 160.  Wide tiles (BN > 128) would leave too few stages and keep one tap per K block.
constexpr int kFoldABytes = 16 * 10 * 128;
constexpr bool conv3d_folds(int BN) { return BN <= 128; }

template <typename T, int BN>
__global__ void __launch_bounds__(kThreads, 1) conv3d_tc_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                const __grid_constant__ CUtensorMap tmB, const Conv3dP p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    constexpr int kChunks = (BN + 63) / 64;
    constexpr bool kFold = conv3d_folds(BN);
    constexpr int a_tile = kFold ? kFoldABytes : kBM * 128;
    constexpr int b_tile = (kFold ? 3 : 1) * BN * 128;
    constexpr int stage_bytes = a_tile + ((b_tile + 1023) & ~1023);
    // bytes the TMA unit delivers per stage (a folded A box holds bw x (bh + 2) rows, at most kFoldABytes)
    const unsigned tx_bytes = (unsigned)((kFold ? p.bw * (p.bh + 2) * 128 : a_tile) + b_tile);
    uint8_t *stage0 = smem;
    uint8_t *staging = smem + (size_t)p.stages * stage_bytes;
    uint64_t *bars = reinterpret_cast<uint64_t *>(staging + kStagingBytes);
    uint64_t *full = bars, *empty = bars + kMaxStages;

    if (threadIdx.x == 0) {
        for (int s = 0; s < p.stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kConsumerWarps); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    }
    __syncthreads();

    const int n_work = p.m_tiles * p.n_tiles;

    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (threadIdx.x == 0) {
            unsigned it = 0;
            for (int t = blockIdx.x; t < n_work; t += gridDim.x) {
                const int nb = t % p.n_tiles, mb = t / p.n_tiles;
                int r = mb;                                            // the output brick of this tile
                const int w0 = (r % p.tw) * p.bw; r /= p.tw;
                const int h0 = (r % p.th) * p.bh; r /= p.th;
                const int d0 = (r % p.td) * p.bd; const int n = r / p.td;
                for (int kb = 0; kb < p.kb_total; ++kb, ++it) {
                    const int s = it % p.stages;
                    mbar_wait(&empty[s], ((it / p.stages) & 1) ^ 1);
                    uint8_t *sa = stage0 + (size_t)s * stage_bytes, *sb = sa + a_tile;
                    mbar_expect_tx(&full[s], tx_bytes);
                    if (kFold) {                                       // K block = (kd, kw, channel box); kh = 0, 1, 2 inside
                        const int kd = kb / (3 * p.cb), kw = (kb / p.cb) % 3, c = (kb % p.cb) * kBK;
                        tma_load_5d(sa, &tmA, c, w0 + kw - 1, h0 - 1, d0 + kd - 1, n, &full[s]);
#pragma unroll
                        for (int kh = 0; kh < 3; ++kh) tma_load_3d(sb + kh * BN * 128, &tmB, c, kd * 9 + kh * 3 + kw, nb * BN, &full[s]);
                    } else {
                        const int tap = kb / p.cb, c = (kb % p.cb) * kBK;
                        const int kd = tap / 9, kh = (tap / 3) % 3, kw = tap % 3;
                        tma_load_5d(sa, &tmA, c, w0 + kw - 1, h0 + kh - 1, d0 + kd - 1, n, &full[s]);
                        tma_load_3d(sb, &tmB, c, tap, nb * BN, &full[s]);
                    }
                }
            }
        }
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
        const int cw = (warp >> 2) - 1, wq = warp & 3;
        T *const out = reinterpret_cast<T *>(p.out);
        uint8_t *stg = staging + (size_t)(warp - 4) * (16 * kPitch);
        const unsigned stage0_addr = smem_u32(stage0);
        float acc[kChunks][32];
        unsigned it = 0;
        for (int t = blockIdx.x; t < n_work; t += gridDim.x) {
            const int nb = t % p.n_tiles, mb = t / p.n_tiles;
            if constexpr (kFold)       // tap kh reads the box bw rows (= one h-row, a multiple of 1024 bytes) further on
                consume_tile<T, BN, 0, 0, 3>(acc, p.stages, nullptr, stage0_addr, stage_bytes, full, empty, 0, p.kb_total, it, cw, lane, a_tile,
                                             p.bw * 128, BN * 128);
            else
                consume_tile<T, BN, 0, 0>(acc, p.stages, nullptr, stage0_addr, stage_bytes, full, empty, 0, p.kb_total, it, cw, lane);
            const int n0 = nb * BN;
            const int m_local0 = cw * 64 + wq * 16;                    // first tile row of this warp
            const auto keep = [](int, float (&)[4]) {};
            const int n_valid = min(BN, p.C_out - n0);
            int r = mb;
            const int w0 = (r % p.tw) * p.bw; r /= p.tw;
            const int h0 = (r % p.th) * p.bh; r /= p.th;
            const int d0 = (r % p.td) * p.bd; const int n = r / p.td;
            store_tile<T, BN>(acc, stg, lane, n_valid, false, keep, [&](int rr) -> T * {
                const int m = m_local0 + rr;
                const int w = w0 + m % p.bw, h = h0 + (m / p.bw) % p.bh, d = d0 + m / (p.bw * p.bh);
                if (w >= p.W || h >= p.H || d >= p.D) return nullptr;
                return out + ((((int64_t)n * p.D + d) * p.H + h) * p.W + w) * p.C_out + n0;
            });
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------------
// Weight gradient.  A work item is (kd, 64-channel block of C_out, BN-channel tile of C_in, K slice) and computes the nine
// (kh, kw) taps of that kd; consumer warpgroup 0 holds taps kh x 3 + kw = 0..4, warpgroup 1 taps 5..8, each one m64 x BN fp32
// fragment per tap (5 x 24 registers at BN = 48).  A K block is one brick of bw x bh x 1 = 8 x 8 x 1 voxels.  Per K block the
// stage holds
//   X    one box of bw x bh rows, unshifted: the N operand of all nine taps (MN-major, C_in along the 128-byte row);
//   dY   three boxes of bw x (bh + 2) rows, one per kw, shifted by -(kw - 1, -1, kd - 1): the A operand (MN-major, C_out
//        along the row).  Tap kh reads its box from row (2 - kh) x bw on -- (2 - kh) x bw x 128 bytes, a multiple of 1024,
//        so the 128-byte swizzle phase is that of the box start.
// So the X brick is fetched once per K block for nine taps, and each dY voxel row once per kw instead of once per tap: per 64
// voxels and nine taps 8 KB of X and 3 x 10 KB of dY (for 64-channel boxes), against 27 x 8 KB with one tap per box.  The
// K slices are spread over the SMs; the partial products go to the zero-initialised fp32 dW with red.global.add (so the
// summation order of dW varies between runs).  Voxels of a brick past the volume are zero in X and may pair with in-volume
// dY rows, which is where a non-finite dY on the last row of a ragged volume reaches taps that read no input.
// ---------------------------------------------------------------------------------------------------------------------------
constexpr int kWgradTapsPerWg = 5;
// K block = one brick of 8 x 8 x 1 voxels: five 38 KB stages, and 128^3 / 64^3 / 32^3 volumes are whole numbers of bricks
// (a brick past the volume pairs zero-filled X with in-volume dY, see above).  16 x 8 bricks would leave room for only two
// 76 KB stages.
constexpr int kWgradBrickW = 8, kWgradBrickH = 8;

// consumer warpgroup of the weight gradient: over all work items of the CTA, acc[j] (64 C_out x BN C_in) = the product of tap
// kTap0 + j (kh x 3 + kw), j < kNTaps, over the item's K blocks, then red.global.add into dW.  Each warpgroup runs its own
// instantiation, so no wgmma sits under a branch on the warpgroup and no accumulator crosses one (ptxas would serialise the
// wgmma otherwise).  `it` counts K blocks over the CTA's life, as the producer does.
template <typename T, int BN, int kTap0, int kNTaps>
__device__ __forceinline__ void wgrad_consumer(const Conv3dP &p, unsigned stage0, int stage_bytes, int x_bytes, int dy_bytes, uint64_t *full,
                                               uint64_t *empty, uint8_t *stg, int wq, int lane) {
    float *const out = reinterpret_cast<float *>(p.out);
    const int kb_per = (p.kb_total + p.split_k - 1) / p.split_k;
    const int n_work = p.m_tiles * p.n_tiles * p.split_k;
    float acc[kNTaps][1][32];
    unsigned it = 0;
    for (int t = blockIdx.x; t < n_work; t += gridDim.x) {
        const int sp = t % p.split_k, nb = (t / p.split_k) % p.n_tiles, mb = t / (p.split_k * p.n_tiles);
        const int kd = mb % 3, co0 = (mb / 3) * 64;
        const int kb0 = sp * kb_per, kb1 = min(p.kb_total, kb0 + kb_per);
        int prev = -1;
        for (int kb = kb0; kb < kb1; ++kb, ++it) {
            const int s = it % p.stages;
            mbar_wait(&full[s], (it / p.stages) & 1);
            wg_fence();
            const unsigned sx = stage0 + (unsigned)(s * stage_bytes), sdy = sx + (unsigned)x_bytes;
#pragma unroll
            for (int k = 0; k < kWgradBrickW * kWgradBrickH / kMmaK; ++k) {
                const uint64_t db = make_desc(sx + k * (kMmaK * 128), 8192, 1024);
                const unsigned acc_on = (kb > kb0 || k > 0) ? 1u : 0u;
#pragma unroll
                for (int j = 0; j < kNTaps; ++j) {
                    const int tap = kTap0 + j, kh = tap / 3, kw = tap % 3;
                    const uint64_t da = make_desc(sdy + (unsigned)(kw * dy_bytes + (2 - kh) * kWgradBrickW * 128 + k * (kMmaK * 128)), 8192, 1024);
                    wgmma_k16<T, BN, 1, 1>(acc[j][0], da, db, acc_on);
                }
            }
            wg_commit();
            if (prev >= 0) {                                  // the group of the previous K block has completed: release its stage
                wg_wait<1>();
                if (lane == 0) mbar_arrive(&empty[prev]);
            }
            prev = s;
        }
        wg_wait<0>();
        if (lane == 0) mbar_arrive(&empty[prev]);

        const int n0 = nb * BN, n_valid = min(BN, p.C_in - n0), co_w = co0 + wq * 16;
        const auto keep = [](int, float (&)[4]) {};
#pragma unroll
        for (int j = 0; j < kNTaps; ++j) {
            store_tile<float, BN>(acc[j], stg, lane, n_valid, true, keep, [&](int rr) -> float * {
                const int co = co_w + rr;
                if (co >= p.C_out) return nullptr;
                return out + ((int64_t)co * kTaps + kd * 9 + kTap0 + j) * p.C_in + n0;
            });
        }
    }
}

template <typename T, int BN>
__global__ void __launch_bounds__(kThreads, 1) conv3d_wgrad_kernel(const __grid_constant__ CUtensorMap tmDy,
                                                                   const __grid_constant__ CUtensorMap tmX, const Conv3dP p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    const int x_bytes = p.bw * p.bh * 128, dy_bytes = p.bw * (p.bh + 2) * 128;
    const int stage_bytes = x_bytes + 3 * dy_bytes;                    // all multiples of 1024
    uint8_t *stage0 = smem;
    uint8_t *staging = smem + (size_t)p.stages * stage_bytes;
    uint64_t *bars = reinterpret_cast<uint64_t *>(staging + kStagingBytes);
    uint64_t *full = bars, *empty = bars + kMaxStages;

    if (threadIdx.x == 0) {
        for (int s = 0; s < p.stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kConsumerWarps); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmDy) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmX) : "memory");
    }
    __syncthreads();

    const int kb_per = (p.kb_total + p.split_k - 1) / p.split_k;
    const int n_work = p.m_tiles * p.n_tiles * p.split_k;             // m_tiles = 3 kd x cob

    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (threadIdx.x == 0) {
            unsigned it = 0;
            for (int t = blockIdx.x; t < n_work; t += gridDim.x) {
                const int sp = t % p.split_k, nb = (t / p.split_k) % p.n_tiles, mb = t / (p.split_k * p.n_tiles);
                const int kd = mb % 3, co0 = (mb / 3) * 64;
                const int kb0 = sp * kb_per, kb1 = min(p.kb_total, kb0 + kb_per);
                for (int kb = kb0; kb < kb1; ++kb, ++it) {             // K block kb = one brick
                    int r = kb;
                    const int w0 = (r % p.tw) * p.bw; r /= p.tw;
                    const int h0 = (r % p.th) * p.bh; r /= p.th;
                    const int d0 = r % p.D, n = r / p.D;
                    const int s = it % p.stages;
                    mbar_wait(&empty[s], ((it / p.stages) & 1) ^ 1);
                    uint8_t *sx = stage0 + (size_t)s * stage_bytes;
                    mbar_expect_tx(&full[s], (unsigned)stage_bytes);
                    tma_load_5d(sx, &tmX, nb * BN, w0, h0, d0, n, &full[s]);
#pragma unroll
                    for (int kw = 0; kw < 3; ++kw)
                        tma_load_5d(sx + x_bytes + kw * dy_bytes, &tmDy, co0, w0 - kw + 1, h0 - 1, d0 - kd + 1, n, &full[s]);
                }
            }
        }
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
        const int cw = (warp >> 2) - 1, wq = warp & 3;
        uint8_t *stg = staging + (size_t)(warp - 4) * (16 * kPitch);
        const unsigned stage0_addr = smem_u32(stage0);
        if (cw == 0)
            wgrad_consumer<T, BN, 0, kWgradTapsPerWg>(p, stage0_addr, stage_bytes, x_bytes, dy_bytes, full, empty, stg, wq, lane);
        else
            wgrad_consumer<T, BN, kWgradTapsPerWg, 9 - kWgradTapsPerWg>(p, stage0_addr, stage_bytes, x_bytes, dy_bytes, full, empty, stg, wq, lane);
    }
}

int pow2_at_least(int v) {
    int p = 1;
    while (p < v) p <<= 1;
    return p;
}

// activation tensor map: dims (C, W, H, D, batch), box (64 channels, bw x box_h x bd voxels)
cudaError_t act_map(CUtensorMap *m, const Conv3dP &p, const void *base, int C, int box_h) {
    const uint64_t dims[5] = {(uint64_t)C, (uint64_t)p.W, (uint64_t)p.H, (uint64_t)p.D, (uint64_t)p.batch};
    const uint64_t es = 2;
    const uint64_t strides[4] = {es * C, es * C * p.W, es * C * p.W * p.H, es * C * p.W * p.H * p.D};
    const uint32_t box[5] = {64, (uint32_t)p.bw, (uint32_t)box_h, (uint32_t)p.bd, 1};
    return encode_tiled(m, base, p.dtype, 5, dims, strides, box);
}

// the N tile of the weight gradient: C_in in the fewest 64-wide tiles, each as narrow as a multiple of 16 allows
// (96 -> 2 x 48, 40 -> 48, 192 -> 3 x 64)
int wgrad_pick_bn(int C_in) {
    const int tiles = (C_in + 63) / 64, per = (C_in + tiles - 1) / tiles;
    return (per + 15) / 16 * 16;
}

}  // namespace

cudaError_t conv3d_tc_launch(Conv3dP p, const void *x, const void *b, cudaStream_t st, const char **where) {
    const char *dummy;
    if (!where) where = &dummy;
    *where = "setup";
    static int sms = 0, max_smem = 0;
    if (!sms) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    }
    const size_t fixed = 1024 + kStagingBytes + 2 * kMaxStages * 8;
    size_t stage_bytes;
    if (!p.wgrad) {
        // brick of 128 output voxels per tile: 16 x 8 x 1 (8 x 16 x 1 for W <= 8) when folded, else powers of two, w first; a
        // brick that reaches past the volume is zero-filled there, so the box always has exactly 128 rows
        p.BN = gemm_pick_bn(p.C_out);
        const bool fold = conv3d_folds(p.BN);
        p.bw = fold ? std::min(16, std::max(8, pow2_at_least(p.W))) : std::min(kBM, pow2_at_least(p.W));
        p.bh = fold ? kBM / p.bw : std::min(kBM / p.bw, pow2_at_least(p.H));
        p.bd = kBM / (p.bw * p.bh);
        p.tw = (p.W + p.bw - 1) / p.bw;
        p.th = (p.H + p.bh - 1) / p.bh;
        p.td = (p.D + p.bd - 1) / p.bd;
        p.cb = (p.C_in + kBK - 1) / kBK;
        p.m_tiles = p.batch * p.tw * p.th * p.td;
        p.n_tiles = (p.C_out + p.BN - 1) / p.BN;
        p.kb_total = (fold ? 9 : kTaps) * p.cb;
        p.split_k = 1;
        const size_t b_tile = (size_t)(fold ? 3 : 1) * p.BN * 128;
        stage_bytes = (size_t)(fold ? kFoldABytes : kBM * 128) + ((b_tile + 1023) & ~(size_t)1023);
    } else {
        // K block = one brick of bw x bh x 1 voxels (see conv3d_wgrad_kernel)
        p.BN = wgrad_pick_bn(p.C_in);
        p.bw = kWgradBrickW;
        p.bh = kWgradBrickH;
        p.bd = 1;
        p.tw = (p.W + p.bw - 1) / p.bw;
        p.th = (p.H + p.bh - 1) / p.bh;
        p.td = p.D;
        p.cob = (p.C_out + 63) / 64;
        p.m_tiles = 3 * p.cob;
        p.n_tiles = (p.C_in + p.BN - 1) / p.BN;
        p.kb_total = p.batch * p.tw * p.th * p.D;
        // K split: the fewest bricks per CTA, counting each work item's pipeline fill and epilogue as kItemCost bricks; every
        // slice holds at least kMinSlice bricks and none is empty
        const int mn = p.m_tiles * p.n_tiles, bricks = p.kb_total;
        constexpr int kItemCost = 8, kMinSlice = 16;
        long best = -1;
        for (int split = 1; split <= std::max(1, std::min(bricks / kMinSlice, 4 * sms)); ++split) {
            const long per = (bricks + split - 1) / split, rounds = ((long)mn * split + sms - 1) / sms;
            const long cost = rounds * (per + kItemCost);
            if (best < 0 || cost < best) { best = cost; p.split_k = split; }
        }
        const int kb_per = (bricks + p.split_k - 1) / p.split_k;
        p.split_k = (bricks + kb_per - 1) / kb_per;
        stage_bytes = (size_t)p.bw * (p.bh + 3 * (p.bh + 2)) * 128;
    }
    int stages = (int)(((size_t)max_smem - fixed) / stage_bytes);
    if (stages > kMaxStages) stages = kMaxStages;
    if (stages < 2) return cudaErrorInvalidConfiguration;
    p.stages = stages;
    const size_t smem = fixed + (size_t)stages * stage_bytes;

    cudaError_t e;
    *where = "cudaPointerGetAttributes(X)";
    if ((e = bind_device_of(x)) != cudaSuccess) return e;
    CUtensorMap tmA, tmB;
    if (!p.wgrad) {
        *where = "tensor map of X (cuTensorMapEncodeTiled)";
        if ((e = act_map(&tmA, p, x, p.C_in, conv3d_folds(p.BN) ? p.bh + 2 : p.bh)) != cudaSuccess) return e;
        *where = "tensor map of the weight (cuTensorMapEncodeTiled)";
        const uint64_t dims[3] = {(uint64_t)p.C_in, (uint64_t)kTaps, (uint64_t)p.C_out};
        const uint64_t strides[2] = {2ull * p.C_in, 2ull * p.C_in * kTaps};
        const uint32_t box[3] = {64, 1, (uint32_t)p.BN};
        if ((e = encode_tiled(&tmB, b, p.dtype, 3, dims, strides, box)) != cudaSuccess) return e;
    } else {
        *where = "tensor map of dY (cuTensorMapEncodeTiled)";
        if ((e = act_map(&tmA, p, b, p.C_out, p.bh + 2)) != cudaSuccess) return e;
        *where = "tensor map of X (cuTensorMapEncodeTiled)";
        if ((e = act_map(&tmB, p, x, p.C_in, p.bh)) != cudaSuccess) return e;
    }

    const long n_work = (long)p.m_tiles * p.n_tiles * p.split_k;
    const int grid = (int)(n_work < (long)sms ? n_work : (long)sms);
#define SMB_CONV_LAUNCH(KERNEL)                                                                                             \
    do {                                                                                                                    \
        static bool set = false;                                                                                            \
        *where = "cudaFuncSetAttribute";                                                                                    \
        if (!set) {                                                                                                         \
            e = cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)max_smem);                   \
            if (e != cudaSuccess) return e;                                                                                 \
            set = true;                                                                                                     \
        }                                                                                                                   \
        *where = "kernel launch";                                                                                           \
        KERNEL<<<grid, kThreads, smem, st>>>(tmA, tmB, p);                                                                  \
    } while (0)
#define SMB_CONV_TYPES(kBN)                                                                                                 \
    do {                                                                                                                    \
        if (p.dtype == 1) SMB_CONV_LAUNCH((conv3d_tc_kernel<__half, kBN>));                                                  \
        else SMB_CONV_LAUNCH((conv3d_tc_kernel<__nv_bfloat16, kBN>));                                                        \
    } while (0)
#define SMB_WGRAD_TYPES(kBN)                                                                                                \
    do {                                                                                                                    \
        if (p.dtype == 1) SMB_CONV_LAUNCH((conv3d_wgrad_kernel<__half, kBN>));                                               \
        else SMB_CONV_LAUNCH((conv3d_wgrad_kernel<__nv_bfloat16, kBN>));                                                     \
    } while (0)
    if (p.wgrad) {
        switch (p.BN) {
            case 16: SMB_WGRAD_TYPES(16); break;
            case 32: SMB_WGRAD_TYPES(32); break;
            case 48: SMB_WGRAD_TYPES(48); break;
            default: SMB_WGRAD_TYPES(64); break;
        }
    } else {
        switch (p.BN) {
            case 16: SMB_CONV_TYPES(16); break;
            case 32: SMB_CONV_TYPES(32); break;
            case 48: SMB_CONV_TYPES(48); break;
            case 64: SMB_CONV_TYPES(64); break;
            case 96: SMB_CONV_TYPES(96); break;
            case 128: SMB_CONV_TYPES(128); break;
            case 192: SMB_CONV_TYPES(192); break;
            default: SMB_CONV_TYPES(256); break;
        }
    }
#undef SMB_WGRAD_TYPES
#undef SMB_CONV_TYPES
#undef SMB_CONV_LAUNCH
    count_launch();
    return cudaGetLastError();
}

}  // namespace smb
