// Implicit-GEMM 3x3x3 convolution (stride 1, padding 1, no bias) on channels-last activations, sm_90a: TMA -> shared memory
// -> wgmma.mma_async -> staged epilogue, on the pipeline of wgmma_pipe.cuh (the one the GEMM of gemm_tc.cu runs).
//
//   forward   Y[t, co] = sum_tap sum_ci X[t + off(tap), ci] . Wt[co, tap, ci]          M = tokens, N = C_out, K = 27 x C_in
//             The data gradient is the same product on dY with the weight flipped in all three axes and C_in / C_out
//             swapped (the caller re-lays the 27 C_in C_out weights).
//   wgrad     dW[co, tap, ci] += sum_t dY[t - off(tap), co] . X[t, ci]                  M = (tap, co), N = C_in, K = tokens
//
// X and dY are read through 5-D tensor maps (C, W, H, D, batch).  The A operand of one tap is a brick of voxels shifted by
// off(tap) = (kw - 1, kh - 1, kd - 1); the TMA unit zero-fills whatever part of the box lies outside the volume, which is the
// padding.  Batch stays its own axis, so a shift past d = 0 reads zeros and never the previous sample.  No im2col is stored.
//
// Forward tile: 128 output voxels = one brick x BN output channels.  With BN <= 128 the brick is 16 x 8 x 1 (8 x 16 x 1 for
// W <= 8) and one K block covers the three kh taps of a (kd, kw) pair from one box of bh + 2 rows (see kFoldABytes); wider
// tiles take a brick of powers of two, w first, and one tap per K block.  Input channels come in boxes of 64 (C = 48 or 96
// leaves the last box a quarter or half zero-filled: 25 % of the MMA work of those passes is spent on zeros).
// Weight-gradient tile: rows 0..63 are one (tap, 64-channel block of C_out) pair, rows 64..127 the next one, each loaded as an
// MN-major box of dY shifted by -off(tap); the N operand is X, unshifted, MN-major.  K = bricks of 64 voxels, split over the
// CTAs; the partial products go to the fp32 dW with red.global.add (so the summation order of dW varies between runs).
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
constexpr bool conv3d_folds(bool wgrad, int BN) { return !wgrad && BN <= 128; }

template <typename TIn, typename TOut, int BN, bool kWgrad>
__global__ void __launch_bounds__(kThreads, 1) conv3d_tc_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                const __grid_constant__ CUtensorMap tmB, const Conv3dP p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    constexpr int kChunks = (BN + 63) / 64;
    constexpr bool kFold = conv3d_folds(kWgrad, BN);
    constexpr int a_tile = kFold ? kFoldABytes : kBM * 128;
    constexpr int b_tile = kWgrad ? kChunks * 8192 : (kFold ? 3 : 1) * BN * 128;
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

    const int kb_per = (p.kb_total + p.split_k - 1) / p.split_k;
    const int n_work = p.m_tiles * p.n_tiles * p.split_k;

    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (threadIdx.x == 0) {
            unsigned it = 0;
            for (int t = blockIdx.x; t < n_work; t += gridDim.x) {
                const int sp = t % p.split_k, nb = (t / p.split_k) % p.n_tiles, mb = t / (p.split_k * p.n_tiles);
                const int kb0 = sp * kb_per, kb1 = min(p.kb_total, kb0 + kb_per);
                int n = 0, d0 = 0, h0 = 0, w0 = 0;
                if (!kWgrad) {                                         // the output brick of this tile
                    int r = mb;
                    w0 = (r % p.tw) * p.bw; r /= p.tw;
                    h0 = (r % p.th) * p.bh; r /= p.th;
                    d0 = (r % p.td) * p.bd; n = r / p.td;
                }
                for (int kb = kb0; kb < kb1; ++kb, ++it) {
                    const int s = it % p.stages;
                    mbar_wait(&empty[s], ((it / p.stages) & 1) ^ 1);
                    uint8_t *sa = stage0 + (size_t)s * stage_bytes, *sb = sa + a_tile;
                    mbar_expect_tx(&full[s], tx_bytes);
                    if (kFold) {                                       // K block = (kd, kw, channel box); kh = 0, 1, 2 inside
                        const int kd = kb / (3 * p.cb), kw = (kb / p.cb) % 3, c = (kb % p.cb) * kBK;
                        tma_load_5d(sa, &tmA, c, w0 + kw - 1, h0 - 1, d0 + kd - 1, n, &full[s]);
#pragma unroll
                        for (int kh = 0; kh < 3; ++kh) tma_load_3d(sb + kh * BN * 128, &tmB, c, kd * 9 + kh * 3 + kw, nb * BN, &full[s]);
                    } else if (!kWgrad) {
                        const int tap = kb / p.cb, c = (kb % p.cb) * kBK;
                        const int kd = tap / 9, kh = (tap / 3) % 3, kw = tap % 3;
                        tma_load_5d(sa, &tmA, c, w0 + kw - 1, h0 + kh - 1, d0 + kd - 1, n, &full[s]);
                        tma_load_3d(sb, &tmB, c, tap, nb * BN, &full[s]);
                    } else {                                           // K block kb = one brick of 64 voxels
                        int r = kb;
                        const int bw0 = (r % p.tw) * p.bw; r /= p.tw;
                        const int bh0 = (r % p.th) * p.bh; r /= p.th;
                        const int bd0 = (r % p.td) * p.bd; const int bn = r / p.td;
#pragma unroll
                        for (int half = 0; half < 2; ++half) {
                            const int hm = 2 * mb + half;
                            const int tap = min(hm / p.cob, kTaps - 1);        // a pad row pair past the last tap: loaded, not stored
                            const int kd = tap / 9, kh = (tap / 3) % 3, kw = tap % 3;
                            tma_load_5d(sa + half * 8192, &tmA, (hm % p.cob) * 64, bw0 - kw + 1, bh0 - kh + 1, bd0 - kd + 1, bn, &full[s]);
                        }
#pragma unroll
                        for (int c = 0; c < kChunks; ++c) tma_load_5d(sb + c * 8192, &tmB, nb * BN + c * 64, bw0, bh0, bd0, bn, &full[s]);
                    }
                }
            }
        }
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
        const int cw = (warp >> 2) - 1, wq = warp & 3;
        TOut *const out = reinterpret_cast<TOut *>(p.out);
        uint8_t *stg = staging + (size_t)(warp - 4) * (16 * kPitch);
        const unsigned stage0_addr = smem_u32(stage0);
        float acc[kChunks][32];
        unsigned it = 0;
        for (int t = blockIdx.x; t < n_work; t += gridDim.x) {
            const int sp = t % p.split_k, nb = (t / p.split_k) % p.n_tiles, mb = t / (p.split_k * p.n_tiles);
            const int kb0 = sp * kb_per, kb1 = min(p.kb_total, kb0 + kb_per);
            if constexpr (kFold)       // tap kh reads the box bw rows (= one h-row, a multiple of 1024 bytes) further on
                consume_tile<TIn, BN, 0, 0, 3>(acc, p.stages, nullptr, stage0_addr, stage_bytes, full, empty, kb0, kb1, it, cw, lane, a_tile,
                                               p.bw * 128, BN * 128);
            else
                consume_tile<TIn, BN, kWgrad ? 1 : 0, kWgrad ? 1 : 0>(acc, p.stages, nullptr, stage0_addr, stage_bytes, full, empty, kb0, kb1,
                                                                       it, cw, lane);
            const int n0 = nb * BN;
            const int m_local0 = cw * 64 + wq * 16;                    // first tile row of this warp
            const auto keep = [](int, float (&)[4]) {};
            if (!kWgrad) {
                const int n_valid = min(BN, p.C_out - n0);
                int r = mb;
                const int w0 = (r % p.tw) * p.bw; r /= p.tw;
                const int h0 = (r % p.th) * p.bh; r /= p.th;
                const int d0 = (r % p.td) * p.bd; const int n = r / p.td;
                store_tile<TOut, BN>(acc, stg, lane, n_valid, false, keep, [&](int rr) -> TOut * {
                    const int m = m_local0 + rr;
                    const int w = w0 + m % p.bw, h = h0 + (m / p.bw) % p.bh, d = d0 + m / (p.bw * p.bh);
                    if (w >= p.W || h >= p.H || d >= p.D) return nullptr;
                    return out + ((((int64_t)n * p.D + d) * p.H + h) * p.W + w) * p.C_out + n0;
                });
            } else {
                const int n_valid = min(BN, p.C_in - n0);
                const int hm = 2 * mb + cw, tap = hm / p.cob, co0 = (hm % p.cob) * 64 + wq * 16;
                store_tile<TOut, BN>(acc, stg, lane, n_valid, true, keep, [&](int rr) -> TOut * {
                    const int co = co0 + rr;
                    if (tap >= kTaps || co >= p.C_out) return nullptr;
                    return out + ((int64_t)co * kTaps + tap) * p.C_in + n0;
                });
            }
        }
    }
}

int pow2_at_least(int v) {
    int p = 1;
    while (p < v) p <<= 1;
    return p;
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
    // brick of voxels per tile (forward, 128 rows) or per K block (wgrad, 64 rows): powers of two, w first; a brick that
    // reaches past the volume is zero-filled there, so the box always has exactly `rows` rows
    p.BN = gemm_pick_bn(p.wgrad ? p.C_in : p.C_out);
    const int BN = p.BN;
    const bool fold = conv3d_folds(p.wgrad != 0, BN);
    const int rows = p.wgrad ? 64 : kBM;
    p.bw = fold ? std::min(16, std::max(8, pow2_at_least(p.W))) : std::min(rows, pow2_at_least(p.W));
    p.bh = fold ? rows / p.bw : std::min(rows / p.bw, pow2_at_least(p.H));
    p.bd = rows / (p.bw * p.bh);
    p.tw = (p.W + p.bw - 1) / p.bw;
    p.th = (p.H + p.bh - 1) / p.bh;
    p.td = (p.D + p.bd - 1) / p.bd;
    const int bricks = p.batch * p.tw * p.th * p.td;
    p.cb = (p.C_in + kBK - 1) / kBK;
    p.cob = (p.C_out + 63) / 64;
    if (!p.wgrad) {
        p.m_tiles = bricks;
        p.n_tiles = (p.C_out + BN - 1) / BN;
        p.kb_total = (fold ? 9 : kTaps) * p.cb;
        p.split_k = 1;
    } else {
        p.m_tiles = (kTaps * p.cob + 1) / 2;
        p.n_tiles = (p.C_in + BN - 1) / BN;
        p.kb_total = bricks;
        // about two work items per SM, each at least 32 bricks long; no slice may be empty
        const int mn = p.m_tiles * p.n_tiles;
        int split = std::max(1, std::min(bricks / 32, (2 * sms + mn - 1) / mn));
        const int kb_per = (bricks + split - 1) / split;
        p.split_k = (bricks + kb_per - 1) / kb_per;
    }
    const size_t b_tile = p.wgrad ? (size_t)((BN + 63) / 64) * 8192 : (size_t)(fold ? 3 : 1) * BN * 128;
    const size_t stage_bytes = (size_t)(fold ? kFoldABytes : kBM * 128) + ((b_tile + 1023) & ~(size_t)1023);
    const size_t fixed = 1024 + kStagingBytes + 2 * kMaxStages * 8;
    int stages = (int)(((size_t)max_smem - fixed) / stage_bytes);
    if (stages > kMaxStages) stages = kMaxStages;
    if (stages < 2) return cudaErrorInvalidConfiguration;
    p.stages = stages;
    const size_t smem = fixed + (size_t)stages * stage_bytes;

    cudaError_t e;
    *where = "cudaPointerGetAttributes(X)";
    if ((e = bind_device_of(x)) != cudaSuccess) return e;
    // activation maps: dims (C, W, H, D, batch), box (64 channels, brick)
    const auto act_map = [&](CUtensorMap *m, const void *base, int C, int box_h) {
        const uint64_t dims[5] = {(uint64_t)C, (uint64_t)p.W, (uint64_t)p.H, (uint64_t)p.D, (uint64_t)p.batch};
        const uint64_t es = 2;
        const uint64_t strides[4] = {es * C, es * C * p.W, es * C * p.W * p.H, es * C * p.W * p.H * p.D};
        const uint32_t box[5] = {64, (uint32_t)p.bw, (uint32_t)box_h, (uint32_t)p.bd, 1};
        return encode_tiled(m, base, p.dtype, 5, dims, strides, box);
    };
    CUtensorMap tmA, tmB;
    if (!p.wgrad) {
        *where = "tensor map of X (cuTensorMapEncodeTiled)";
        if ((e = act_map(&tmA, x, p.C_in, fold ? p.bh + 2 : p.bh)) != cudaSuccess) return e;
        *where = "tensor map of the weight (cuTensorMapEncodeTiled)";
        const uint64_t dims[3] = {(uint64_t)p.C_in, (uint64_t)kTaps, (uint64_t)p.C_out};
        const uint64_t strides[2] = {2ull * p.C_in, 2ull * p.C_in * kTaps};
        const uint32_t box[3] = {64, 1, (uint32_t)BN};
        if ((e = encode_tiled(&tmB, b, p.dtype, 3, dims, strides, box)) != cudaSuccess) return e;
    } else {
        *where = "tensor map of dY (cuTensorMapEncodeTiled)";
        if ((e = act_map(&tmA, b, p.C_out, p.bh)) != cudaSuccess) return e;
        *where = "tensor map of X (cuTensorMapEncodeTiled)";
        if ((e = act_map(&tmB, x, p.C_in, p.bh)) != cudaSuccess) return e;
    }

    const long n_work = (long)p.m_tiles * p.n_tiles * p.split_k;
    const int grid = (int)(n_work < (long)sms ? n_work : (long)sms);
#define SMB_CONV_LAUNCH(TIn, TOut, kBN, kW)                                                                                 \
    do {                                                                                                                    \
        static bool set = false;                                                                                            \
        *where = "cudaFuncSetAttribute";                                                                                    \
        if (!set) {                                                                                                         \
            e = cudaFuncSetAttribute(conv3d_tc_kernel<TIn, TOut, kBN, kW>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)max_smem); \
            if (e != cudaSuccess) return e;                                                                                 \
            set = true;                                                                                                     \
        }                                                                                                                   \
        *where = "kernel launch";                                                                                           \
        conv3d_tc_kernel<TIn, TOut, kBN, kW><<<grid, kThreads, smem, st>>>(tmA, tmB, p);                                    \
    } while (0)
#define SMB_CONV_TYPES(kBN)                                                                                                 \
    do {                                                                                                                    \
        if (p.dtype == 1) {                                                                                                 \
            if (p.wgrad) SMB_CONV_LAUNCH(__half, float, kBN, true);                                                         \
            else SMB_CONV_LAUNCH(__half, __half, kBN, false);                                                               \
        } else {                                                                                                            \
            if (p.wgrad) SMB_CONV_LAUNCH(__nv_bfloat16, float, kBN, true);                                                  \
            else SMB_CONV_LAUNCH(__nv_bfloat16, __nv_bfloat16, kBN, false);                                                 \
        }                                                                                                                   \
    } while (0)
    switch (BN) {
        case 16: SMB_CONV_TYPES(16); break;
        case 32: SMB_CONV_TYPES(32); break;
        case 48: SMB_CONV_TYPES(48); break;
        case 64: SMB_CONV_TYPES(64); break;
        case 96: SMB_CONV_TYPES(96); break;
        case 128: SMB_CONV_TYPES(128); break;
        case 192: SMB_CONV_TYPES(192); break;
        default: SMB_CONV_TYPES(256); break;
    }
#undef SMB_CONV_TYPES
#undef SMB_CONV_LAUNCH
    count_launch();
    return cudaGetLastError();
}

}  // namespace smb
