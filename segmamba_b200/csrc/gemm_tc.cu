// Tensor-core GEMM for the pointwise contractions of the SegMamba hot path (sm_90a: TMA -> shared memory -> wgmma.mma_async with
// the accumulator in registers -> staged, coalesced epilogue).
//
//     D[M, N] (+)= epilogue( A[M, K] . B[N, K]^T )          16-bit operands, fp32 accumulation
//
// replaces the library calls behind   Mamba.in_proj / out_proj (mamba_simple.py:204-208,264),  MlpChannel.fc1 / fc2
// (segmamba.py:81-89),  GSC.proj3 / proj4 (segmamba.py:103-107,121-128),  UnetResBlock.conv3 (dynunet_block.py:66-69,105-109)
// -- 1x1x1 convolutions on channels-last activations are plain (tokens, C_in) x (C_out, C_in)^T products -- and their two
// backward products (data gradient: the same kernel on the transposed weight view; weight gradient: contraction over the token
// axis, both operands MN-major, split over CTAs along K with fp32 atomics).
//
// Structure (one persistent CTA per SM, 384 threads = three warpgroups, warp-specialised):
//   warpgroup 0     TMA producer (one thread; the warpgroup gives its registers up with setmaxnreg): cp.async.bulk.tensor 2-D
//                   boxes of A (128 x 64) and B (BN x 64) per 64-wide K block into a ring of shared-memory stages
//                   (CU_TENSOR_MAP_SWIZZLE_128B), completion on the stage's `full` mbarrier
//   warpgroups 1,2  consumers: each owns 64 rows of the 128 x BN tile.  Per K block four wgmma.mma_async k16 steps per 64-column
//                   chunk of the tile (m64n64k16, or n16 / n32 / n48 for the last chunk), one commit group per K block with one
//                   group in flight; a stage is released to the producer (`empty` mbarrier, one arrival per warp) when the
//                   group that read it has completed.  Epilogue by the same warps: bias / GELU -> convert -> warp-private
//                   padded staging tile in shared memory -> coalesced 16-byte global stores (or fp32 atomics for split-K),
//                   while the producer already fills the ring for the next tile.
// BN is a template parameter (the wgmma shape is part of the instruction): 16, 32, 48, 64, 96, 128, 192 or 256.
// Either operand may be K-major (rows = M or N index, K contiguous) or MN-major (rows = K index, M or N contiguous); the
// shared-memory matrix descriptors and the instruction's transpose bits carry the difference, the TMA boxes stay (64 elements =
// 128 bytes) x rows.  Out-of-range rows / columns of a box are zero-filled by the TMA unit, so ragged M, N and K need no separate
// path on the load side; the store side bounds every access.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <cstring>

#include "gemm_internal.h"

namespace smb {
void count_launch();

namespace {

constexpr int kBM = 128;            // two consumer warpgroups x wgmma M = 64
constexpr int kBK = 64;             // K block: 64 sixteen-bit elements = one 128-byte swizzle row
constexpr int kMmaK = 16;
constexpr int kThreads = 384;       // warpgroup 0 TMA, warpgroups 1..2 wgmma + epilogue
constexpr int kConsumerWarps = 8;
constexpr int kMaxStages = 6;
constexpr int kPitch = 144;         // staging row pitch: 128 + 16 bytes -> conflict-free 16-byte reads
constexpr int kStagingBytes = kConsumerWarps * 16 * kPitch;

__device__ __forceinline__ unsigned smem_u32(const void *p) { return static_cast<unsigned>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// bounded wait: a phase that does not complete within ~2^24 polls means a mis-armed barrier or a faulted copy; trap so the
// launch fails visibly instead of holding the GPU
__device__ __forceinline__ void mbar_wait(uint64_t *bar, unsigned parity) {
    const unsigned addr = smem_u32(bar);
    for (unsigned spins = 0;; ++spins) {
        unsigned done;
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}\n"
            : "=r"(done)
            : "r"(addr), "r"(parity)
            : "memory");
        if (done) return;
        if (spins > (1u << 24)) __trap();
    }
}
// optional profiling (GemmP::prof != nullptr): cycles a role spends inside a barrier wait, summed over the grid
__device__ __forceinline__ void mbar_wait_prof(uint64_t *bar, unsigned parity, unsigned long long *acc) {
    if (!acc) { mbar_wait(bar, parity); return; }
    const long long t0 = clock64();
    mbar_wait(bar, parity);
    atomicAdd(acc, (unsigned long long)(clock64() - t0));
}
__device__ __forceinline__ void tma_load_2d(void *smem, const CUtensorMap *m, int c0, int c1, uint64_t *bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
                     smem_u32(smem)),
                 "l"(m), "r"(c0), "r"(c1), "r"(smem_u32(bar))
                 : "memory");
}
template <typename T> constexpr bool kIsBf16 = false;
template <> constexpr bool kIsBf16<__nv_bfloat16> = true;

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int kPending> __device__ __forceinline__ void wg_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(kPending) : "memory");
}

// D (64 x N fp32, in registers) = A . B (+ D when scale_d != 0), both operands through shared-memory descriptors; TA / TB = 1
// marks an MN-major operand.  The accumulator fragment of a thread: d[4 j + {0, 1}] = row (lane / 4) of its warp's 16 rows,
// columns 8 j + 2 (lane % 4) + {0, 1}; d[4 j + {2, 3}] = row (lane / 4) + 8, same columns.
#define SMB_ACC8(o) "+f"(d[o]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), "+f"(d[o + 6]), "+f"(d[o + 7])
#define SMB_D8 "%0, %1, %2, %3, %4, %5, %6, %7"
#define SMB_D16 SMB_D8 ", %8, %9, %10, %11, %12, %13, %14, %15"
#define SMB_D24 SMB_D16 ", %16, %17, %18, %19, %20, %21, %22, %23"
#define SMB_D32 SMB_D24 ", %24, %25, %26, %27, %28, %29, %30, %31"
#define SMB_WGMMA(SHAPE, TYPE, DREGS, OA, OB, OS, OTA, OTB, ...)                                                             \
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %" OS ", 0;\n"                                                             \
                 "wgmma.mma_async.sync.aligned." SHAPE ".f32." TYPE "." TYPE " {" DREGS "}, %" OA ", %" OB ", p, 1, 1, %" OTA \
                 ", %" OTB ";\n}\n"                                                                                           \
                 : __VA_ARGS__                                                                                                \
                 : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB))
#define SMB_WGMMA_N(TYPE)                                                                                                     \
    if constexpr (N == 64) SMB_WGMMA("m64n64k16", TYPE, SMB_D32, "32", "33", "34", "35", "36", SMB_ACC8(0), SMB_ACC8(8), SMB_ACC8(16), SMB_ACC8(24)); \
    else if constexpr (N == 48) SMB_WGMMA("m64n48k16", TYPE, SMB_D24, "24", "25", "26", "27", "28", SMB_ACC8(0), SMB_ACC8(8), SMB_ACC8(16));        \
    else if constexpr (N == 32) SMB_WGMMA("m64n32k16", TYPE, SMB_D16, "16", "17", "18", "19", "20", SMB_ACC8(0), SMB_ACC8(8));                     \
    else SMB_WGMMA("m64n16k16", TYPE, SMB_D8, "8", "9", "10", "11", "12", SMB_ACC8(0))
template <typename TIn, int N, int TA, int TB>
__device__ __forceinline__ void wgmma_k16(float (&d)[32], uint64_t da, uint64_t db, unsigned scale_d) {
    static_assert(N == 16 || N == 32 || N == 48 || N == 64, "chunk width");
    if constexpr (kIsBf16<TIn>) { SMB_WGMMA_N("bf16"); } else { SMB_WGMMA_N("f16"); }
}
#undef SMB_WGMMA_N
#undef SMB_WGMMA
#undef SMB_D32
#undef SMB_D24
#undef SMB_D16
#undef SMB_D8
#undef SMB_ACC8
__device__ __forceinline__ void red_add_v4f(float *a, float x, float y, float z, float w) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(a), "f"(x), "f"(y), "f"(z), "f"(w) : "memory");
}

// shared-memory matrix descriptor, 128-byte swizzle (start >> 4 at [0,14), leading byte offset >> 4 at [16,30), stride byte
// offset >> 4 at [32,46), swizzle mode 128B = 1 at [62,64)).
//   K-major  tile = rows x 128 B : 8-row groups are 1024 B apart (SBO); the leading offset is unused inside one swizzle row.
//   MN-major tile = 64 K-rows x 128 B per 64 MN elements: 8-K-row groups 1024 B apart (SBO), next 64 MN elements one tile on (LBO).
__device__ __forceinline__ uint64_t make_desc(unsigned smem_addr, unsigned lbo_bytes, unsigned sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

struct alignas(16) F4 { float x, y, z, w; };

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }

template <typename T> __device__ __forceinline__ unsigned pack2(float a, float b);
template <> __device__ __forceinline__ unsigned pack2<__nv_bfloat16>(float a, float b) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<unsigned *>(&h);
}
template <> __device__ __forceinline__ unsigned pack2<__half>(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<unsigned *>(&h);
}

template <typename T> __device__ __forceinline__ unsigned sum2(unsigned a, unsigned b);
template <> __device__ __forceinline__ unsigned sum2<__nv_bfloat16>(unsigned a, unsigned b) {
    const __nv_bfloat162 x = *reinterpret_cast<const __nv_bfloat162 *>(&a), y = *reinterpret_cast<const __nv_bfloat162 *>(&b);
    return pack2<__nv_bfloat16>(__low2float(x) + __low2float(y), __high2float(x) + __high2float(y));
}
template <> __device__ __forceinline__ unsigned sum2<__half>(unsigned a, unsigned b) {
    const __half2 x = *reinterpret_cast<const __half2 *>(&a), y = *reinterpret_cast<const __half2 *>(&b);
    return pack2<__half>(__low2float(x) + __low2float(y), __high2float(x) + __high2float(y));
}

// ---------------------------------------------------------------------------------------------------------------------------
// main loop of one tile for one consumer warpgroup: acc (64 x BN) = A[64 rows] . B^T over the K blocks [kb0, kb1)
// ---------------------------------------------------------------------------------------------------------------------------
template <typename TIn, int BN, int TA, int TB>
__device__ __forceinline__ void consume_tile(float (&acc)[(BN + 63) / 64][32], const GemmP &p, unsigned stage0, int stage_bytes,
                                             uint64_t *full, uint64_t *empty, int kb0, int kb1, unsigned &it, int cw, int lane) {
    constexpr int kChunks = (BN + 63) / 64, kLast = BN - 64 * (kChunks - 1);
    int prev = -1;
    for (int kb = kb0; kb < kb1; ++kb, ++it) {
        const int s = it % p.stages;
        mbar_wait_prof(&full[s], (it / p.stages) & 1, (p.prof && cw == 0 && threadIdx.x % 128 == 0) ? p.prof + 2 : nullptr);
        const unsigned sa = stage0 + (unsigned)(s * stage_bytes) + (unsigned)(cw * 8192), sb = stage0 + (unsigned)(s * stage_bytes) + kBM * 128;
        wg_fence();
        // a K tail needs no shorter loop: the TMA unit zero-filled the K positions past p.K in both operands
#pragma unroll
        for (int k = 0; k < kBK / kMmaK; ++k) {
            const uint64_t da = TA ? make_desc(sa + k * (kMmaK * 128), 8192, 1024) : make_desc(sa + k * (kMmaK * 2), 16, 1024);
            const unsigned acc_on = (kb > kb0 || k > 0) ? 1u : 0u;
#pragma unroll
            for (int c = 0; c < kChunks; ++c) {
                const uint64_t db = TB ? make_desc(sb + c * 8192 + k * (kMmaK * 128), 8192, 1024)
                                       : make_desc(sb + c * 8192 + k * (kMmaK * 2), 16, 1024);
                if (c + 1 < kChunks) wgmma_k16<TIn, 64, TA, TB>(acc[c], da, db, acc_on);
                else wgmma_k16<TIn, kLast, TA, TB>(acc[c], da, db, acc_on);
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
}

// ---------------------------------------------------------------------------------------------------------------------------
// TIn: __nv_bfloat16 / __half operands.  TOut: TIn (store) or float (store, or atomic accumulate when p.atomic)
// ---------------------------------------------------------------------------------------------------------------------------
template <typename TIn, typename TOut, int BN>
__global__ void __launch_bounds__(kThreads, 1) gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA,
                                                              const __grid_constant__ CUtensorMap tmB, const GemmP p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    constexpr int kChunks = (BN + 63) / 64;
    constexpr int a_tile = kBM * 128;                       // bytes per stage
    const int b_tile = p.b_mn ? kChunks * 8192 : BN * 128;
    const int stage_bytes = a_tile + ((b_tile + 1023) & ~1023);
    uint8_t *stage0 = smem;
    uint8_t *staging = smem + (size_t)p.stages * stage_bytes;                 // 8 warps x 16 rows x 144 bytes
    uint64_t *bars = reinterpret_cast<uint64_t *>(staging + kStagingBytes);
    uint64_t *full = bars, *empty = bars + kMaxStages;

    if (threadIdx.x == 0) {
        for (int s = 0; s < p.stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kConsumerWarps); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    }
    __syncthreads();
    const long long t_start = clock64();

    const int m_tiles = (p.M + kBM - 1) / kBM;
    const int n_tiles = (p.N + BN - 1) / BN;
    const int kb_total = (p.K + kBK - 1) / kBK;
    const int kb_per = (kb_total + p.split_k - 1) / p.split_k;
    const int n_work = m_tiles * n_tiles * p.split_k;

    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (threadIdx.x == 0) {
            unsigned it = 0;
            for (int t = blockIdx.x; t < n_work; t += gridDim.x) {
                const int sp = t % p.split_k, nb = (t / p.split_k) % n_tiles, mb = t / (p.split_k * n_tiles);
                const int kb0 = sp * kb_per, kb1 = min(kb_total, kb0 + kb_per);
                for (int kb = kb0; kb < kb1; ++kb, ++it) {
                    const int s = it % p.stages;
                    const unsigned ph = (it / p.stages) & 1;
                    mbar_wait_prof(&empty[s], ph ^ 1, p.prof ? p.prof + 0 : nullptr);
                    uint8_t *sa = stage0 + (size_t)s * stage_bytes, *sb = sa + a_tile;
                    mbar_expect_tx(&full[s], (unsigned)(a_tile + b_tile));
                    if (!p.a_mn) {
                        tma_load_2d(sa, &tmA, kb * kBK, mb * kBM, &full[s]);
                    } else {
                        tma_load_2d(sa, &tmA, mb * kBM, kb * kBK, &full[s]);
                        tma_load_2d(sa + 8192, &tmA, mb * kBM + 64, kb * kBK, &full[s]);
                    }
                    if (!p.b_mn) {
                        tma_load_2d(sb, &tmB, kb * kBK, nb * BN, &full[s]);
                    } else {
                        for (int c = 0; c < kChunks; ++c) tma_load_2d(sb + c * 8192, &tmB, nb * BN + c * 64, kb * kBK, &full[s]);
                    }
                }
            }
        }
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
        // ------------------------------------ consumer warpgroups: rows 64 cw .. 64 cw + 63 ------------------------------------
        // After the main loop a warp holds 16 rows of the tile.  It parks kGC converted columns at a time in its private staging
        // tile of 16 rows x 128 bytes and writes the tile out with 8 lanes per row, i.e. one full 128-byte line per row and four
        // lines per store instruction (the fragment's own layout would store 4- or 8-byte pieces).  No CTA-level barrier: the
        // tile is private to the warp.
        const int cw = (warp >> 2) - 1, wq = warp & 3;
        const int r0 = lane >> 2, q = lane & 3;
        TOut *const D = reinterpret_cast<TOut *>(p.D);
        constexpr int kGC = 128 / (int)sizeof(TOut);     // columns per staged group: 64 (16-bit) or 32 (fp32)
        constexpr int kVec = 16 / (int)sizeof(TOut);
        uint8_t *stg = staging + (size_t)(warp - 4) * (16 * kPitch);
        const unsigned stage0_addr = smem_u32(stage0);
        float acc[kChunks][32];
        unsigned it = 0;
        for (int t = blockIdx.x; t < n_work; t += gridDim.x) {
            const int nb = (t / p.split_k) % n_tiles, mb = t / (p.split_k * n_tiles);
            const int sp = t % p.split_k;
            const int kb0 = sp * kb_per, kb1 = min(kb_total, kb0 + kb_per);
            switch (p.a_mn * 2 + p.b_mn) {
                case 0: consume_tile<TIn, BN, 0, 0>(acc, p, stage0_addr, stage_bytes, full, empty, kb0, kb1, it, cw, lane); break;
                case 1: consume_tile<TIn, BN, 0, 1>(acc, p, stage0_addr, stage_bytes, full, empty, kb0, kb1, it, cw, lane); break;
                case 2: consume_tile<TIn, BN, 1, 0>(acc, p, stage0_addr, stage_bytes, full, empty, kb0, kb1, it, cw, lane); break;
                default: consume_tile<TIn, BN, 1, 1>(acc, p, stage0_addr, stage_bytes, full, empty, kb0, kb1, it, cw, lane); break;
            }
            const long long t_tile0 = p.prof ? clock64() : 0;
            const int n0 = nb * BN;
            const int m0 = mb * kBM + cw * 64 + wq * 16;   // first row of this warp
            const int n_valid = min(BN, p.N - n0);
            const bool bias_m_on = p.epilogue == GEMM_EPI_BIAS_M && p.bias && sp == 0;
            const float bias_m0 = (bias_m_on && m0 + r0 < p.M) ? p.bias[m0 + r0] : 0.f;
            const float bias_m1 = (bias_m_on && m0 + r0 + 8 < p.M) ? p.bias[m0 + r0 + 8] : 0.f;
            if (m0 < p.M) {
#pragma unroll
                for (int g0 = 0; g0 < BN; g0 += kGC) {
                    if (g0 < n_valid) {
#pragma unroll
                        for (int jj = 0; jj < kGC / 8; ++jj) {
                            const int j = g0 / 8 + jj;                    // 8-column block of the tile
                            if (8 * j < BN) {
                                const float *a4 = &acc[j / 8][4 * (j % 8)];
                                float v[4] = {a4[0], a4[1], a4[2], a4[3]};
                                const int col = 8 * j + 2 * q;
                                if (p.epilogue == GEMM_EPI_BIAS_N || p.epilogue == GEMM_EPI_BIAS_N_GELU) {
                                    if (p.bias && sp == 0) {
                                        const float b0 = (n0 + col < p.N) ? __ldg(p.bias + n0 + col) : 0.f;
                                        const float b1 = (n0 + col + 1 < p.N) ? __ldg(p.bias + n0 + col + 1) : 0.f;
                                        v[0] += b0; v[1] += b1; v[2] += b0; v[3] += b1;
                                    }
                                    if (p.epilogue == GEMM_EPI_BIAS_N_GELU) {
#pragma unroll
                                        for (int i = 0; i < 4; ++i) v[i] = gelu_erf(v[i]);
                                    }
                                } else if (p.epilogue == GEMM_EPI_BIAS_M) {
                                    v[0] += bias_m0; v[1] += bias_m0; v[2] += bias_m1; v[3] += bias_m1;
                                }
                                uint8_t *s0 = stg + r0 * kPitch + (8 * jj + 2 * q) * (int)sizeof(TOut), *s1 = s0 + 8 * kPitch;
                                if constexpr (sizeof(TOut) == 4) {
                                    *reinterpret_cast<float2 *>(s0) = make_float2(v[0], v[1]);
                                    *reinterpret_cast<float2 *>(s1) = make_float2(v[2], v[3]);
                                } else {
                                    *reinterpret_cast<unsigned *>(s0) = pack2<TOut>(v[0], v[1]);
                                    *reinterpret_cast<unsigned *>(s1) = pack2<TOut>(v[2], v[3]);
                                }
                            }
                        }
                        __syncwarp();
                        // ---- write the group out: lane -> (row = 4 i4 + lane / 8, 16-byte piece = lane % 8) ----
#pragma unroll
                        for (int i4 = 0; i4 < 4; ++i4) {
                            const int r = 4 * i4 + (lane >> 3), pc = lane & 7;
                            const int col = g0 + pc * kVec, m = m0 + r;
                            if (m < p.M && col < n_valid) {
                                const uint8_t *src = stg + r * kPitch + pc * 16;
                                TOut *dst = D + (int64_t)m * p.ldd + n0 + col;
                                const bool full16 = (col + kVec <= n_valid) && ((reinterpret_cast<uintptr_t>(dst) & 15) == 0);
                                if constexpr (sizeof(TOut) == 4) {
                                    const F4 sv = *reinterpret_cast<const F4 *>(src);
                                    float *fd = reinterpret_cast<float *>(dst);
                                    if (full16) {
                                        if (p.atomic) red_add_v4f(fd, sv.x, sv.y, sv.z, sv.w);
                                        else *reinterpret_cast<F4 *>(fd) = sv;
                                    } else {
                                        const float e4[4] = {sv.x, sv.y, sv.z, sv.w};
#pragma unroll
                                        for (int i = 0; i < 4; ++i) {
                                            if (col + i < n_valid) {
                                                if (p.atomic) atomicAdd(fd + i, e4[i]);
                                                else fd[i] = e4[i];
                                            }
                                        }
                                    }
                                } else {
                                    uint4 sv = *reinterpret_cast<const uint4 *>(src);
                                    if (full16) {
                                        if (p.atomic) {                   // D += product (16-bit outputs: read-modify-write, no split-K)
                                            const uint4 o = *reinterpret_cast<const uint4 *>(dst);
                                            sv = make_uint4(sum2<TOut>(o.x, sv.x), sum2<TOut>(o.y, sv.y), sum2<TOut>(o.z, sv.z), sum2<TOut>(o.w, sv.w));
                                        }
                                        *reinterpret_cast<uint4 *>(dst) = sv;
                                    } else {
                                        const TOut *se = reinterpret_cast<const TOut *>(&sv);
#pragma unroll
                                        for (int i = 0; i < kVec; ++i) {
                                            if (col + i < n_valid) {
                                                const float o = p.atomic ? static_cast<float>(dst[i]) + static_cast<float>(se[i]) : static_cast<float>(se[i]);
                                                dst[i] = static_cast<TOut>(o);
                                            }
                                        }
                                    }
                                }
                            }
                        }
                        __syncwarp();
                    }
                }
            }
            if (p.prof && warp == 4 && lane == 0) atomicAdd(p.prof + 11, (unsigned long long)(clock64() - t_tile0));
        }
        if (p.prof && warp == 4 && lane == 0) atomicAdd(p.prof + 7, (unsigned long long)(clock64() - t_start));
    }
}

// ---------------------------------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                             const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                             CUtensorMapFloatOOBfill);

cudaError_t encode_2d(CUtensorMap *m, const void *base, int dtype, uint64_t inner, uint64_t outer, uint64_t outer_stride_bytes,
                      uint32_t box_inner, uint32_t box_outer) {
    static EncodeFn fn = nullptr;
    if (!fn) {
        void *ptr = nullptr;
        cudaDriverEntryPointQueryResult q;
        cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q);
        if (e != cudaSuccess) return e;
        if (q != cudaDriverEntryPointSuccess || !ptr) return cudaErrorNotSupported;
        fn = reinterpret_cast<EncodeFn>(ptr);
    }
    cuuint64_t dims[2] = {inner, outer};
    cuuint64_t strides[1] = {outer_stride_bytes};
    cuuint32_t box[2] = {box_inner, box_outer};
    cuuint32_t estr[2] = {1, 1};
    const CUresult r = fn(m, dtype == 1 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void *>(base),
                          dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                          CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r == CUDA_ERROR_INVALID_CONTEXT || r == CUDA_ERROR_NOT_INITIALIZED) return cudaErrorDeviceUninitialized;
    return r == CUDA_SUCCESS ? cudaSuccess : cudaErrorInvalidValue;
}

}  // namespace

// the narrowest instantiated tile that covers N (256 for anything wider)
int gemm_pick_bn(int N) {
    for (int bn : {16, 32, 48, 64, 96, 128, 192}) {
        if (N <= bn) return bn;
    }
    return 256;
}

cudaError_t gemm_tc_launch(GemmP p, const void *A, int64_t lda, const void *B, int64_t ldb, cudaStream_t st, const char **where) {
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
    if (p.BN <= 0) p.BN = gemm_pick_bn(p.N);
    if (p.BN != gemm_pick_bn(p.BN)) return cudaErrorInvalidValue;      // a preset BN must be one of the instantiated tiles
    const int BN = p.BN;
    const size_t b_tile = p.b_mn ? (size_t)((BN + 63) / 64) * 8192 : (size_t)BN * 128;
    const size_t stage_bytes = (size_t)kBM * 128 + ((b_tile + 1023) & ~(size_t)1023);
    const size_t fixed = 1024 + kStagingBytes + 2 * kMaxStages * 8;
    int stages = (int)(((size_t)max_smem - fixed) / stage_bytes);
    if (stages > kMaxStages) stages = kMaxStages;
    const int kb_total = (p.K + kBK - 1) / kBK;
    if (stages < 2) return cudaErrorInvalidConfiguration;
    p.stages = stages;
    if (p.split_k < 1) p.split_k = 1;
    if (p.split_k > kb_total) p.split_k = kb_total;
    {   // no K slice may be empty: an accumulator that no wgmma wrote would be added as is
        const int kb_per = (kb_total + p.split_k - 1) / p.split_k;
        p.split_k = (kb_total + kb_per - 1) / kb_per;
    }
    const size_t smem = fixed + (size_t)stages * stage_bytes;

    CUtensorMap tmA, tmB;
    cudaError_t e;
    {   // cuTensorMapEncodeTiled is a DRIVER call: it needs a current context in the calling thread.  PyTorch's autograd worker
        // threads select their device lazily, so a backward whose first CUDA work is this GEMM arrives here with no context
        // bound (seen on hardware as CUDA_ERROR_INVALID_CONTEXT).  Bind the primary context of the device that owns A.
        *where = "cudaPointerGetAttributes(A)";
        cudaPointerAttributes attr;
        if ((e = cudaPointerGetAttributes(&attr, A)) != cudaSuccess) return e;
        if (attr.type != cudaMemoryTypeDevice && attr.type != cudaMemoryTypeManaged) return cudaErrorInvalidDevicePointer;
        if ((e = cudaSetDevice(attr.device)) != cudaSuccess) return e;
    }
    *where = "tensor map of A (cuTensorMapEncodeTiled)";
    // A: K-major -> dims (K, M), box (64, 128); MN-major -> dims (M, K), box (64, 64) loaded twice per stage
    e = p.a_mn ? encode_2d(&tmA, A, p.dtype, (uint64_t)p.M, (uint64_t)p.K, (uint64_t)lda * 2, 64, 64)
               : encode_2d(&tmA, A, p.dtype, (uint64_t)p.K, (uint64_t)p.M, (uint64_t)lda * 2, 64, kBM);
    if (e != cudaSuccess) return e;
    *where = "tensor map of B (cuTensorMapEncodeTiled)";
    e = p.b_mn ? encode_2d(&tmB, B, p.dtype, (uint64_t)p.N, (uint64_t)p.K, (uint64_t)ldb * 2, 64, 64)
               : encode_2d(&tmB, B, p.dtype, (uint64_t)p.K, (uint64_t)p.N, (uint64_t)ldb * 2, 64, (uint32_t)BN);
    if (e != cudaSuccess) return e;

    const int m_tiles = (p.M + kBM - 1) / kBM, n_tiles = (p.N + BN - 1) / BN;
    const long n_work = (long)m_tiles * n_tiles * p.split_k;
    const int grid = (int)(n_work < (long)sms ? n_work : (long)sms);
#define SMB_GEMM_LAUNCH(TIn, TOut, kBN)                                                                                     \
    do {                                                                                                                    \
        static bool set = false;                                                                                            \
        *where = "cudaFuncSetAttribute";                                                                                    \
        if (!set) {                                                                                                         \
            e = cudaFuncSetAttribute(gemm_tc_kernel<TIn, TOut, kBN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)max_smem); \
            if (e != cudaSuccess) return e;                                                                                 \
            set = true;                                                                                                     \
        }                                                                                                                   \
        *where = "kernel launch";                                                                                           \
        gemm_tc_kernel<TIn, TOut, kBN><<<grid, kThreads, smem, st>>>(tmA, tmB, p);                                          \
    } while (0)
#define SMB_GEMM_TYPES(kBN)                                                                                                 \
    do {                                                                                                                    \
        if (p.dtype == 1 && p.out_dtype == 0) SMB_GEMM_LAUNCH(__half, float, kBN);                                          \
        else if (p.dtype == 1) SMB_GEMM_LAUNCH(__half, __half, kBN);                                                        \
        else if (p.out_dtype == 0) SMB_GEMM_LAUNCH(__nv_bfloat16, float, kBN);                                              \
        else SMB_GEMM_LAUNCH(__nv_bfloat16, __nv_bfloat16, kBN);                                                            \
    } while (0)
    switch (BN) {
        case 16: SMB_GEMM_TYPES(16); break;
        case 32: SMB_GEMM_TYPES(32); break;
        case 48: SMB_GEMM_TYPES(48); break;
        case 64: SMB_GEMM_TYPES(64); break;
        case 96: SMB_GEMM_TYPES(96); break;
        case 128: SMB_GEMM_TYPES(128); break;
        case 192: SMB_GEMM_TYPES(192); break;
        default: SMB_GEMM_TYPES(256); break;
    }
#undef SMB_GEMM_TYPES
#undef SMB_GEMM_LAUNCH
    count_launch();
    return cudaGetLastError();
}

}  // namespace smb
