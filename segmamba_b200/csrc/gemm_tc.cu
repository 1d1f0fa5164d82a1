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
#include "wgmma_pipe.cuh"

namespace smb {
void count_launch();

namespace {

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }

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
        // After the main loop a warp holds 16 rows of the tile and writes them through its private staging tile (store_tile):
        // no CTA-level barrier, so the producer already fills the ring for the next tile.
        const int cw = (warp >> 2) - 1, wq = warp & 3;
        const int r0 = lane >> 2;
        TOut *const D = reinterpret_cast<TOut *>(p.D);
        uint8_t *stg = staging + (size_t)(warp - 4) * (16 * kPitch);
        const unsigned stage0_addr = smem_u32(stage0);
        float acc[kChunks][32];
        unsigned it = 0;
        for (int t = blockIdx.x; t < n_work; t += gridDim.x) {
            const int nb = (t / p.split_k) % n_tiles, mb = t / (p.split_k * n_tiles);
            const int sp = t % p.split_k;
            const int kb0 = sp * kb_per, kb1 = min(kb_total, kb0 + kb_per);
            switch (p.a_mn * 2 + p.b_mn) {
                case 0: consume_tile<TIn, BN, 0, 0>(acc, p.stages, p.prof, stage0_addr, stage_bytes, full, empty, kb0, kb1, it, cw, lane); break;
                case 1: consume_tile<TIn, BN, 0, 1>(acc, p.stages, p.prof, stage0_addr, stage_bytes, full, empty, kb0, kb1, it, cw, lane); break;
                case 2: consume_tile<TIn, BN, 1, 0>(acc, p.stages, p.prof, stage0_addr, stage_bytes, full, empty, kb0, kb1, it, cw, lane); break;
                default: consume_tile<TIn, BN, 1, 1>(acc, p.stages, p.prof, stage0_addr, stage_bytes, full, empty, kb0, kb1, it, cw, lane); break;
            }
            const long long t_tile0 = p.prof ? clock64() : 0;
            const int n0 = nb * BN;
            const int m0 = mb * kBM + cw * 64 + wq * 16;   // first row of this warp
            const int n_valid = min(BN, p.N - n0);
            const bool bias_m_on = p.epilogue == GEMM_EPI_BIAS_M && p.bias && sp == 0;
            const float bias_m0 = (bias_m_on && m0 + r0 < p.M) ? p.bias[m0 + r0] : 0.f;
            const float bias_m1 = (bias_m_on && m0 + r0 + 8 < p.M) ? p.bias[m0 + r0 + 8] : 0.f;
            if (m0 < p.M) {
                store_tile<TOut, BN>(
                    acc, stg, lane, n_valid, p.atomic != 0,
                    [&](int col, float (&v)[4]) {
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
                    },
                    [&](int r) -> TOut * { return m0 + r < p.M ? D + (int64_t)(m0 + r) * p.ldd + n0 : nullptr; });
            }
            if (p.prof && warp == 4 && lane == 0) atomicAdd(p.prof + 11, (unsigned long long)(clock64() - t_tile0));
        }
        if (p.prof && warp == 4 && lane == 0) atomicAdd(p.prof + 7, (unsigned long long)(clock64() - t_start));
    }
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
    *where = "cudaPointerGetAttributes(A)";
    if ((e = bind_device_of(A)) != cudaSuccess) return e;
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
