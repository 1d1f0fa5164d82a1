// The TMA -> shared memory -> wgmma pipeline shared by the tensor-core GEMM (gemm_tc.cu) and the implicit-GEMM 3x3x3
// convolution (conv3d_tc.cu): mbarrier and wgmma wrappers, shared-memory matrix descriptors, the consumer side of the stage
// ring, the staged epilogue and the tensor-map encoder.
//
// Tile geometry (both kernels): 128 rows (two consumer warpgroups x wgmma M = 64) x BN columns, K blocks of 64 sixteen-bit
// elements = one 128-byte swizzle row (CU_TENSOR_MAP_SWIZZLE_128B).  One persistent CTA per SM, 384 threads: warpgroup 0 is the
// TMA producer (one thread), warpgroups 1 and 2 run wgmma and the epilogue.  A stage holds the A tile (128 rows x 128 B, the
// rows of consumer warpgroup cw at cw * 8192) followed by the B tile at kBM * 128.
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cstdint>

namespace smb {
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
// optional profiling (acc != nullptr): cycles a role spends inside a barrier wait, summed over the grid
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
__device__ __forceinline__ void tma_load_3d(void *smem, const CUtensorMap *m, int c0, int c1, int c2, uint64_t *bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(
                     smem_u32(smem)),
                 "l"(m), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar))
                 : "memory");
}
// coordinates are signed: a box that starts before the tensor (a convolution tap at the border) is zero-filled there
__device__ __forceinline__ void tma_load_5d(void *smem, const CUtensorMap *m, int c0, int c1, int c2, int c3, int c4, uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5, %6}], [%7];" ::"r"(
            smem_u32(smem)),
        "l"(m), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4), "r"(smem_u32(bar))
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
// consumer side of the ring, one tile for one consumer warpgroup: acc (64 x BN) = A[64 rows] . B^T over K blocks [kb0, kb1).
// `it` counts K blocks over the CTA's whole life (the producer counts the same way), so stage and phase follow from it.
// ---------------------------------------------------------------------------------------------------------------------------
//   kSub > 1: a stage holds kSub K blocks that share one A box, at byte offsets a_sub (A) and b_sub (B) apart (both multiples of
//   1024, so the swizzle phase is unchanged); b_offset is where the B operand starts within a stage.
template <typename TIn, int BN, int TA, int TB, int kSub = 1>
__device__ __forceinline__ void consume_tile(float (&acc)[(BN + 63) / 64][32], int stages, unsigned long long *prof, unsigned stage0,
                                             int stage_bytes, uint64_t *full, uint64_t *empty, int kb0, int kb1, unsigned &it, int cw,
                                             int lane, int b_offset = kBM * 128, int a_sub = 0, int b_sub = 0) {
    constexpr int kChunks = (BN + 63) / 64, kLast = BN - 64 * (kChunks - 1);
    int prev = -1;
    for (int kb = kb0; kb < kb1; ++kb, ++it) {
        const int s = it % stages;
        mbar_wait_prof(&full[s], (it / stages) & 1, (prof && cw == 0 && threadIdx.x % 128 == 0) ? prof + 2 : nullptr);
        wg_fence();
#pragma unroll
        for (int j = 0; j < kSub; ++j) {
            const unsigned sa = stage0 + (unsigned)(s * stage_bytes) + (unsigned)(cw * 8192 + j * a_sub);
            const unsigned sb = stage0 + (unsigned)(s * stage_bytes) + (unsigned)(b_offset + j * b_sub);
            // a K tail needs no shorter loop: the TMA unit zero-filled the K positions past the end in both operands
#pragma unroll
            for (int k = 0; k < kBK / kMmaK; ++k) {
                const uint64_t da = TA ? make_desc(sa + k * (kMmaK * 128), 8192, 1024) : make_desc(sa + k * (kMmaK * 2), 16, 1024);
                const unsigned acc_on = (kb > kb0 || j > 0 || k > 0) ? 1u : 0u;
#pragma unroll
                for (int c = 0; c < kChunks; ++c) {
                    const uint64_t db = TB ? make_desc(sb + c * 8192 + k * (kMmaK * 128), 8192, 1024)
                                           : make_desc(sb + c * 8192 + k * (kMmaK * 2), 16, 1024);
                    if (c + 1 < kChunks) wgmma_k16<TIn, 64, TA, TB>(acc[c], da, db, acc_on);
                    else wgmma_k16<TIn, kLast, TA, TB>(acc[c], da, db, acc_on);
                }
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
// staged epilogue of one warp (16 rows of the tile): converts kGC columns at a time into the warp-private staging tile
// (16 rows x 128 bytes, pitch kPitch) and writes it out with 8 lanes per row, i.e. one full 128-byte line per row.
//   xform(col, v[4])  adjusts the four accumulator values of tile column col, col + 1 (rows lane / 4 and lane / 4 + 8)
//   row_ptr(r)        the address of tile column 0 of the warp's row r (0..15), or nullptr for a row that is not stored
//   accumulate        fp32: red.global.add into D (split-K); 16-bit: D += product (read-modify-write)
// ---------------------------------------------------------------------------------------------------------------------------
template <typename TOut, int BN, typename Xform, typename RowPtr>
__device__ __forceinline__ void store_tile(const float (&acc)[(BN + 63) / 64][32], uint8_t *stg, int lane, int n_valid, bool accumulate,
                                           Xform xform, RowPtr row_ptr) {
    constexpr int kGC = 128 / (int)sizeof(TOut);     // columns per staged group: 64 (16-bit) or 32 (fp32)
    constexpr int kVec = 16 / (int)sizeof(TOut);
    const int r0 = lane >> 2, q = lane & 3;
#pragma unroll
    for (int g0 = 0; g0 < BN; g0 += kGC) {
        if (g0 < n_valid) {
#pragma unroll
            for (int jj = 0; jj < kGC / 8; ++jj) {
                const int j = g0 / 8 + jj;                    // 8-column block of the tile
                if (8 * j < BN) {
                    const float *a4 = &acc[j / 8][4 * (j % 8)];
                    float v[4] = {a4[0], a4[1], a4[2], a4[3]};
                    xform(8 * j + 2 * q, v);
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
                const int col = g0 + pc * kVec;
                TOut *const row = row_ptr(r);
                if (row != nullptr && col < n_valid) {
                    const uint8_t *src = stg + r * kPitch + pc * 16;
                    TOut *dst = row + col;
                    const bool full16 = (col + kVec <= n_valid) && ((reinterpret_cast<uintptr_t>(dst) & 15) == 0);
                    if constexpr (sizeof(TOut) == 4) {
                        const F4 sv = *reinterpret_cast<const F4 *>(src);
                        float *fd = reinterpret_cast<float *>(dst);
                        if (full16) {
                            if (accumulate) red_add_v4f(fd, sv.x, sv.y, sv.z, sv.w);
                            else *reinterpret_cast<F4 *>(fd) = sv;
                        } else {
                            const float e4[4] = {sv.x, sv.y, sv.z, sv.w};
#pragma unroll
                            for (int i = 0; i < 4; ++i) {
                                if (col + i < n_valid) {
                                    if (accumulate) atomicAdd(fd + i, e4[i]);
                                    else fd[i] = e4[i];
                                }
                            }
                        }
                    } else {
                        uint4 sv = *reinterpret_cast<const uint4 *>(src);
                        if (full16) {
                            if (accumulate) {                   // D += product (16-bit outputs: read-modify-write, no split-K)
                                const uint4 o = *reinterpret_cast<const uint4 *>(dst);
                                sv = make_uint4(sum2<TOut>(o.x, sv.x), sum2<TOut>(o.y, sv.y), sum2<TOut>(o.z, sv.z), sum2<TOut>(o.w, sv.w));
                            }
                            *reinterpret_cast<uint4 *>(dst) = sv;
                        } else {
                            const TOut *se = reinterpret_cast<const TOut *>(&sv);
#pragma unroll
                            for (int i = 0; i < kVec; ++i) {
                                if (col + i < n_valid) {
                                    const float o = accumulate ? static_cast<float>(dst[i]) + static_cast<float>(se[i]) : static_cast<float>(se[i]);
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

// ---------------------------------------------------------------------------------------------------------------------------
// tiled tensor map with a 128-byte swizzle.  dims[0] is the contiguous axis (elements); strides[i] is the byte stride of
// dims[i + 1].  cuTensorMapEncodeTiled is resolved at run time (libcuda is not linked), so the library loads without a driver.
// ---------------------------------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                             const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                             CUtensorMapFloatOOBfill);

inline cudaError_t encode_tiled(CUtensorMap *m, const void *base, int dtype, int rank, const uint64_t *dims, const uint64_t *strides_bytes,
                                const uint32_t *box) {
    static EncodeFn fn = nullptr;
    if (!fn) {
        void *ptr = nullptr;
        cudaDriverEntryPointQueryResult q;
        cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q);
        if (e != cudaSuccess) return e;
        if (q != cudaDriverEntryPointSuccess || !ptr) return cudaErrorNotSupported;
        fn = reinterpret_cast<EncodeFn>(ptr);
    }
    cuuint64_t d[5], s[4];
    cuuint32_t b[5], estr[5];
    for (int i = 0; i < rank; ++i) { d[i] = dims[i]; b[i] = box[i]; estr[i] = 1; }
    for (int i = 0; i + 1 < rank; ++i) s[i] = strides_bytes[i];
    const CUresult r = fn(m, dtype == 1 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank,
                          const_cast<void *>(base), d, s, b, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                          CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r == CUDA_ERROR_INVALID_CONTEXT || r == CUDA_ERROR_NOT_INITIALIZED) return cudaErrorDeviceUninitialized;
    return r == CUDA_SUCCESS ? cudaSuccess : cudaErrorInvalidValue;
}

inline cudaError_t encode_2d(CUtensorMap *m, const void *base, int dtype, uint64_t inner, uint64_t outer, uint64_t outer_stride_bytes,
                             uint32_t box_inner, uint32_t box_outer) {
    const uint64_t dims[2] = {inner, outer}, strides[1] = {outer_stride_bytes};
    const uint32_t box[2] = {box_inner, box_outer};
    return encode_tiled(m, base, dtype, 2, dims, strides, box);
}

// cuTensorMapEncodeTiled is a DRIVER call: it needs a current context in the calling thread.  PyTorch's autograd worker threads
// select their device lazily, so a backward whose first CUDA work is one of these kernels arrives with no context bound (seen on
// hardware as CUDA_ERROR_INVALID_CONTEXT).  Bind the primary context of the device that owns `p`.
inline cudaError_t bind_device_of(const void *p) {
    cudaPointerAttributes attr;
    cudaError_t e = cudaPointerGetAttributes(&attr, p);
    if (e != cudaSuccess) return e;
    if (attr.type != cudaMemoryTypeDevice && attr.type != cudaMemoryTypeManaged) return cudaErrorInvalidDevicePointer;
    return cudaSetDevice(attr.device);
}

}  // namespace
}  // namespace smb
