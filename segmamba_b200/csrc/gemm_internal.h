// internal interface of the tensor-core GEMM (gemm_tc.cu); the C ABI wrapper lives in capi.cu
#pragma once

#include <cuda_runtime.h>

#include <cstdint>

namespace smb {

enum { GEMM_EPI_NONE = 0, GEMM_EPI_BIAS_N = 1, GEMM_EPI_BIAS_N_GELU = 2, GEMM_EPI_BIAS_M = 3 };

struct GemmP {
    int M, N, K;            // D[M, N] = A[M, K] . B[N, K]^T
    int dtype;              // operand type: 1 fp16, 2 bf16
    int out_dtype;          // 0 fp32, 1 fp16, 2 bf16
    int a_mn, b_mn;         // 0: K-major (K contiguous), 1: MN-major (M / N contiguous, rows = K index)
    int epilogue;           // GEMM_EPI_*
    int atomic;             // fp32 output only: atomicAdd into D (split-K partial products; D zero-initialised by the caller)
    int split_k;            // number of K slices handled by different CTAs (requires atomic when > 1)
    int BN, stages;         // filled by the launcher (BN may be preset: one of the tile widths gemm_pick_bn returns)
    const float *bias;
    void *D;
    int64_t ldd;            // elements
    unsigned long long *prof;   // optional 16 device counters: cycles in barrier waits per role (gemm_tc.cu), else nullptr
};

int gemm_pick_bn(int N);
cudaError_t gemm_tc_launch(GemmP p, const void *A, int64_t lda, const void *B, int64_t ldb, cudaStream_t st,
                           const char **where = nullptr);

}  // namespace smb
