// Internal interface of the training-patch augmentation kernels (augment.cu) for capi.cu.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "../../include/segmamba_b200.h"

namespace smb {

// jobs per launch: the records travel by value in the kernel parameters (no host-to-device copy, no allocation, and the
// caller's host array may be reused as soon as the entry point returns); longer lists are split into several launches
constexpr int kAugMaxJobs = 8;
// longest axis of a training patch (crop, blur, emit) and of a mirror-boundary prefilter line
constexpr int kAugMaxAxis = 256;
// longest prefilter line staged whole in shared memory (n + 24 samples per line); longer edge-boundary lines stream
constexpr int kAugShortLine = 256;
// blocks per stats job (partial sums land in the job's scratch, then one ordered reduction: deterministic)
constexpr int kAugStatsBlocks = SMB_AUG_STATS_SCRATCH / 4;

// Philox4x32-10 (Salmon et al., SC'11): counter (c0..c3), key (k0, k1) -> four 32-bit words.  Host and device.
__host__ __device__ inline void philox4x32_10(uint32_t c[4], uint32_t k0, uint32_t k1) {
    for (int r = 0; r < 10; ++r) {
        const uint64_t p0 = (uint64_t)0xD2511F53u * c[0], p1 = (uint64_t)0xCD9E8D57u * c[2];
        const uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0, hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
        const uint32_t n0 = hi1 ^ c[1] ^ k0, n2 = hi0 ^ c[3] ^ k1;
        c[0] = n0; c[1] = lo1; c[2] = n2; c[3] = lo0;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
}

cudaError_t aug_crop_launch(const smb_aug_crop_args &a, cudaStream_t st);
cudaError_t aug_prefilter_launch(const smb_aug_prefilter_job *jobs, int n, cudaStream_t st);
cudaError_t aug_resample_launch(const smb_aug_resample_job *jobs, int n, cudaStream_t st);
cudaError_t aug_blur_launch(const smb_aug_blur_job *jobs, int n, cudaStream_t st);
cudaError_t aug_stats_launch(const smb_aug_stats_job *jobs, int n, cudaStream_t st);
cudaError_t aug_pointwise_launch(const smb_aug_point_job *jobs, int n, cudaStream_t st);
cudaError_t aug_emit_launch(const smb_aug_emit_args &a, cudaStream_t st);

}  // namespace smb
