// Strided 2-D copy with 16-byte vectors: rows x row_bytes, arbitrary (16-byte multiple) row pitches on both sides.
//
// Used for torch.cat((up, skip), dim=1) of UnetrUpBlock (monai/networks/blocks/unetr_block.py:81-86) on channels-last activations:
// a channel concatenation of two (tokens, C) matrices is two such copies into the (tokens, 2C) result, and its backward two copies
// out of it.  ATen runs these as generic strided elementwise kernels; this one
// streams full 16-byte vectors with consecutive threads on consecutive vectors of a row.
#include <cuda_runtime.h>

#include <cstdint>

#include "conv_internal.h"

namespace smb {
void count_launch();

__global__ void __launch_bounds__(256) copy2d_kernel(const uint4 *__restrict__ src, uint4 *__restrict__ dst, int64_t rows, int vecs,
                                                     int64_t src_pitch, int64_t dst_pitch) {
    // thread -> (row, vector): `vecs` threads per row, several rows per CTA; four vectors in flight per thread
    const int64_t total = rows * vecs;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (; i + 3 * stride < total; i += 4 * stride) {
        uint4 v[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int64_t j = i + k * stride, r = j / vecs;
            v[k] = __ldg(src + r * src_pitch + (j - r * vecs));
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int64_t j = i + k * stride, r = j / vecs;
            dst[r * dst_pitch + (j - r * vecs)] = v[k];
        }
    }
    for (; i < total; i += stride) {
        const int64_t r = i / vecs;
        dst[r * dst_pitch + (i - r * vecs)] = __ldg(src + r * src_pitch + (i - r * vecs));
    }
}

cudaError_t copy2d_launch(const void *src, int64_t src_pitch_bytes, void *dst, int64_t dst_pitch_bytes, int64_t rows, int64_t row_bytes,
                          cudaStream_t st) {
    const int vecs = (int)(row_bytes / 16);
    const int64_t total = rows * vecs;
    int64_t blocks = (total + 256 * 4 - 1) / (256 * 4);
    if (blocks > 132 * 32) blocks = 132 * 32;
    if (blocks < 1) blocks = 1;
    copy2d_kernel<<<(unsigned)blocks, 256, 0, st>>>(reinterpret_cast<const uint4 *>(src), reinterpret_cast<uint4 *>(dst), rows, vecs,
                                                    src_pitch_bytes / 16, dst_pitch_bytes / 16);
    count_launch();
    return cudaGetLastError();
}

}  // namespace smb
