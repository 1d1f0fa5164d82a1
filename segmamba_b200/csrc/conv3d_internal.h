// internal interface of the implicit-GEMM 3x3x3 convolution (conv3d_tc.cu); the C ABI wrapper lives in capi.cu
#pragma once

#include <cuda_runtime.h>

#include <cstdint>

namespace smb {

struct Conv3dP {
    int batch, D, H, W;     // spatial extent of input and output (stride 1, padding 1)
    int C_in, C_out;        // channels of X and Y
    int dtype;              // operand type: 1 fp16, 2 bf16
    int wgrad;              // 0: Y = conv(X, Wt) (16-bit out);  1: dW += X (*) dY (fp32 out, accumulated)
    void *out;              // Y (batch, D, H, W, C_out) or dW (C_out, 27, C_in), fp32, zero-initialised by the caller
    // filled by the launcher
    int BN, stages, bw, bh, bd, tw, th, td, cb, cob, m_tiles, n_tiles, kb_total, split_k;
};

// forward:  x = X (batch, D, H, W, C_in), b = Wt (C_out, 27, C_in)          -> Y
// wgrad:    x = X (batch, D, H, W, C_in), b = dY (batch, D, H, W, C_out)    -> dW
cudaError_t conv3d_tc_launch(Conv3dP p, const void *x, const void *b, cudaStream_t st, const char **where = nullptr);

}  // namespace smb
