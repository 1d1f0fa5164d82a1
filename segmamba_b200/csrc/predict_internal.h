// Internal interface of the case-prediction kernels (predict.cu) for capi.cu.
#pragma once
#include <cuda_runtime.h>

#include "../../include/segmamba_b200.h"

namespace smb {

cudaError_t pred_restore_launch(const smb_pred_restore_args &a, cudaStream_t st);
size_t pred_cc_workspace_bytes(int batch, int d, int h, int w);
cudaError_t pred_cc_launch(const smb_pred_cc_args &a, cudaStream_t st);

}  // namespace smb
