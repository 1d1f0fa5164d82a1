// Internal interface of the case-preprocessing kernels (preprocess.cu) for capi.cu.
#pragma once
#include <cuda_runtime.h>

#include "../../include/segmamba_b200.h"

namespace smb {

cudaError_t prep_mask_launch(const smb_prep_mask_args &a, cudaStream_t st);
cudaError_t prep_crop_launch(const smb_prep_crop_args &a, cudaStream_t st);
cudaError_t prep_normalize_launch(const smb_prep_norm_job *jobs, int n, cudaStream_t st);
cudaError_t prep_ct_normalize_launch(const smb_prep_ct_norm_job *jobs, int n, cudaStream_t st);
cudaError_t prep_label_resize_launch(const smb_prep_label_resize_args &a, cudaStream_t st);
cudaError_t prep_count_launch(const smb_prep_compact_job *jobs, int n, cudaStream_t st);
cudaError_t prep_compact_launch(const smb_prep_compact_job *jobs, int n, cudaStream_t st);
cudaError_t prep_gather_launch(const smb_prep_gather_args &a, cudaStream_t st);

}  // namespace smb
