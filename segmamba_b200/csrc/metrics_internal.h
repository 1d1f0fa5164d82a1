// Internal interface of the segmentation-metric kernels (metrics.cu) for capi.cu.
#pragma once
#include <cuda_runtime.h>

#include "../../include/segmamba_b200.h"

namespace smb {

cudaError_t metric_bits_launch(const smb_metric_bits_args &a, cudaStream_t st);
cudaError_t metric_count_launch(const smb_metric_count_args &a, cudaStream_t st);
cudaError_t metric_edt_launch(const smb_metric_edt_args &a, cudaStream_t st);
cudaError_t metric_select_launch(const smb_metric_select_args &a, cudaStream_t st);
cudaError_t metric_class_count_launch(const smb_metric_class_count_args &a, cudaStream_t st);
cudaError_t metric_class_edt_launch(const smb_metric_class_edt_args &a, cudaStream_t st);
cudaError_t metric_class_reduce_launch(const smb_metric_class_reduce_args &a, cudaStream_t st);

}  // namespace smb
