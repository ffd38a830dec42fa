// lcp_band_launch.h -- host-side launch interface of the banded large-scene kernel (lcp_band_kernels.cu).
#pragma once
#include <cuda_runtime.h>
#include "lcp_banded.cuh"

namespace lcpb200 {
namespace bnd {

cudaError_t launch_band_forward(const BArgs& a, int grid, cudaStream_t st);
cudaError_t launch_band_backward(const BBwdArgs& a, int grid, cudaStream_t st);
cudaError_t launch_band_jvp(const BJvpArgs& a, int grid, cudaStream_t st);
cudaError_t configure_band(int smem_bytes, int dyn_max, int* occ);

}  // namespace bnd
}  // namespace lcpb200
