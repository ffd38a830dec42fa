// lcp_band_kernels.cu -- the banded large-scene kernel (lcp_banded.cuh), fp64 only.
#define LCP_BAND_DEVICE
#include "lcp_band_launch.h"

namespace lcpb200 {
namespace bnd {

cudaError_t launch_band_forward(const BArgs& a, int grid, cudaStream_t st) {
  band_forward_kernel<<<grid, NT, a.P.smem_bytes, st>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_band_backward(const BBwdArgs& a, int grid, cudaStream_t st) {
  band_backward_kernel<<<grid, NT, a.P.smem_bytes, st>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_band_jvp(const BJvpArgs& a, int grid, cudaStream_t st) {
  band_jvp_kernel<<<grid, NT, a.P.smem_bytes, st>>>(a);
  return cudaGetLastError();
}

cudaError_t configure_band(int smem_bytes, int dyn_max, int* occ) {
  cudaError_t e;
  if ((e = cudaFuncSetAttribute(band_jvp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn_max)) != cudaSuccess) return e;
  if ((e = cudaFuncSetAttribute(band_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn_max)) != cudaSuccess) return e;
  if ((e = cudaFuncSetAttribute(band_forward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn_max)) != cudaSuccess) return e;
  return cudaOccupancyMaxActiveBlocksPerMultiprocessor(occ, band_forward_kernel, NT, smem_bytes);
}

}  // namespace bnd
}  // namespace lcpb200
