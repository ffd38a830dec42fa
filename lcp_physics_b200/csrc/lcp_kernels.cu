// lcp_kernels.cu -- one instantiation of the forward / backward / JVP kernels.
// Compiled with -DLCP_T=float|double -DLCP_MODE=0|1|2 (see build.py).
#include "lcp_launch.h"

namespace lcpb200 {

template <>
cudaError_t launch_forward_t<LCP_T, LCP_MODE>(const FwdArgs<LCP_T>& a, int grid, cudaStream_t st) {
  lcp_forward_kernel<LCP_T, LCP_MODE><<<grid, a.P.nt, a.P.smem_bytes, st>>>(a);
  return cudaGetLastError();
}

template <>
cudaError_t launch_backward_t<LCP_T, LCP_MODE>(const BwdArgs<LCP_T>& a, int grid, cudaStream_t st) {
  lcp_backward_kernel<LCP_T, LCP_MODE><<<grid, a.P.nt, a.P.smem_bytes, st>>>(a);
  return cudaGetLastError();
}

template <>
cudaError_t launch_jvp_t<LCP_T, LCP_MODE>(const JvpArgs<LCP_T>& a, int grid, cudaStream_t st) {
  lcp_jvp_kernel<LCP_T, LCP_MODE><<<grid, a.P.nt, a.P.smem_bytes, st>>>(a);
  return cudaGetLastError();
}

template <>
cudaError_t configure_t<LCP_T, LCP_MODE>(int nt, int smem_bytes, int dyn_max, int* occ) {
  cudaError_t e;
  // the attribute is per kernel, not per handle: always raise it to the device maximum
  if ((e = cudaFuncSetAttribute(lcp_forward_kernel<LCP_T, LCP_MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn_max)) != cudaSuccess) return e;
  if ((e = cudaFuncSetAttribute(lcp_backward_kernel<LCP_T, LCP_MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn_max)) != cudaSuccess) return e;
  if ((e = cudaFuncSetAttribute(lcp_jvp_kernel<LCP_T, LCP_MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn_max)) != cudaSuccess) return e;
  int of = 0, ob = 0, oj = 0;
  if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&of, lcp_forward_kernel<LCP_T, LCP_MODE>, nt, smem_bytes)) != cudaSuccess) return e;
  if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ob, lcp_backward_kernel<LCP_T, LCP_MODE>, nt, smem_bytes)) != cudaSuccess) return e;
  if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&oj, lcp_jvp_kernel<LCP_T, LCP_MODE>, nt, smem_bytes)) != cudaSuccess) return e;
  *occ = of < ob ? of : ob;
  if (oj < *occ) *occ = oj;      // the JVP runs on the backward's plan and grid
  return cudaSuccess;
}

}  // namespace lcpb200
