// lcp_cond_kernels.cu -- one instantiation of the condensed-KKT kernels (lcp_condensed.cuh).
// Compiled with -DLCP_T=float|double -DLCP_NS=2|3|4|6|8 (see build.py). Every kernel exists twice: without and
// with the per-phase cycle counters (a.prof != nullptr, lcpb200_profile).
#include "lcp_cond_launch.h"

namespace lcpb200 {
namespace cnd {

template <>
cudaError_t launch_cond_forward_t<LCP_T, LCP_NS>(const CFwdArgs<LCP_T>& a, int grid, cudaStream_t st) {
  if (a.prof) cond_forward_kernel<LCP_T, LCP_NS, true><<<grid, NT, a.P.smem_bytes, st>>>(a);
  else cond_forward_kernel<LCP_T, LCP_NS, false><<<grid, NT, a.P.smem_bytes, st>>>(a);
  return cudaGetLastError();
}

template <>
cudaError_t launch_cond_backward_t<LCP_T, LCP_NS>(const CBwdArgs<LCP_T>& a, int grid, cudaStream_t st) {
  if (a.prof) cond_backward_kernel<LCP_T, LCP_NS, true><<<grid, NT, a.P.smem_bytes, st>>>(a);
  else cond_backward_kernel<LCP_T, LCP_NS, false><<<grid, NT, a.P.smem_bytes, st>>>(a);
  return cudaGetLastError();
}

template <>
cudaError_t launch_cond_jvp_t<LCP_T, LCP_NS>(const CJvpArgs<LCP_T>& a, int grid, cudaStream_t st) {
  const bool dense = a.soa.mass == nullptr;
  if (a.prof) {
    if (dense) cond_jvp_kernel<LCP_T, LCP_NS, true, true><<<grid, NT, a.P.smem_bytes, st>>>(a);
    else cond_jvp_kernel<LCP_T, LCP_NS, true, false><<<grid, NT, a.P.smem_bytes, st>>>(a);
  } else {
    if (dense) cond_jvp_kernel<LCP_T, LCP_NS, false, true><<<grid, NT, a.P.smem_bytes, st>>>(a);
    else cond_jvp_kernel<LCP_T, LCP_NS, false, false><<<grid, NT, a.P.smem_bytes, st>>>(a);
  }
  return cudaGetLastError();
}

template <>
cudaError_t configure_cond_t<LCP_T, LCP_NS>(int smem_bytes, int dyn_max, int* occ) {
  cudaError_t e;
  const void* fns[4] = {(const void*)cond_forward_kernel<LCP_T, LCP_NS, false>, (const void*)cond_backward_kernel<LCP_T, LCP_NS, false>,
                        (const void*)cond_forward_kernel<LCP_T, LCP_NS, true>, (const void*)cond_backward_kernel<LCP_T, LCP_NS, true>};
  for (const void* f : fns)
    if ((e = cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn_max)) != cudaSuccess) return e;
  const void* jvp[4] = {(const void*)cond_jvp_kernel<LCP_T, LCP_NS, false, false>, (const void*)cond_jvp_kernel<LCP_T, LCP_NS, true, false>,
                        (const void*)cond_jvp_kernel<LCP_T, LCP_NS, false, true>, (const void*)cond_jvp_kernel<LCP_T, LCP_NS, true, true>};
  for (const void* f : jvp)
    if ((e = cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn_max)) != cudaSuccess) return e;
  // the grid is sized by the production kernels; the profiling ones run on the same grid
  int of = 0, ob = 0;
  if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&of, fns[0], NT, smem_bytes)) != cudaSuccess) return e;
  if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ob, fns[1], NT, smem_bytes)) != cudaSuccess) return e;
  *occ = of < ob ? of : ob;
  return cudaSuccess;
}

}  // namespace cnd
}  // namespace lcpb200
