// lcp_ray_kernels.cu -- the batched ray cast (lcp_raycast.cuh) and signed distance (lcp_sdf.cuh), fp32 and fp64, in a
// translation unit of their own so that the contact, assembly and solver objects do not change.
#include "lcp_raycast.cuh"
#include "lcp_sdf.cuh"

namespace lcpb200 {
namespace ray {

template <typename T>
cudaError_t launch_raycast(const RayArgs<T>& a, int num_sms, cudaStream_t st) {
  const int nth = a.R >= NT ? NT : (a.R + 31) / 32 * 32;    // one ray per thread; short ray lists use fewer threads
  const int chunks = (a.R + nth - 1) / nth;
  const long long items = (long long)a.B * chunks;
  const long long cap = 16LL * num_sms;
  const int grid = (int)(items < cap ? items : cap);
  raycast_kernel<T><<<grid, nth, 0, st>>>(a, chunks);
  return cudaGetLastError();
}

template cudaError_t launch_raycast<float>(const RayArgs<float>&, int, cudaStream_t);
template cudaError_t launch_raycast<double>(const RayArgs<double>&, int, cudaStream_t);

template <typename T>
cudaError_t launch_sdf(const SdfArgs<T>& a, int num_sms, cudaStream_t st) {
  const int nth = a.Q >= NT ? NT : (a.Q + 31) / 32 * 32;    // one point per thread; short point lists use fewer threads
  const int chunks = (a.Q + nth - 1) / nth;
  const long long items = (long long)a.B * chunks;
  const long long cap = 16LL * num_sms;
  const int grid = (int)(items < cap ? items : cap);
  sdf_kernel<T><<<grid, nth, 0, st>>>(a, chunks);
  return cudaGetLastError();
}

template cudaError_t launch_sdf<float>(const SdfArgs<float>&, int, cudaStream_t);
template cudaError_t launch_sdf<double>(const SdfArgs<double>&, int, cudaStream_t);

}  // namespace ray
}  // namespace lcpb200
