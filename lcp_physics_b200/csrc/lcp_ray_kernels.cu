// lcp_ray_kernels.cu -- the batched ray cast (lcp_raycast.cuh), signed distance (lcp_sdf.cuh), body distance
// (lcp_distance.cuh), shape cast (lcp_shapecast.cuh) and time of impact (lcp_toi.cuh), fp32 and fp64, in a
// translation unit of their own so that the contact, assembly and solver objects do not change.
#include "lcp_raycast.cuh"
#include "lcp_sdf.cuh"
#include "lcp_distance.cuh"
#include "lcp_shapecast.cuh"
#include "lcp_toi.cuh"

namespace lcpb200 {
namespace ray {

// Launch shape of n rays, points or body queries in each of B scenes: CTAs of nth threads, one ray or point per thread (short lists
// use fewer threads), each CTA walking (scene, chunk) items; at most 16 CTAs per SM.
struct Shape { int nth, chunks, grid; };

static Shape launch_shape(int B, int n, int num_sms) {
  const int nth = n >= NT ? NT : (n + 31) / 32 * 32;
  const int chunks = (n + nth - 1) / nth;
  const long long items = (long long)B * chunks;
  const long long cap = 16LL * num_sms;
  return {nth, chunks, (int)(items < cap ? items : cap)};
}

template <typename T>
cudaError_t launch_raycast(const RayArgs<T>& a, int num_sms, cudaStream_t st) {
  const Shape s = launch_shape(a.B, a.R, num_sms);
  raycast_kernel<T><<<s.grid, s.nth, 0, st>>>(a, s.chunks);
  return cudaGetLastError();
}

template cudaError_t launch_raycast<float>(const RayArgs<float>&, int, cudaStream_t);
template cudaError_t launch_raycast<double>(const RayArgs<double>&, int, cudaStream_t);

template <typename T>
cudaError_t launch_sdf(const SdfArgs<T>& a, int num_sms, cudaStream_t st) {
  const Shape s = launch_shape(a.B, a.Q, num_sms);
  sdf_kernel<T><<<s.grid, s.nth, 0, st>>>(a, s.chunks);
  return cudaGetLastError();
}

template cudaError_t launch_sdf<float>(const SdfArgs<float>&, int, cudaStream_t);
template cudaError_t launch_sdf<double>(const SdfArgs<double>&, int, cudaStream_t);

template <typename T>
cudaError_t launch_distance(const DistArgs<T>& a, int num_sms, cudaStream_t st) {
  const Shape s = launch_shape(a.B, a.K, num_sms);
  distance_kernel<T><<<s.grid, s.nth, 0, st>>>(a, s.chunks);
  return cudaGetLastError();
}

template cudaError_t launch_distance<float>(const DistArgs<float>&, int, cudaStream_t);
template cudaError_t launch_distance<double>(const DistArgs<double>&, int, cudaStream_t);

template <typename T>
cudaError_t launch_shapecast(const CastArgs<T>& a, int num_sms, cudaStream_t st) {
  const Shape s = launch_shape(a.B, a.K, num_sms);
  shapecast_kernel<T><<<s.grid, s.nth, 0, st>>>(a, s.chunks);
  return cudaGetLastError();
}

template cudaError_t launch_shapecast<float>(const CastArgs<float>&, int, cudaStream_t);
template cudaError_t launch_shapecast<double>(const CastArgs<double>&, int, cudaStream_t);

template <typename T>
cudaError_t launch_toi(const ToiArgs<T>& a, int num_sms, cudaStream_t st) {
  const Shape s = launch_shape(a.B, a.K, num_sms);
  toi_kernel<T><<<s.grid, s.nth, 0, st>>>(a, s.chunks);
  return cudaGetLastError();
}

template cudaError_t launch_toi<float>(const ToiArgs<float>&, int, cudaStream_t);
template cudaError_t launch_toi<double>(const ToiArgs<double>&, int, cudaStream_t);

}  // namespace ray
}  // namespace lcpb200
