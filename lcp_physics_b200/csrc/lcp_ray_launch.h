// lcp_ray_launch.h -- host-side launch interface of the batched ray cast (lcp_ray_kernels.cu, lcp_raycast.cuh).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "lcp_contacts.cuh"

namespace lcpb200 {
namespace ray {

// One batch of rays against the bodies of lcpb200_raycast. bd: pos / rad (circles), pverts (dynamic polygons) and overts
// (obstacles), in the layout of cts::Bodies (the material and centroid pointers are not read). origin / dir [B,R,2]
// (dir of unit length), active [B, ceil(nt / 32)] or nullptr; outputs t / body / feat [B,R], normal [B,R,2] or nullptr.
template <typename T>
struct RayArgs {
  cts::Bodies<T> bd;
  int B, R;
  T max_dist;
  const T* origin;
  const T* dir;
  const uint32_t* active;
  T* t;
  int32_t* body;
  int32_t* feat;
  T* normal;
};

template <typename T>
cudaError_t launch_raycast(const RayArgs<T>& a, int num_sms, cudaStream_t st);

}  // namespace ray
}  // namespace lcpb200
