// lcp_ray_launch.h -- host-side launch interface of the batched ray cast, signed distance, body distance and shape cast
// and time of impact (lcp_ray_kernels.cu, lcp_raycast.cuh, lcp_sdf.cuh, lcp_distance.cuh, lcp_shapecast.cuh, lcp_toi.cuh).
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

// One batch of query points against the bodies of lcpb200_signed_distance, bd as in RayArgs. points [B,Q,2], or [Q,2]
// read by every scene when shared_points != 0; active as in RayArgs; outputs sdf / body / feat [B,Q], normal [B,Q,2]
// or nullptr.
template <typename T>
struct SdfArgs {
  cts::Bodies<T> bd;
  int B, Q;
  T max_dist;
  const T* points;
  int shared_points;
  const uint32_t* active;
  T* sdf;
  int32_t* body;
  int32_t* feat;
  T* normal;
};

template <typename T>
cudaError_t launch_sdf(const SdfArgs<T>& a, int num_sms, cudaStream_t st);

// One batch of body-distance queries of lcpb200_body_distance, bd as in RayArgs. body_a [B,K], or [K] read by every
// scene when shared_queries != 0; body_b likewise for pair mode, nullptr for nearest mode. active as in RayArgs;
// no_contact: nullptr, or the pair bitmask of lcpb200_contacts_active (scene s at no_contact + s nc_stride), read in
// nearest mode only. Outputs dist / body / feat [B,K], normal / point_a [B,K,2].
template <typename T>
struct DistArgs {
  cts::Bodies<T> bd;
  int B, K;
  T max_dist;
  const int32_t* body_a;
  const int32_t* body_b;
  int shared_queries;
  const uint32_t* active;
  const uint32_t* no_contact;
  long long nc_stride;
  T* dist;
  int32_t* body;
  int32_t* feat;
  T* normal;
  T* point_a;
};

template <typename T>
cudaError_t launch_distance(const DistArgs<T>& a, int num_sms, cudaStream_t st);

// One batch of shape casts or sweeps of lcpb200_shapecast, bd as in RayArgs. dir [B,K,2] (unit length). Disk mode
// (body_q == nullptr): origin [B,K,2], radius [B,K] and max_dist are read. Body mode: body_q [B,K] and limit [B,K] are
// read, and no_contact as in DistArgs. active as in RayArgs. Outputs dist / body / feat [B,K], normal / point [B,K,2].
template <typename T>
struct CastArgs {
  cts::Bodies<T> bd;
  int B, K;
  T max_dist;
  const T* origin;
  const T* radius;
  const int32_t* body_q;
  const T* dir;
  const T* limit;
  const uint32_t* active;
  const uint32_t* no_contact;
  long long nc_stride;
  T* dist;
  int32_t* body;
  int32_t* feat;
  T* normal;
  T* point;
};

template <typename T>
cudaError_t launch_shapecast(const CastArgs<T>& a, int num_sms, cudaStream_t st);

// One batch of time-of-impact queries of lcpb200_time_of_impact, bd as in RayArgs plus pcen [B,np,2], the polygons'
// centres. motion [B,nb+np,3] (dth, dx, dy). body_a / body_b / shared_queries as in DistArgs (body_b nullptr: first
// mode); active and no_contact (first mode only) as in DistArgs. Outputs frac / body / feat / dist [B,K], normal /
// point_a [B,K,2].
template <typename T>
struct ToiArgs {
  cts::Bodies<T> bd;
  int B, K;
  T gap, skip, tol;
  const T* motion;
  const int32_t* body_a;
  const int32_t* body_b;
  int shared_queries;
  const uint32_t* active;
  const uint32_t* no_contact;
  long long nc_stride;
  T* frac;
  int32_t* body;
  int32_t* feat;
  T* dist;
  T* normal;
  T* point_a;
};

template <typename T>
cudaError_t launch_toi(const ToiArgs<T>& a, int num_sms, cudaStream_t st);

}  // namespace ray
}  // namespace lcpb200
