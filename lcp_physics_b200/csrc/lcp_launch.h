// lcp_launch.h -- host-side launch interface between the C ABI (lcpb200.cu) and the kernel
// translation units (lcp_kernels.cu is compiled once per (dtype, residency mode)).
#pragma once
#include <cuda_runtime.h>
#include "lcp_solver.cuh"

namespace lcpb200 {

template <typename T, int MODE> cudaError_t launch_forward_t(const FwdArgs<T>& a, int grid, cudaStream_t st);
template <typename T, int MODE> cudaError_t launch_backward_t(const BwdArgs<T>& a, int grid, cudaStream_t st);
template <typename T, int MODE> cudaError_t launch_jvp_t(const JvpArgs<T>& a, int grid, cudaStream_t st);
// sets the dynamic shared memory limit of the three kernels and returns their min occupancy (CTAs / SM)
template <typename T, int MODE> cudaError_t configure_t(int nt, int smem_bytes, int dyn_max, int* occ);

}  // namespace lcpb200
