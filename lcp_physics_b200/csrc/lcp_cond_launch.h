// lcp_cond_launch.h -- host-side launch interface of the condensed-KKT kernels
// (lcp_cond_kernels.cu is compiled once per (dtype, NS = padded system size / 16)).
#pragma once
#include <cuda_runtime.h>
#include "lcp_condensed.cuh"

namespace lcpb200 {
namespace cnd {

template <typename T, int NS> cudaError_t launch_cond_forward_t(const CFwdArgs<T>& a, int grid, cudaStream_t st);
template <typename T, int NS> cudaError_t launch_cond_backward_t(const CBwdArgs<T>& a, int grid, cudaStream_t st);
template <typename T, int NS> cudaError_t launch_cond_jvp_t(const CJvpArgs<T>& a, int grid, cudaStream_t st);
template <typename T, int NS> cudaError_t configure_cond_t(int smem_bytes, int dyn_max, int* occ);

}  // namespace cnd
}  // namespace lcpb200
