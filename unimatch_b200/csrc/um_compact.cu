// The ordered scan of the count ops' block counts (um_tsdf_surface_count, um_tsdf_mesh_count, um_cloud_down_sample_count,
// um_mesh_bin_count, um_depth_points_count) and the zeroed tables of the runs kernels (um_cloud_ranges, um_mesh_ranges).
#include "um_geometry.cuh"

namespace {

// One CTA turns the block counts into exclusive offsets in place, COMPACT_THREADS at a time, in order; the total follows
// them at offsets[nb].
__global__ void __launch_bounds__(COMPACT_THREADS) offsets_scan_kernel(long long* __restrict__ offsets, long long nb) {
  __shared__ long long warp_sums[COMPACT_WARPS];
  __shared__ long long carry;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (long long base = 0; base < nb; base += COMPACT_THREADS) {
    const long long i = base + threadIdx.x;
    const long long x = i < nb ? offsets[i] : 0;
    long long incl = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long y = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += y;
    }
    if (lane == 31) warp_sums[wid] = incl;
    __syncthreads();
    long long before = carry, all = 0;
#pragma unroll
    for (int q = 0; q < COMPACT_WARPS; ++q) {
      before += q < wid ? warp_sums[q] : 0;
      all += warp_sums[q];
    }
    if (i < nb) offsets[i] = before + incl - x;
    __syncthreads();
    if (threadIdx.x == 0) carry += all;
    __syncthreads();
  }
  if (threadIdx.x == 0) offsets[nb] = carry;
}

}  // namespace

namespace um {

int offsets_scan_launch(long long* offsets, long long nb, const char* what, cudaStream_t st) {
  offsets_scan_kernel<<<1, COMPACT_THREADS, 0, st>>>(offsets, nb);
  return check_launch(what);
}

int zero_runs(int* start, int* end, long long n, const char* what, cudaStream_t st) {
  cudaError_t e = cudaMemsetAsync(start, 0, 4 * n, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(end, 0, 4 * n, st);
  if (e != cudaSuccess) {
    set_error("%s: %s", what, cudaGetErrorString(e));
    return UM_ECUDA;
  }
  return UM_OK;
}

}  // namespace um
