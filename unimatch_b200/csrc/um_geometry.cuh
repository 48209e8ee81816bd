// Building blocks of the reconstruction kernels (um_fusion.cu, um_icp.cu, um_cloud.cu, um_raster.cu, um_consistency.cu):
// stream compaction through an offsets table, the fp32 pinhole camera, the fixed-order fp64 sums and runs of sorted keys.
// Each fixes an order or a format that include/unimatch_sm100.h states once for every op that uses it.
#pragma once
#include "um_common.cuh"

// ---- compaction ---------------------------------------------------------------------------------------------------
// A count op launches a count pass over blocks of COMPACT_THREADS items, then one CTA's ordered exclusive scan of the
// block counts in place (offsets_scan_launch), the total at offsets[nb]; its fill pass writes each item at its block's
// offset plus its slot among the block's items.  The count and fill passes of an op use the same slot helper.
constexpr int COMPACT_THREADS = UM_TSDF_THREADS, COMPACT_WARPS = COMPACT_THREADS / 32;

// Block-wide exclusive sum of one count per thread, in thread order; also returns the block's total.
template <typename T>
__device__ __forceinline__ T block_exclusive_sum(T x, T* total) {
  __shared__ T warp_sums[COMPACT_WARPS];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  T incl = x;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T y = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += y;
  }
  if (lane == 31) warp_sums[wid] = incl;
  __syncthreads();
  T before = 0, all = 0;
#pragma unroll
  for (int q = 0; q < COMPACT_WARPS; ++q) {
    const T s = warp_sums[q];
    before += q < wid ? s : 0;
    all += s;
  }
  *total = all;
  return before + incl - x;
}

// The number of threads before this one in the block whose flag is set; also returns the block's count.
__device__ __forceinline__ int block_rank(bool flag, int* total) {
  __shared__ int warp_counts[COMPACT_WARPS];
  const unsigned ballot = __ballot_sync(0xffffffffu, flag);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) warp_counts[wid] = __popc(ballot);
  __syncthreads();
  int before = __popc(ballot & ((1u << lane) - 1u)), all = 0;
#pragma unroll
  for (int q = 0; q < COMPACT_WARPS; ++q) {
    const int s = warp_counts[q];
    before += q < wid ? s : 0;
    all += s;
  }
  *total = all;
  return before;
}

// ---- runs of sorted keys ------------------------------------------------------------------------------------------
// Position i of n sorted keys, key = keys[i]: the first position of its run into start[key], one past the last into
// end[key].
__device__ __forceinline__ void mark_run(const long long* __restrict__ keys, long long i, long long n, long long key,
                                         int* __restrict__ start, int* __restrict__ end) {
  if (i == 0 || __ldg(keys + i - 1) != key) start[key] = (int)i;
  if (i == n - 1 || __ldg(keys + i + 1) != key) end[key] = (int)(i + 1);
}

// ---- the fp32 pinhole camera --------------------------------------------------------------------------------------
struct Pinhole {
  float fx, fy, cx, cy;
};

__device__ __forceinline__ bool valid_depth(float d) { return isfinite(d) && d > 0.f; }

// Rows read from global memory through the read-only cache.
struct GlobalRows {
  const float* __restrict__ m;
  __device__ __forceinline__ float operator[](int i) const { return __ldg(m + i); }
};

// Row r of the rows m [3, 4] (row-major) applied to p: fma(m[4r+2], z, fma(m[4r+1], y, fma(m[4r], x, m[4r+3]))).
template <class Rows>
__device__ __forceinline__ float apply_row(const Rows& m, int r, float3 p) {
  return __fmaf_rn(m[4 * r + 2], p.z, __fmaf_rn(m[4 * r + 1], p.y, __fmaf_rn(m[4 * r], p.x, m[4 * r + 3])));
}

__device__ __forceinline__ float3 apply_rows(const float* m, float3 p) {
  return make_float3(apply_row(m, 0, p), apply_row(m, 1, p), apply_row(m, 2, p));
}

// The camera point c (c.z > 0) to pixel coordinates (fma(fx, x / z, cx), fma(fy, y / z, cy)).
__device__ __forceinline__ float2 project(const Pinhole& k, float3 c) {
  return make_float2(__fmaf_rn(k.fx, __fdiv_rn(c.x, c.z), k.cx), __fmaf_rn(k.fy, __fdiv_rn(c.y, c.z), k.cy));
}

// Integration's nearest pixel of (u, v): xf = floor(u + 0.5f), yf = floor(v + 0.5f); false unless it lies in the w x h
// frame (a NaN does not).
__device__ __forceinline__ bool nearest_pixel(float2 uv, int w, int h, float& xf, float& yf) {
  const float x = floorf(__fadd_rn(uv.x, 0.5f)), y = floorf(__fadd_rn(uv.y, 0.5f));
  xf = x, yf = y;
  return x >= 0.f && x < (float)w && y >= 0.f && y < (float)h;
}

// Pixel coordinates (u, v) at camera z-depth d -> camera point ((u - cx) / fx * d, (v - cy) / fy * d, d).
__device__ __forceinline__ float3 back_project(const Pinhole& k, float u, float v, float d) {
  return make_float3(__fmul_rn(__fdiv_rn(__fsub_rn(u, k.cx), k.fx), d), __fmul_rn(__fdiv_rn(__fsub_rn(v, k.cy), k.fy), d),
                     d);
}

// ---- fixed-order fp64 sums ----------------------------------------------------------------------------------------
// The warp's sum in lane 0: a shfl_down tree (16, 8, 4, 2, 1).
__device__ __forceinline__ double warp_sum_ordered(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_down_sync(0xffffffffu, v, o));
  return v;
}

// One warp sums the n block partials p[b * stride] in lane 0: lane l adds blocks l, l + 32, ... in order from 0, then
// the shfl_down tree adds the lanes.
__device__ __forceinline__ double partials_sum_ordered(const double* __restrict__ p, long long n, long long stride) {
  double s = 0.0;
  for (long long b = threadIdx.x & 31; b < n; b += 32) s = __dadd_rn(s, __ldg(p + b * stride));
  return warp_sum_ordered(s);
}

namespace um {

// The count ops' scan (um_compact.cu): offsets [nb] block counts -> exclusive offsets, the total at offsets[nb].
int offsets_scan_launch(long long* offsets, long long nb, const char* what, cudaStream_t st);
// Zeroes the start / end tables [n] of a runs kernel.
int zero_runs(int* start, int* end, long long n, const char* what, cudaStream_t st);

}  // namespace um
