// Multi-view geometric consistency of depth maps (um_depth_consistency) and the export of valid depths as coloured world
// points (um_depth_points_count, um_depth_points).  Semantics and the order of operations: include/unimatch_sm100.h; the
// numpy statement is tests/refops_consistency.py.
#include "um_geometry.cuh"

namespace {

constexpr int CONS_THREADS = COMPACT_THREADS;

__device__ __forceinline__ void load_rows(float* dst, const float* __restrict__ rows, int i) {
#pragma unroll
  for (int k = 0; k < 12; ++k) dst[k] = __ldg(rows + 12LL * i + k);
}

// One thread per pixel of reference blockIdx.y; sources in table order.
__global__ void __launch_bounds__(CONS_THREADS)
depth_consistency_kernel(const float* __restrict__ depth, int N, int H, int W, Pinhole k, const float* __restrict__ c2w,
                         const float* __restrict__ w2c, const int* __restrict__ refs, const int* __restrict__ src, int S,
                         float max_pixel, float max_relative, int min_views, uint8_t* __restrict__ views,
                         float* __restrict__ out) {
  const long long hw = (long long)H * W;
  const long long pix = (long long)blockIdx.x * CONS_THREADS + threadIdx.x;
  if (pix >= hw) return;
  const int ri = blockIdx.y;
  const int x = (int)(pix % W), y = (int)(pix / W);
  const int r = __ldg(refs + ri);
  const bool ref_ok = r >= 0 && r < N;
  const float d = ref_ok ? __ldg(depth + r * hw + pix) : 0.f;
  int count = 0;
  if (ref_ok && valid_depth(d)) {
    float c2w_r[12], w2c_r[12];
    load_rows(c2w_r, c2w, r);
    load_rows(w2c_r, w2c, r);
    const float xf = (float)x, yf = (float)y;
    const float3 world = apply_rows(c2w_r, back_project(k, xf, yf, d));
    for (int j = 0; j < S; ++j) {
      const int s = __ldg(src + (long long)ri * S + j);
      if (s < 0 || s >= N) continue;
      float m[12];
      load_rows(m, w2c, s);
      const float3 c = apply_rows(m, world);
      if (!(c.z > 0.f)) continue;
      const float2 uv = project(k, c);
      const float u = uv.x, v = uv.y;
      if (!(u >= 0.f && u <= (float)(W - 1) && v >= 0.f && v <= (float)(H - 1))) continue;
      const float fx0 = floorf(u), fy0 = floorf(v);
      const int x0 = (int)fx0, y0 = (int)fy0, x1 = min(x0 + 1, W - 1), y1 = min(y0 + 1, H - 1);
      const float* plane = depth + s * hw;
      const float d00 = __ldg(plane + (long long)y0 * W + x0), d01 = __ldg(plane + (long long)y0 * W + x1);
      const float d10 = __ldg(plane + (long long)y1 * W + x0), d11 = __ldg(plane + (long long)y1 * W + x1);
      if (!(valid_depth(d00) && valid_depth(d01) && valid_depth(d10) && valid_depth(d11))) continue;
      const float ax = __fsub_rn(u, fx0), ay = __fsub_rn(v, fy0);
      const float top = __fmaf_rn(ax, __fsub_rn(d01, d00), d00), bot = __fmaf_rn(ax, __fsub_rn(d11, d10), d10);
      const float ds = __fmaf_rn(ay, __fsub_rn(bot, top), top);
      load_rows(m, c2w, s);
      const float3 back = apply_rows(w2c_r, apply_rows(m, back_project(k, u, v, ds)));
      if (!(back.z > 0.f)) continue;
      const float2 uv2 = project(k, back);
      const float dx = __fsub_rn(uv2.x, xf), dy = __fsub_rn(uv2.y, yf);
      const float err = __fsqrt_rn(__fmaf_rn(dy, dy, __fmul_rn(dx, dx)));
      const float rel = __fdiv_rn(fabsf(__fsub_rn(back.z, d)), d);
      if (err < max_pixel && rel < max_relative) ++count;
    }
  }
  const long long o = (long long)ri * hw + pix;
  views[o] = (uint8_t)count;
  out[o] = count >= min_views ? d : 0.f;
}

// Pass 1: per block of 256 pixels (frame-major, then row-major), the number of valid depths.
__global__ void __launch_bounds__(CONS_THREADS)
depth_points_count_kernel(const float* __restrict__ depth, long long total, long long* __restrict__ block_counts) {
  const long long i = (long long)blockIdx.x * CONS_THREADS + threadIdx.x;
  int all;
  block_rank(i < total && valid_depth(__ldg(depth + i)), &all);
  if (threadIdx.x == 0) block_counts[blockIdx.x] = all;
}

// Pass 3: each valid depth writes its world point and colour at offsets[block] + the valid depths before it in the block.
__global__ void __launch_bounds__(CONS_THREADS)
depth_points_kernel(const float* __restrict__ depth, const uint8_t* __restrict__ frames, int H, int W, Pinhole k,
                    const float* __restrict__ c2w, long long total, const long long* __restrict__ offsets,
                    float* __restrict__ points, uint8_t* __restrict__ colors) {
  const long long i = (long long)blockIdx.x * CONS_THREADS + threadIdx.x;
  const float d = i < total ? __ldg(depth + i) : 0.f;
  const bool ok = valid_depth(d);
  int all;
  const int before = block_rank(ok, &all);
  if (!ok) return;
  const long long o = __ldg(offsets + blockIdx.x) + before;
  const long long hw = (long long)H * W;
  const int t = (int)(i / hw);
  const long long pix = i - t * hw;
  const int x = (int)(pix % W), y = (int)(pix / W);
  float m[12];
  load_rows(m, c2w, t);
  const float3 p = apply_rows(m, back_project(k, (float)x, (float)y, d));
  points[3 * o] = p.x, points[3 * o + 1] = p.y, points[3 * o + 2] = p.z;
  colors[3 * o] = __ldg(frames + 3 * i), colors[3 * o + 1] = __ldg(frames + 3 * i + 1);
  colors[3 * o + 2] = __ldg(frames + 3 * i + 2);
}

}  // namespace

namespace um {

static unsigned pixel_blocks(long long n) { return (unsigned)((n + CONS_THREADS - 1) / CONS_THREADS); }

int depth_consistency_launch(const float* depth, int N, int H, int W, float fx, float fy, float cx, float cy,
                             const float* c2w, const float* w2c, const int* refs, int R, const int* src, int S,
                             float max_pixel, float max_relative, int min_views, uint8_t* views, float* out,
                             cudaStream_t st) {
  const Pinhole k = {fx, fy, cx, cy};
  depth_consistency_kernel<<<dim3(pixel_blocks((long long)H * W), R), CONS_THREADS, 0, st>>>(
      depth, N, H, W, k, c2w, w2c, refs, src, S, max_pixel, max_relative, min_views, views, out);
  return check_launch("um_depth_consistency");
}

int depth_points_count_launch(const float* depth, long long total, long long* offsets, cudaStream_t st) {
  const unsigned nb = pixel_blocks(total);
  depth_points_count_kernel<<<nb, CONS_THREADS, 0, st>>>(depth, total, offsets);
  if (int rc = check_launch("um_depth_points_count (count)")) return rc;
  return offsets_scan_launch(offsets, nb, "um_depth_points_count (scan)", st);
}

int depth_points_launch(const float* depth, const uint8_t* frames, int N, int H, int W, float fx, float fy, float cx,
                        float cy, const float* c2w, const long long* offsets, float* points, uint8_t* colors,
                        cudaStream_t st) {
  const Pinhole k = {fx, fy, cx, cy};
  const long long total = (long long)N * H * W;
  depth_points_kernel<<<pixel_blocks(total), CONS_THREADS, 0, st>>>(depth, frames, H, W, k, c2w, total, offsets, points,
                                                                     colors);
  return check_launch("um_depth_points");
}

}  // namespace um
