// Triangle-mesh rasterisation and the ops built on it: the per-(view, face) pixel rectangles and their 16 x 16 tile bins
// (um_mesh_bin_count, um_mesh_bin), the per-tile start / end table of the sorted bins (um_mesh_ranges), the tile
// rasteriser (um_mesh_raster), the visibility of points in depth maps (um_visible_points) and the per-frame sums of the
// 2D depth metrics (um_depth_metrics).  Semantics and the order of operations: include/unimatch_sm100.h; the numpy
// statement is tests/refops_raster.py.
#include "um_geometry.cuh"

namespace {

constexpr int RASTER_TILE = 16, RASTER_THREADS = RASTER_TILE * RASTER_TILE, RASTER_WARPS = RASTER_THREADS / 32;
static_assert(RASTER_THREADS == COMPACT_THREADS, "the bin passes are compaction passes");
constexpr int METRIC_TERMS = UM_DEPTH_METRIC_TERMS;

struct RasterCam {
  int h, w, tiles_x, tiles_y;
  float fx, fy, cx, cy, near, far;
};

// camera coordinates of point i by the fp32 world-to-camera rows m
__device__ __forceinline__ float3 to_camera(const float* m, const float* __restrict__ p, long long i) {
  return apply_rows(m, make_float3(__ldg(p + 3 * i), __ldg(p + 3 * i + 1), __ldg(p + 3 * i + 2)));
}

// ---- the fp64 pixel rectangle of one (view, face) ----------------------------------------------------------------
struct Rect {
  int x0, x1, y0, y1;
};

__device__ __forceinline__ double dcam(const float* m, int r, double x, double y, double z) {
  return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn((double)m[4 * r], x), __dmul_rn((double)m[4 * r + 1], y)),
                             __dmul_rn((double)m[4 * r + 2], z)),
                   (double)m[4 * r + 3]);
}

struct Bounds {
  double u0, u1, v0, v1;
};

__device__ __forceinline__ void extend(Bounds& b, const RasterCam& cam, double x, double y, double z) {
  const double u = __dadd_rn(__dmul_rn((double)cam.fx, __ddiv_rn(x, z)), (double)cam.cx);
  const double v = __dadd_rn(__dmul_rn((double)cam.fy, __ddiv_rn(y, z)), (double)cam.cy);
  b.u0 = fmin(b.u0, u), b.u1 = fmax(b.u1, u), b.v0 = fmin(b.v0, v), b.v1 = fmax(b.v1, v);
}

// One bound pair to pixels: [floor(lo) - 1, ceil(hi) + 1] clamped to [0, n - 1]; false when that is empty (a NaN too).
__device__ __forceinline__ bool pixel_span(double lo, double hi, int n, int& a, int& b) {
  const double l = __dsub_rn(floor(lo), 1.0), r = __dadd_rn(ceil(hi), 1.0);
  if (!(r >= 0.0 && l <= (double)(n - 1) && l <= r)) return false;
  a = (int)fmax(l, 0.0), b = (int)fmin(r, (double)(n - 1));
  return true;
}

__device__ bool face_rect(const float* __restrict__ p, const int* __restrict__ faces, long long f, const float* m,
                          const RasterCam& cam, Rect& rect) {
  double c[3][3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const long long i = __ldg(faces + 3 * f + k);
    const double x = __ldg(p + 3 * i), y = __ldg(p + 3 * i + 1), z = __ldg(p + 3 * i + 2);
#pragma unroll
    for (int r = 0; r < 3; ++r) c[k][r] = dcam(m, r, x, y, z);
  }
  const double near = cam.near, far = cam.far;
  if (c[0][2] < near && c[1][2] < near && c[2][2] < near) return false;
  if (c[0][2] > far && c[1][2] > far && c[2][2] > far) return false;
  Bounds b = {INFINITY, -INFINITY, INFINITY, -INFINITY};
#pragma unroll
  for (int k = 0; k < 3; ++k) {           // the polygon clipped to z >= near, edge by edge (Sutherland-Hodgman)
    const double* P = c[k];
    const double* Q = c[(k + 1) % 3];
    const bool pin = P[2] >= near, qin = Q[2] >= near;
    if (pin) extend(b, cam, P[0], P[1], P[2]);
    if (pin != qin) {
      const double s = __ddiv_rn(__dsub_rn(near, P[2]), __dsub_rn(Q[2], P[2]));
      extend(b, cam, __dadd_rn(P[0], __dmul_rn(s, __dsub_rn(Q[0], P[0]))),
             __dadd_rn(P[1], __dmul_rn(s, __dsub_rn(Q[1], P[1]))), near);
    }
  }
  return pixel_span(b.u0, b.u1, cam.w, rect.x0, rect.x1) && pixel_span(b.v0, b.v1, cam.h, rect.y0, rect.y1);
}

__device__ __forceinline__ long long rect_tiles(const Rect& r) {
  return (long long)((r.x1 >> 4) - (r.x0 >> 4) + 1) * ((r.y1 >> 4) - (r.y0 >> 4) + 1);
}

__device__ __forceinline__ void load_rows(float* m, const float* __restrict__ w2c, int v) {
  if (threadIdx.x < 12) m[threadIdx.x] = __ldg(w2c + 12LL * v + threadIdx.x);
  __syncthreads();
}

// Pass 1: per block of 256 faces of view blockIdx.y, the number of tile entries their rectangles cover.
__global__ void __launch_bounds__(RASTER_THREADS)
mesh_bin_count_kernel(const float* __restrict__ p, const int* __restrict__ faces, long long T,
                      const float* __restrict__ w2c, RasterCam cam, long long* __restrict__ block_counts) {
  __shared__ float m[12];
  load_rows(m, w2c, blockIdx.y);
  const long long f = (long long)blockIdx.x * RASTER_THREADS + threadIdx.x;
  long long c = 0;
  Rect r;
  if (f < T && face_rect(p, faces, f, m, cam, r)) c = rect_tiles(r);
  long long all;
  block_exclusive_sum(c, &all);
  if (threadIdx.x == 0) block_counts[(long long)blockIdx.y * gridDim.x + blockIdx.x] = all;
}

// Pass 3: each (view, face) writes its entries from offsets[block] + the entries of the block's earlier faces: per
// covered tile (row by row) the key view * tiles + tile and the value face << 16 | the rectangle within the tile.
__global__ void __launch_bounds__(RASTER_THREADS)
mesh_bin_kernel(const float* __restrict__ p, const int* __restrict__ faces, long long T, const float* __restrict__ w2c,
                RasterCam cam, const long long* __restrict__ offsets, long long* __restrict__ keys,
                long long* __restrict__ values) {
  __shared__ float m[12];
  load_rows(m, w2c, blockIdx.y);
  const long long f = (long long)blockIdx.x * RASTER_THREADS + threadIdx.x;
  long long c = 0;
  Rect r;
  if (f < T && face_rect(p, faces, f, m, cam, r)) c = rect_tiles(r);
  long long all;
  const long long before = block_exclusive_sum(c, &all);
  if (c == 0) return;
  long long o = __ldg(offsets + (long long)blockIdx.y * gridDim.x + blockIdx.x) + before;
  const long long view_base = (long long)blockIdx.y * cam.tiles_x * cam.tiles_y;
  for (int ty = r.y0 >> 4; ty <= r.y1 >> 4; ++ty) {
    const int y0 = max(r.y0, 16 * ty) - 16 * ty, y1 = min(r.y1, 16 * ty + 15) - 16 * ty;
    for (int tx = r.x0 >> 4; tx <= r.x1 >> 4; ++tx, ++o) {
      const int x0 = max(r.x0, 16 * tx) - 16 * tx, x1 = min(r.x1, 16 * tx + 15) - 16 * tx;
      keys[o] = view_base + (long long)ty * cam.tiles_x + tx;
      values[o] = (f << 16) | (x0 | x1 << 4 | y0 << 8 | y1 << 12);
    }
  }
}

// One thread per sorted entry: the first and one-past-last position of each run of equal keys into the zeroed tables.
__global__ void __launch_bounds__(RASTER_THREADS)
mesh_ranges_kernel(const long long* __restrict__ keys, long long n, int* __restrict__ start, int* __restrict__ end) {
  const long long i = (long long)blockIdx.x * RASTER_THREADS + threadIdx.x;
  if (i >= n) return;
  mark_run(keys, i, n, __ldg(keys + i), start, end);
}

// ---- the tile rasteriser -----------------------------------------------------------------------------------------
struct __align__(16) StagedFace {
  float c[9];        // the signed canonical cross products of edges AB, BC and CA
  float det;         // A . (signed cross of BC)
  int face, rect;    // face index; in-tile rectangle x0 | x1 << 4 | y0 << 8 | y1 << 12
};

__device__ __forceinline__ float3 cross3(float3 a, float3 b) {
  return make_float3(__fsub_rn(__fmul_rn(a.y, b.z), __fmul_rn(a.z, b.y)),
                     __fsub_rn(__fmul_rn(a.z, b.x), __fmul_rn(a.x, b.z)),
                     __fsub_rn(__fmul_rn(a.x, b.y), __fmul_rn(a.y, b.x)));
}

// The face's edge i -> j: V_lo x V_hi (lo, hi the two vertex indices in ascending order), negated when i > j.
__device__ __forceinline__ void edge_cross(int i, int j, float3 vi, float3 vj, float* out) {
  const float3 c = i <= j ? cross3(vi, vj) : cross3(vj, vi);
  const float s = i <= j ? 1.f : -1.f;
  out[0] = s * c.x, out[1] = s * c.y, out[2] = s * c.z;
}

__device__ __forceinline__ float edge_value(const float* c, float xc, float yc) {
  return __fmaf_rn(c[0], xc, __fmaf_rn(c[1], yc, c[2]));
}

// One CTA per (tile, view), one thread per pixel.  The tile's entries (ascending face index) are staged 256 at a time;
// each thread walks them in order and keeps the least t with a strict <, so ties go to the least face index.
__global__ void __launch_bounds__(RASTER_THREADS)
mesh_raster_kernel(const float* __restrict__ p, const int* __restrict__ faces, const uint8_t* __restrict__ colors,
                   const float* __restrict__ w2c, RasterCam cam, const long long* __restrict__ order,
                   const long long* __restrict__ values, const int* __restrict__ start, const int* __restrict__ end,
                   float* __restrict__ depth, int* __restrict__ face_out, uint8_t* __restrict__ rgb) {
  __shared__ StagedFace staged[RASTER_THREADS];
  __shared__ float m[12];
  const int v = blockIdx.y, tile = blockIdx.x, tid = threadIdx.x;
  const int lx = tid & (RASTER_TILE - 1), ly = tid / RASTER_TILE;
  const int ty = tile / cam.tiles_x, tx = tile - ty * cam.tiles_x;
  const int x = tx * RASTER_TILE + lx, y = ty * RASTER_TILE + ly;
  load_rows(m, w2c, v);
  const long long bin = (long long)v * gridDim.x + tile;
  const int s0 = __ldg(start + bin), s1 = __ldg(end + bin);
  const float xc = __fdiv_rn(__fsub_rn((float)x, cam.cx), cam.fx), yc = __fdiv_rn(__fsub_rn((float)y, cam.cy), cam.fy);
  float best = INFINITY, e_ab = 0.f, e_bc = 0.f, e_ca = 0.f, e_sum = 0.f;
  int best_face = -1;
  for (int base = s0; base < s1; base += RASTER_THREADS) {
    const int n_staged = min(RASTER_THREADS, s1 - base);
    if (tid < n_staged) {
      const long long val = __ldg(values + __ldg(order + base + tid));
      const int f = (int)(val >> 16);
      const int i0 = __ldg(faces + 3LL * f), i1 = __ldg(faces + 3LL * f + 1), i2 = __ldg(faces + 3LL * f + 2);
      const float3 a = to_camera(m, p, i0), b = to_camera(m, p, i1), c = to_camera(m, p, i2);
      StagedFace& s = staged[tid];
      edge_cross(i0, i1, a, b, s.c);
      edge_cross(i1, i2, b, c, s.c + 3);
      edge_cross(i2, i0, c, a, s.c + 6);
      s.det = __fmaf_rn(a.z, s.c[5], __fmaf_rn(a.y, s.c[4], __fmul_rn(a.x, s.c[3])));
      s.face = f;
      s.rect = (int)(val & 0xffff);
    }
    __syncthreads();
    for (int k = 0; k < n_staged; ++k) {
      const StagedFace& s = staged[k];
      const int r = s.rect;
      if (lx < (r & 15) || lx > ((r >> 4) & 15) || ly < ((r >> 8) & 15) || ly > ((r >> 12) & 15)) continue;
      const float e0 = edge_value(s.c, xc, yc), e1 = edge_value(s.c + 3, xc, yc), e2 = edge_value(s.c + 6, xc, yc);
      if (!((e0 >= 0.f && e1 >= 0.f && e2 >= 0.f) || (e0 <= 0.f && e1 <= 0.f && e2 <= 0.f))) continue;
      const float sum = __fadd_rn(__fadd_rn(e0, e1), e2);
      if (sum == 0.f) continue;
      const float t = __fdiv_rn(s.det, sum);
      if (!(isfinite(t) && t >= cam.near && t <= cam.far && t < best)) continue;
      best = t, best_face = s.face, e_ab = e0, e_bc = e1, e_ca = e2, e_sum = sum;
    }
    __syncthreads();
  }
  if (x >= cam.w || y >= cam.h) return;
  const long long pix = ((long long)v * cam.h + y) * cam.w + x;
  depth[pix] = best_face >= 0 ? best : 0.f;
  face_out[pix] = best_face;
  if (!rgb) return;
  uint8_t out[3] = {0, 0, 0};
  if (best_face >= 0) {
    const float ba = __fdiv_rn(e_bc, e_sum), bb = __fdiv_rn(e_ca, e_sum), bc = __fdiv_rn(e_ab, e_sum);
    const long long ia = __ldg(faces + 3LL * best_face), ib = __ldg(faces + 3LL * best_face + 1),
                    ic = __ldg(faces + 3LL * best_face + 2);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const float val = __fmaf_rn(bc, (float)__ldg(colors + 3 * ic + ch),
                                  __fmaf_rn(bb, (float)__ldg(colors + 3 * ib + ch),
                                            __fmul_rn(ba, (float)__ldg(colors + 3 * ia + ch))));
      out[ch] = (uint8_t)min(max(__float2int_rn(val), 0), 255);
    }
  }
  rgb[3 * pix] = out[0], rgb[3 * pix + 1] = out[1], rgb[3 * pix + 2] = out[2];
}

// ---- visibility of points in depth maps ---------------------------------------------------------------------------
// One thread per point, the views in order; stops at the first view that sees it.
__global__ void __launch_bounds__(RASTER_THREADS)
visible_points_kernel(const float* __restrict__ p, long long P, const float* __restrict__ depth, int n, int h, int w,
                      const float* __restrict__ w2c, float fx, float fy, float cx, float cy, float tolerance,
                      uint8_t* __restrict__ visible) {
  const long long i = (long long)blockIdx.x * RASTER_THREADS + threadIdx.x;
  if (i >= P) return;
  const float3 q = make_float3(__ldg(p + 3 * i), __ldg(p + 3 * i + 1), __ldg(p + 3 * i + 2));
  const Pinhole cam = {fx, fy, cx, cy};
  const long long plane = (long long)h * w;
  bool seen = false;
  for (int t = 0; t < n && !seen; ++t) {
    const GlobalRows m = {w2c + 12 * t};
    const float czz = apply_row(m, 2, q);
    if (!(czz > 0.f)) continue;
    float xf, yf;
    if (!nearest_pixel(project(cam, make_float3(apply_row(m, 0, q), apply_row(m, 1, q), czz)), w, h, xf, yf)) continue;
    const float d = __ldg(depth + t * plane + (long long)yf * w + (long long)xf);
    seen = valid_depth(d) && czz <= __fadd_rn(d, tolerance);
  }
  visible[i] = seen ? 1 : 0;
}

// ---- the 2D depth metrics' sums ------------------------------------------------------------------------------------
// One thread per pixel of frame blockIdx.y; per block of 256 pixels the 10 terms summed by a shfl_down tree per warp,
// then the block's warps in order.
__global__ void __launch_bounds__(RASTER_THREADS)
depth_metrics_kernel(const float* __restrict__ pred, const float* __restrict__ gt, long long hw, float max_depth,
                     double* __restrict__ partials) {
  __shared__ double warp_sums[RASTER_WARPS][METRIC_TERMS];
  const long long i = (long long)blockIdx.x * RASTER_THREADS + threadIdx.x;
  const long long at = (long long)blockIdx.y * hw + i;
  const float p = i < hw ? __ldg(pred + at) : 0.f, g = i < hw ? __ldg(gt + at) : 0.f;
  const bool has = valid_depth(p);
  const bool in = has && valid_depth(g) && g < max_depth;
  double term[METRIC_TERMS];
#pragma unroll
  for (int k = 0; k < METRIC_TERMS; ++k) term[k] = 0.0;
  if (in) {
    const double dp = p, dg = g;
    const double d = __dsub_rn(dp, dg), a = fabs(d), d2 = __dmul_rn(d, d);
    const double l = __dsub_rn(log(dp), log(dg));
    const float ratio = fmaxf(__fdiv_rn(g, p), __fdiv_rn(p, g));
    term[0] = 1.0;
    term[1] = a;
    term[2] = __ddiv_rn(a, dg);
    term[3] = __ddiv_rn(d2, dg);
    term[4] = d2;
    term[5] = __dmul_rn(l, l);
    term[6] = ratio < 1.25f ? 1.0 : 0.0;
    term[7] = ratio < 1.5625f ? 1.0 : 0.0;
    term[8] = ratio < 1.953125f ? 1.0 : 0.0;
  }
  term[9] = has ? 1.0 : 0.0;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < METRIC_TERMS; ++k) {
    const double s = warp_sum_ordered(term[k]);
    if (lane == 0) warp_sums[wid][k] = s;
  }
  __syncthreads();
  if (threadIdx.x < METRIC_TERMS) {
    double s = warp_sums[0][threadIdx.x];
#pragma unroll
    for (int q = 1; q < RASTER_WARPS; ++q) s = __dadd_rn(s, warp_sums[q][threadIdx.x]);
    partials[((long long)blockIdx.y * gridDim.x + blockIdx.x) * METRIC_TERMS + threadIdx.x] = s;
  }
}

// One block per frame, warp k sums term k: lane l adds blocks l, l + 32, ... in order from 0, then a shfl_down tree.
__global__ void __launch_bounds__(32 * METRIC_TERMS)
depth_metrics_sum_kernel(const double* __restrict__ partials, long long nb, double* __restrict__ out) {
  const int lane = threadIdx.x & 31, k = threadIdx.x >> 5, f = blockIdx.x;
  const double s = partials_sum_ordered(partials + (long long)f * nb * METRIC_TERMS + k, nb, METRIC_TERMS);
  if (lane == 0) out[(long long)f * METRIC_TERMS + k] = s;
}

RasterCam raster_cam(int h, int w, float fx, float fy, float cx, float cy, float near, float far) {
  RasterCam c;
  c.h = h, c.w = w;
  c.tiles_x = (int)(((long long)w + RASTER_TILE - 1) / RASTER_TILE);
  c.tiles_y = (int)(((long long)h + RASTER_TILE - 1) / RASTER_TILE);
  c.fx = fx, c.fy = fy, c.cx = cx, c.cy = cy, c.near = near, c.far = far;
  return c;
}

}  // namespace

namespace um {

static unsigned face_blocks(long long T) { return (unsigned)((T + RASTER_THREADS - 1) / RASTER_THREADS); }

int mesh_bin_count_launch(const float* points, const int* faces, long long T, const float* w2c, int n, int h, int w,
                          float fx, float fy, float cx, float cy, float near, float far, long long* offsets,
                          cudaStream_t st) {
  const RasterCam cam = raster_cam(h, w, fx, fy, cx, cy, near, far);
  const unsigned fb = face_blocks(T);
  if (fb) {
    mesh_bin_count_kernel<<<dim3(fb, n), RASTER_THREADS, 0, st>>>(points, faces, T, w2c, cam, offsets);
    if (int rc = check_launch("um_mesh_bin_count (count)")) return rc;
  }
  return offsets_scan_launch(offsets, (long long)fb * n, "um_mesh_bin_count (scan)", st);
}

int mesh_bin_launch(const float* points, const int* faces, long long T, const float* w2c, int n, int h, int w, float fx,
                    float fy, float cx, float cy, float near, float far, const long long* offsets, long long* keys,
                    long long* values, cudaStream_t st) {
  const RasterCam cam = raster_cam(h, w, fx, fy, cx, cy, near, far);
  mesh_bin_kernel<<<dim3(face_blocks(T), n), RASTER_THREADS, 0, st>>>(points, faces, T, w2c, cam, offsets, keys, values);
  return check_launch("um_mesh_bin");
}

int mesh_ranges_launch(const long long* sorted_keys, long long total, long long n_bins, int* start, int* end,
                       cudaStream_t st) {
  if (int rc = zero_runs(start, end, n_bins, "um_mesh_ranges", st)) return rc;
  if (total == 0) return UM_OK;
  mesh_ranges_kernel<<<(unsigned)((total + RASTER_THREADS - 1) / RASTER_THREADS), RASTER_THREADS, 0, st>>>(
      sorted_keys, total, start, end);
  return check_launch("um_mesh_ranges");
}

int mesh_raster_launch(const float* points, const int* faces, const uint8_t* colors, const float* w2c, int n, int h,
                       int w, float fx, float fy, float cx, float cy, float near, float far, const long long* order,
                       const long long* values, const int* start, const int* end, float* depth, int* face,
                       uint8_t* rgb, cudaStream_t st) {
  const RasterCam cam = raster_cam(h, w, fx, fy, cx, cy, near, far);
  mesh_raster_kernel<<<dim3((unsigned)cam.tiles_x * cam.tiles_y, n), RASTER_THREADS, 0, st>>>(
      points, faces, colors, w2c, cam, order, values, start, end, depth, face, rgb);
  return check_launch("um_mesh_raster");
}

int visible_points_launch(const float* points, long long P, const float* depth, int n, int h, int w, const float* w2c,
                          float fx, float fy, float cx, float cy, float tolerance, uint8_t* visible, cudaStream_t st) {
  visible_points_kernel<<<(unsigned)((P + RASTER_THREADS - 1) / RASTER_THREADS), RASTER_THREADS, 0, st>>>(
      points, P, depth, n, h, w, w2c, fx, fy, cx, cy, tolerance, visible);
  return check_launch("um_visible_points");
}

int depth_metrics_launch(const float* pred, const float* gt, int n, int h, int w, float max_depth, double* partials,
                         double* out, cudaStream_t st) {
  const long long hw = (long long)h * w, nb = (hw + RASTER_THREADS - 1) / RASTER_THREADS;
  depth_metrics_kernel<<<dim3((unsigned)nb, n), RASTER_THREADS, 0, st>>>(pred, gt, hw, max_depth, partials);
  if (int rc = check_launch("um_depth_metrics (blocks)")) return rc;
  depth_metrics_sum_kernel<<<n, 32 * METRIC_TERMS, 0, st>>>(partials, nb, out);
  return check_launch("um_depth_metrics (frames)");
}

}  // namespace um
