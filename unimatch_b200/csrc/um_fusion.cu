// TSDF fusion of posed depth maps into a dense voxel volume (um_tsdf_integrate), the zero-crossing points of the fused
// surface (um_tsdf_surface_count, um_tsdf_surface_points), its marching-cubes mesh (um_tsdf_mesh_count, um_tsdf_mesh)
// and its ray-cast depth, colour and normal images (um_tsdf_raycast).
// Semantics and the fp32 order of operations: include/unimatch_sm100.h; the float32 and float64 statements are
// tests/refops_fusion.py, tests/refops_mesh.py and tests/refops_render.py.
#include "um_geometry.cuh"
#include "um_mc_table.cuh"

namespace {

constexpr int FUSE_THREADS = COMPACT_THREADS;

struct Volume {
  int X, Y, Z;
  float ox, oy, oz, vs;
};

__device__ __forceinline__ float centre(int idx, float voxel_size, float origin) {
  return __fmaf_rn(__fadd_rn((float)idx, 0.5f), voxel_size, origin);
}

// One thread per voxel, x fastest.  The voxel's state is read at its first update and written once after its last, so a
// voxel no frame reaches moves no state bytes; the frames are walked in order, so the result does not depend on how a
// sequence is split into launches.
__global__ void __launch_bounds__(FUSE_THREADS)
tsdf_integrate_kernel(float* __restrict__ tsdf, float* __restrict__ weight, float* __restrict__ color, Volume vol,
                      float trunc, const float* __restrict__ depth, const uint8_t* __restrict__ frames,
                      const float* __restrict__ w2c, int n, int h, int w, float fx, float fy, float cx, float cy,
                      const int* __restrict__ n_valid) {
  const long long total = (long long)vol.X * vol.Y * vol.Z;
  const long long i = (long long)blockIdx.x * FUSE_THREADS + threadIdx.x;
  if (i >= total) return;
  const int nv = min(max(__ldg(n_valid), 0), n);
  if (nv == 0) return;
  const int xy = vol.X * vol.Y;
  const int k = (int)(i / xy), r = (int)(i - (long long)k * xy);
  const int j = r / vol.X, ii = r - j * vol.X;
  const float3 p = make_float3(centre(ii, vol.vs, vol.ox), centre(j, vol.vs, vol.oy), centre(k, vol.vs, vol.oz));
  const Pinhole cam = {fx, fy, cx, cy};
  const long long plane = (long long)h * w;
  bool loaded = false;
  float F = 0.f, Wt = 0.f, R = 0.f, G = 0.f, B = 0.f;
  for (int t = 0; t < nv; ++t) {
    const GlobalRows m = {w2c + 12 * t};
    const float czz = apply_row(m, 2, p);
    if (!(czz > 0.f)) continue;
    float xf, yf;
    if (!nearest_pixel(project(cam, make_float3(apply_row(m, 0, p), apply_row(m, 1, p), czz)), w, h, xf, yf)) continue;
    const long long pix = (long long)yf * w + (long long)xf;
    const float d = __ldg(depth + t * plane + pix);
    if (!valid_depth(d)) continue;
    const float sdf = __fsub_rn(d, czz);
    if (sdf < -trunc) continue;
    const float f = fminf(1.f, __fdiv_rn(sdf, trunc));
    if (!loaded) {
      F = tsdf[i], Wt = weight[i];
      R = color[i], G = color[total + i], B = color[2 * total + i];
      loaded = true;
    }
    const uint8_t* rgb = frames + 3 * (t * plane + pix);
    const float w1 = __fadd_rn(Wt, 1.f);
    F = __fdiv_rn(__fmaf_rn(F, Wt, f), w1);
    R = __fdiv_rn(__fmaf_rn(R, Wt, (float)__ldg(rgb)), w1);
    G = __fdiv_rn(__fmaf_rn(G, Wt, (float)__ldg(rgb + 1)), w1);
    B = __fdiv_rn(__fmaf_rn(B, Wt, (float)__ldg(rgb + 2)), w1);
    Wt = w1;
  }
  if (loaded) {
    tsdf[i] = F, weight[i] = Wt;
    color[i] = R, color[total + i] = G, color[2 * total + i] = B;
  }
}

// The zero crossing on the edge from voxel i to its neighbour at +1 along `axis` (step voxels away in the layout), if both
// have been observed and their TSDF signs differ: s = F0 / (F0 - F1) along the edge.
struct Crossing {
  bool hit;
  float s;
};

__device__ __forceinline__ Crossing crossing(const float* __restrict__ tsdf, const float* __restrict__ weight, long long i,
                                             long long step, float F0, float W0) {
  const float W1 = __ldg(weight + i + step);
  const float F1 = __ldg(tsdf + i + step);
  if (!(W0 > 0.f && W1 > 0.f) || (F0 < 0.f) == (F1 < 0.f)) return {false, 0.f};
  return {true, __fdiv_rn(F0, __fsub_rn(F0, F1))};
}

struct VoxelEdges {
  int ii, j, k;
  float F0, W0;
  Crossing e[3];               // +x, +y, +z
  __device__ int count() const { return (int)e[0].hit + (int)e[1].hit + (int)e[2].hit; }
};

__device__ __forceinline__ VoxelEdges voxel_edges(const float* __restrict__ tsdf, const float* __restrict__ weight,
                                                  const Volume& vol, long long i) {
  VoxelEdges v;
  const int xy = vol.X * vol.Y;
  v.k = (int)(i / xy);
  const int r = (int)(i - (long long)v.k * xy);
  v.j = r / vol.X, v.ii = r - v.j * vol.X;
  v.F0 = __ldg(tsdf + i), v.W0 = __ldg(weight + i);
  const Crossing none = {false, 0.f};
  v.e[0] = v.ii + 1 < vol.X ? crossing(tsdf, weight, i, 1, v.F0, v.W0) : none;
  v.e[1] = v.j + 1 < vol.Y ? crossing(tsdf, weight, i, vol.X, v.F0, v.W0) : none;
  v.e[2] = v.k + 1 < vol.Z ? crossing(tsdf, weight, i, xy, v.F0, v.W0) : none;
  return v;
}

// Pass 1: the number of points each block of FUSE_THREADS voxels emits.
__global__ void __launch_bounds__(FUSE_THREADS)
tsdf_count_kernel(const float* __restrict__ tsdf, const float* __restrict__ weight, Volume vol, long long total,
                  long long* __restrict__ block_counts) {
  const long long i = (long long)blockIdx.x * FUSE_THREADS + threadIdx.x;
  const int c = i < total ? voxel_edges(tsdf, weight, vol, i).count() : 0;
  int all;
  block_exclusive_sum(c, &all);
  if (threadIdx.x == 0) block_counts[blockIdx.x] = all;
}

// The gradient of F at voxel i (value F) along one axis, step voxels away in the layout: the central difference when both
// neighbours are inside the grid (has_lo, has_hi) and observed, else the one-sided difference to the one that is, else 0.
__device__ __forceinline__ float gradient(const float* __restrict__ tsdf, const float* __restrict__ weight, long long i,
                                          long long step, bool has_lo, bool has_hi, float F) {
  const bool lo = has_lo && __ldg(weight + i - step) > 0.f;
  const bool hi = has_hi && __ldg(weight + i + step) > 0.f;
  const float Fm = lo ? __ldg(tsdf + i - step) : 0.f, Fp = hi ? __ldg(tsdf + i + step) : 0.f;
  if (lo && hi) return __fmul_rn(__fsub_rn(Fp, Fm), 0.5f);
  if (hi) return __fsub_rn(Fp, F);
  if (lo) return __fsub_rn(F, Fm);
  return 0.f;
}

__device__ __forceinline__ void voxel_gradient(const float* __restrict__ tsdf, const float* __restrict__ weight,
                                               const Volume& vol, long long i, int ii, int j, int k, float g[3]) {
  const float F = __ldg(tsdf + i);
  g[0] = gradient(tsdf, weight, i, 1, ii > 0, ii + 1 < vol.X, F);
  g[1] = gradient(tsdf, weight, i, vol.X, j > 0, j + 1 < vol.Y, F);
  g[2] = gradient(tsdf, weight, i, (long long)vol.X * vol.Y, k > 0, k + 1 < vol.Z, F);
}

// Every voxel writes its points at its block's offset plus the points of the voxels before it in the block.  kMesh also
// writes each point's normal and the voxel's first point index (read by the face pass).
template <bool kMesh>
__device__ __forceinline__ void surface_points(const float* __restrict__ tsdf, const float* __restrict__ weight,
                                               const float* __restrict__ color, const Volume& vol, long long total,
                                               const long long* __restrict__ offsets, float* __restrict__ points,
                                               uint8_t* __restrict__ colors, float* __restrict__ normals,
                                               int* __restrict__ first_vertex) {
  const long long i = (long long)blockIdx.x * FUSE_THREADS + threadIdx.x;
  VoxelEdges v;
  int c = 0;
  if (i < total) {
    v = voxel_edges(tsdf, weight, vol, i);
    c = v.count();
  }
  int all;
  const int before = block_exclusive_sum(c, &all);
  if (c == 0) return;
  long long o = __ldg(offsets + blockIdx.x) + before;
  const float p0[3] = {centre(v.ii, vol.vs, vol.ox), centre(v.j, vol.vs, vol.oy), centre(v.k, vol.vs, vol.oz)};
  const long long steps[3] = {1, vol.X, (long long)vol.X * vol.Y};
  float c0[3];
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) c0[ch] = __ldg(color + ch * total + i);
  float g0[3];
  if constexpr (kMesh) {
    first_vertex[i] = (int)o;
    voxel_gradient(tsdf, weight, vol, i, v.ii, v.j, v.k, g0);
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    if (!v.e[a].hit) continue;
    const float s = v.e[a].s;
#pragma unroll
    for (int q = 0; q < 3; ++q) points[3 * o + q] = q == a ? __fmaf_rn(s, vol.vs, p0[q]) : p0[q];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const float c1 = __ldg(color + ch * total + i + steps[a]);
      const int q = __float2int_rn(__fmaf_rn(s, __fsub_rn(c1, c0[ch]), c0[ch]));
      colors[3 * o + ch] = (uint8_t)min(max(q, 0), 255);
    }
    if constexpr (kMesh) {
      float g1[3], n[3];
      voxel_gradient(tsdf, weight, vol, i + steps[a], v.ii + (a == 0), v.j + (a == 1), v.k + (a == 2), g1);
#pragma unroll
      for (int q = 0; q < 3; ++q) n[q] = __fmaf_rn(s, __fsub_rn(g1[q], g0[q]), g0[q]);
      const float len = __fsqrt_rn(__fmaf_rn(n[2], n[2], __fmaf_rn(n[1], n[1], __fmul_rn(n[0], n[0]))));
#pragma unroll
      for (int q = 0; q < 3; ++q) normals[3 * o + q] = len == 0.f ? 0.f : __fdiv_rn(n[q], len);
    }
    ++o;
  }
}

// Pass 3 of the point extraction.
__global__ void __launch_bounds__(FUSE_THREADS)
tsdf_points_kernel(const float* __restrict__ tsdf, const float* __restrict__ weight, const float* __restrict__ color,
                   Volume vol, long long total, const long long* __restrict__ offsets, float* __restrict__ points,
                   uint8_t* __restrict__ colors) {
  surface_points<false>(tsdf, weight, color, vol, total, offsets, points, colors, nullptr, nullptr);
}

// The mesh's vertex pass: the points of tsdf_points_kernel with their normals and each voxel's first point.
__global__ void __launch_bounds__(FUSE_THREADS)
tsdf_mesh_vertices_kernel(const float* __restrict__ tsdf, const float* __restrict__ weight, const float* __restrict__ color,
                          Volume vol, long long total, const long long* __restrict__ offsets, float* __restrict__ points,
                          uint8_t* __restrict__ colors, float* __restrict__ normals, int* __restrict__ first_vertex) {
  surface_points<true>(tsdf, weight, color, vol, total, offsets, points, colors, normals, first_vertex);
}

// The case-table entry of the cube whose low corner is voxel i = (ii, j, k): 0 unless the cube lies inside the grid and
// all 8 corners are observed; corner c = bx + 2 by + 4 bz sets bit c of the configuration when its F < 0.
__device__ __forceinline__ unsigned long long cube_case(const float* __restrict__ tsdf, const float* __restrict__ weight,
                                                        const Volume& vol, long long i, int ii, int j, int k) {
  if (!(ii + 1 < vol.X && j + 1 < vol.Y && k + 1 < vol.Z)) return 0ull;
  const long long xy = (long long)vol.X * vol.Y;
  int cfg = 0;
  bool seen = true;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const long long at = i + (c & 1) + ((c >> 1) & 1) * (long long)vol.X + (c >> 2) * xy;
    seen &= __ldg(weight + at) > 0.f;
    cfg |= (__ldg(tsdf + at) < 0.f) << c;
  }
  return seen ? __ldg(um_mc_table + cfg) : 0ull;
}

struct Coords {
  int ii, j, k;
};

__device__ __forceinline__ Coords voxel_coords(const Volume& vol, long long i) {
  const int xy = vol.X * vol.Y;
  const int k = (int)(i / xy), r = (int)(i - (long long)k * xy);
  const int j = r / vol.X;
  return {r - j * vol.X, j, k};
}

// Mesh pass 1: the number of triangles of each block's cubes.
__global__ void __launch_bounds__(FUSE_THREADS)
tsdf_mesh_count_kernel(const float* __restrict__ tsdf, const float* __restrict__ weight, Volume vol, long long total,
                       long long* __restrict__ block_counts) {
  const long long i = (long long)blockIdx.x * FUSE_THREADS + threadIdx.x;
  int n = 0;
  if (i < total) {
    const Coords c = voxel_coords(vol, i);
    n = (int)(cube_case(tsdf, weight, vol, i, c.ii, c.j, c.k) >> 60);
  }
  int all;
  block_exclusive_sum(n, &all);
  if (threadIdx.x == 0) block_counts[blockIdx.x] = all;
}

// The point on edge e of the cube at voxel i = (ii, j, k): edge e = 4 axis + b0 + 2 b1 is the `axis` edge of the voxel
// offset by b0, b1 on the other two axes, whose points come in axis order from its first one.
__device__ __forceinline__ int edge_vertex(const float* __restrict__ tsdf, const float* __restrict__ weight,
                                           const int* __restrict__ first_vertex, const Volume& vol, long long i, int ii,
                                           int j, int k, int e) {
  const int axis = e >> 2, b0 = e & 1, b1 = (e >> 1) & 1;
  const int dx = axis == 0 ? 0 : b0, dy = axis == 0 ? b0 : axis == 1 ? 0 : b1, dz = axis == 2 ? 0 : b1;
  const long long owner = i + dx + (long long)dy * vol.X + (long long)dz * vol.X * vol.Y;
  int idx = __ldg(first_vertex + owner);
  const float F0 = __ldg(tsdf + owner), W0 = __ldg(weight + owner);
  if (axis > 0 && ii + dx + 1 < vol.X) idx += crossing(tsdf, weight, owner, 1, F0, W0).hit;
  if (axis > 1 && j + dy + 1 < vol.Y) idx += crossing(tsdf, weight, owner, vol.X, F0, W0).hit;
  return idx;
}

// Mesh pass 2: every cube writes its triangles at its block's offset plus the triangles of the cubes before it.
__global__ void __launch_bounds__(FUSE_THREADS)
tsdf_faces_kernel(const float* __restrict__ tsdf, const float* __restrict__ weight, Volume vol, long long total,
                  const long long* __restrict__ offsets, const int* __restrict__ first_vertex, int* __restrict__ faces) {
  const long long i = (long long)blockIdx.x * FUSE_THREADS + threadIdx.x;
  Coords c = {0, 0, 0};
  unsigned long long cs = 0ull;
  if (i < total) {
    c = voxel_coords(vol, i);
    cs = cube_case(tsdf, weight, vol, i, c.ii, c.j, c.k);
  }
  const int n = (int)(cs >> 60);
  int all;
  const int before = block_exclusive_sum(n, &all);
  if (n == 0) return;
  long long o = __ldg(offsets + blockIdx.x) + before;
  for (int t = 0; t < n; ++t, ++o) {
#pragma unroll
    for (int q = 0; q < 3; ++q)
      faces[3 * o + q] = edge_vertex(tsdf, weight, first_vertex, vol, i, c.ii, c.j, c.k, (int)(cs >> (12 * t + 4 * q)) & 15);
  }
}

// ---- ray casting --------------------------------------------------------------------------------------------------------
constexpr int RAY_TX = 16, RAY_TY = 8;          // a 2-D pixel tile per block: neighbouring rays read the same cache lines

// A ray in grid coordinates: g(t) = fma(t, gd, go) per axis, where g = (p - origin) / voxel_size - 0.5 puts voxel centres
// on the integers.
struct Ray {
  float gd[3], go[3];
};

// The trilinear cell of the sample at t: its low corner's linear index and the fractions along x, y, z.
struct Cell {
  long long base;
  float f[3];
};

__device__ __forceinline__ Cell ray_cell(const Ray& r, const Volume& vol, float t) {
  const int dims[3] = {vol.X, vol.Y, vol.Z};
  int idx[3];
  Cell c;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float g = __fmaf_rn(t, r.gd[a], r.go[a]);
    idx[a] = min(max((int)floorf(g), 0), dims[a] - 2);
    c.f[a] = __fsub_rn(g, (float)idx[a]);
  }
  c.base = ((long long)idx[2] * vol.Y + idx[1]) * vol.X + idx[0];
  return c;
}

__device__ __forceinline__ float lerp(float f, float a, float b) { return __fmaf_rn(f, __fsub_rn(b, a), a); }

// Trilinear interpolation of the 8 corner values v[c] (corner c = bx + 2 by + 4 bz): x, then y, then z.
__device__ __forceinline__ float trilinear(const float v[8], const float f[3]) {
  const float x00 = lerp(f[0], v[0], v[1]), x10 = lerp(f[0], v[2], v[3]);
  const float x01 = lerp(f[0], v[4], v[5]), x11 = lerp(f[0], v[6], v[7]);
  return lerp(f[2], lerp(f[1], x00, x10), lerp(f[1], x01, x11));
}

__device__ __forceinline__ long long corner(const Volume& vol, long long base, int c) {
  return base + (c & 1) + ((c >> 1) & 1) * (long long)vol.X + (long long)(c >> 2) * vol.X * vol.Y;
}

// The sample at t: known iff all 8 corner weights are > 0 (the TSDF values are loaded only then), F the trilinear TSDF.
struct Sample {
  bool known;
  float F;
};

__device__ __forceinline__ Sample ray_sample(const float* __restrict__ tsdf, const float* __restrict__ weight,
                                             const Volume& vol, const Ray& r, float t) {
  const Cell c = ray_cell(r, vol, t);
  bool known = true;
#pragma unroll
  for (int q = 0; q < 8; ++q) known &= __ldg(weight + corner(vol, c.base, q)) > 0.f;
  if (!known) return {false, 0.f};
  float v[8];
#pragma unroll
  for (int q = 0; q < 8; ++q) v[q] = __ldg(tsdf + corner(vol, c.base, q));
  return {true, trilinear(v, c.f)};
}

// Fine stepping applies after a known sample with F < 1 (NaN and F >= 1 step coarsely).
__device__ __forceinline__ bool fine(Sample s) { return s.known && s.F < 1.f; }

// The trilinear colour (3 channels) and TSDF gradient (3 components, um_tsdf_mesh's per-voxel gradient) at t.
__device__ __forceinline__ void ray_shade(const float* __restrict__ tsdf, const float* __restrict__ weight,
                                          const float* __restrict__ color, const Volume& vol, long long total,
                                          const Ray& r, float t, float rgb[3], float grad[3]) {
  const Cell c = ray_cell(r, vol, t);
  float v[8];
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
#pragma unroll
    for (int q = 0; q < 8; ++q) v[q] = __ldg(color + ch * total + corner(vol, c.base, q));
    rgb[ch] = trilinear(v, c.f);
  }
  const Coords lo = voxel_coords(vol, c.base);
  const long long xy = (long long)vol.X * vol.Y;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const long long i = corner(vol, c.base, q);
      const int at[3] = {lo.ii + (q & 1), lo.j + ((q >> 1) & 1), lo.k + (q >> 2)};
      const int dims[3] = {vol.X, vol.Y, vol.Z};
      v[q] = gradient(tsdf, weight, i, a == 0 ? 1 : a == 1 ? vol.X : xy, at[a] > 0, at[a] + 1 < dims[a], __ldg(tsdf + i));
    }
    grad[a] = trilinear(v, c.f);
  }
}

// One thread per pixel of n views of h x w pixels; see include/unimatch_sm100.h (um_tsdf_raycast) for every operation.
__global__ void __launch_bounds__(RAY_TX * RAY_TY)
tsdf_raycast_kernel(const float* __restrict__ tsdf, const float* __restrict__ weight, const float* __restrict__ color,
                    Volume vol, float trunc, const float* __restrict__ c2w, int h, int w, float fx, float fy, float cx,
                    float cy, float near, float far, float* __restrict__ depth, uint8_t* __restrict__ rgb_out,
                    float* __restrict__ normal) {
  const int x = blockIdx.x * RAY_TX + threadIdx.x, y = blockIdx.y * RAY_TY + threadIdx.y, view = blockIdx.z;
  if (x >= w || y >= h) return;
  const long long px = ((long long)view * h + y) * w + x;
  const float* m = c2w + 12 * view;
  const float xc = __fdiv_rn(__fsub_rn((float)x, cx), fx), yc = __fdiv_rn(__fsub_rn((float)y, cy), fy);
  const float origin[3] = {vol.ox, vol.oy, vol.oz};
  const int dims[3] = {vol.X, vol.Y, vol.Z};
  Ray r;
  float t_lo = near, t_hi = far;
  bool ok = vol.X >= 2 && vol.Y >= 2 && vol.Z >= 2;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float d = __fmaf_rn(__ldg(m + 4 * a), xc, __fmaf_rn(__ldg(m + 4 * a + 1), yc, __ldg(m + 4 * a + 2)));
    r.gd[a] = __fdiv_rn(d, vol.vs);
    r.go[a] = __fsub_rn(__fdiv_rn(__fsub_rn(__ldg(m + 4 * a + 3), origin[a]), vol.vs), 0.5f);
    ok &= isfinite(r.gd[a]) && isfinite(r.go[a]);
    const float top = (float)(dims[a] - 1);
    if (r.gd[a] == 0.f) {
      ok &= r.go[a] >= 0.f && r.go[a] <= top;
    } else {
      const float t0 = __fdiv_rn(-r.go[a], r.gd[a]), t1 = __fdiv_rn(__fsub_rn(top, r.go[a]), r.gd[a]);
      t_lo = fmaxf(t_lo, fminf(t0, t1));
      t_hi = fminf(t_hi, fmaxf(t0, t1));
    }
  }
  ok &= t_lo <= t_hi && isfinite(t_hi);
  float out_d = 0.f, out_n[3] = {0.f, 0.f, 0.f};
  int out_c[3] = {0, 0, 0};
  bool hit = false;
  if (ok) {
    const float step_fine = __fmul_rn(vol.vs, 0.5f), step_coarse = __fmul_rn(trunc, 0.5f);
    float ta = t_lo, tb = t_lo;
    Sample A = ray_sample(tsdf, weight, vol, r, ta), B = A;
    while (ta < t_hi) {
      tb = fminf(__fadd_rn(ta, fine(A) ? step_fine : step_coarse), t_hi);
      if (!(tb > ta)) tb = t_hi;
      B = ray_sample(tsdf, weight, vol, r, tb);
      if (!fine(A) && fine(B)) {                               // take the coarse step back: one fine step instead
        tb = fminf(__fadd_rn(ta, step_fine), t_hi);
        if (!(tb > ta)) tb = t_hi;
        B = ray_sample(tsdf, weight, vol, r, tb);
      }
      if (A.known && B.known && (A.F < 0.f) != (B.F < 0.f)) {
        hit = B.F < 0.f;                                       // a change to non-negative is a back face: a miss
        break;
      }
      ta = tb, A = B;
    }
    if (hit) {
      const float s = __fdiv_rn(A.F, __fsub_rn(A.F, B.F));
      out_d = __fmaf_rn(s, __fsub_rn(tb, ta), ta);
      const long long total = (long long)vol.X * vol.Y * vol.Z;
      float ca[3], cb[3], ga[3], gb[3];
      ray_shade(tsdf, weight, color, vol, total, r, ta, ca, ga);
      ray_shade(tsdf, weight, color, vol, total, r, tb, cb, gb);
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        out_c[a] = min(max(__float2int_rn(lerp(s, ca[a], cb[a])), 0), 255);
        out_n[a] = lerp(s, ga[a], gb[a]);
      }
      const float len =
          __fsqrt_rn(__fmaf_rn(out_n[2], out_n[2], __fmaf_rn(out_n[1], out_n[1], __fmul_rn(out_n[0], out_n[0]))));
#pragma unroll
      for (int a = 0; a < 3; ++a) out_n[a] = len == 0.f ? 0.f : __fdiv_rn(out_n[a], len);
    }
  }
  depth[px] = out_d;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    rgb_out[3 * px + a] = (uint8_t)out_c[a];
    normal[3 * px + a] = out_n[a];
  }
}

}  // namespace

namespace um {

static Volume make_volume(int X, int Y, int Z, const float* origin, float voxel_size) {
  return Volume{X, Y, Z, origin[0], origin[1], origin[2], voxel_size};
}

static unsigned volume_blocks(int X, int Y, int Z) {
  return (unsigned)(((long long)X * Y * Z + FUSE_THREADS - 1) / FUSE_THREADS);
}

// Arguments are checked by the entry points (um_api.cu).
int tsdf_integrate_launch(float* tsdf, float* weight, float* color, int X, int Y, int Z, const float* origin,
                          float voxel_size, float trunc, const float* depth, const uint8_t* frames, const float* w2c, int n,
                          int h, int w, float fx, float fy, float cx, float cy, const int* n_valid, cudaStream_t st) {
  tsdf_integrate_kernel<<<volume_blocks(X, Y, Z), FUSE_THREADS, 0, st>>>(
      tsdf, weight, color, make_volume(X, Y, Z, origin, voxel_size), trunc, depth, frames, w2c, n, h, w, fx, fy, cx, cy,
      n_valid);
  return check_launch("um_tsdf_integrate");
}

int tsdf_surface_count_launch(const float* tsdf, const float* weight, int X, int Y, int Z, long long* offsets,
                              cudaStream_t st) {
  const unsigned nb = volume_blocks(X, Y, Z);
  const float origin[3] = {0.f, 0.f, 0.f};
  tsdf_count_kernel<<<nb, FUSE_THREADS, 0, st>>>(tsdf, weight, make_volume(X, Y, Z, origin, 1.f),
                                                 (long long)X * Y * Z, offsets);
  if (int rc = check_launch("um_tsdf_surface_count")) return rc;
  return offsets_scan_launch(offsets, nb, "um_tsdf_surface_count", st);
}

int tsdf_mesh_count_launch(const float* tsdf, const float* weight, int X, int Y, int Z, long long* offsets, cudaStream_t st) {
  const unsigned nb = volume_blocks(X, Y, Z);
  const float origin[3] = {0.f, 0.f, 0.f};
  tsdf_mesh_count_kernel<<<nb, FUSE_THREADS, 0, st>>>(tsdf, weight, make_volume(X, Y, Z, origin, 1.f),
                                                      (long long)X * Y * Z, offsets);
  if (int rc = check_launch("um_tsdf_mesh_count")) return rc;
  return offsets_scan_launch(offsets, nb, "um_tsdf_mesh_count", st);
}

// n_points > 0 (the entry point launches nothing for an empty surface).
int tsdf_mesh_launch(const float* tsdf, const float* weight, const float* color, int X, int Y, int Z, const float* origin,
                     float voxel_size, const long long* point_offsets, const long long* face_offsets, long long n_faces,
                     int* first_vertex, float* points, uint8_t* colors, float* normals, int* faces, cudaStream_t st) {
  const Volume vol = make_volume(X, Y, Z, origin, voxel_size);
  const long long total = (long long)X * Y * Z;
  tsdf_mesh_vertices_kernel<<<volume_blocks(X, Y, Z), FUSE_THREADS, 0, st>>>(tsdf, weight, color, vol, total, point_offsets,
                                                                             points, colors, normals, first_vertex);
  if (int rc = check_launch("um_tsdf_mesh")) return rc;
  if (n_faces == 0) return UM_OK;
  tsdf_faces_kernel<<<volume_blocks(X, Y, Z), FUSE_THREADS, 0, st>>>(tsdf, weight, vol, total, face_offsets, first_vertex,
                                                                     faces);
  return check_launch("um_tsdf_mesh");
}

int tsdf_surface_points_launch(const float* tsdf, const float* weight, const float* color, int X, int Y, int Z,
                               const float* origin, float voxel_size, const long long* offsets, float* points,
                               uint8_t* colors, cudaStream_t st) {
  tsdf_points_kernel<<<volume_blocks(X, Y, Z), FUSE_THREADS, 0, st>>>(
      tsdf, weight, color, make_volume(X, Y, Z, origin, voxel_size), (long long)X * Y * Z, offsets, points, colors);
  return check_launch("um_tsdf_surface_points");
}

int tsdf_raycast_launch(const float* tsdf, const float* weight, const float* color, int X, int Y, int Z, const float* origin,
                        float voxel_size, float trunc, const float* c2w, int n, int h, int w, float fx, float fy, float cx,
                        float cy, float near, float far, float* depth, uint8_t* rgb, float* normal, cudaStream_t st) {
  const dim3 grid((unsigned)((w + RAY_TX - 1) / RAY_TX), (unsigned)((h + RAY_TY - 1) / RAY_TY), (unsigned)n);
  tsdf_raycast_kernel<<<grid, dim3(RAY_TX, RAY_TY), 0, st>>>(tsdf, weight, color, make_volume(X, Y, Z, origin, voxel_size),
                                                            trunc, c2w, h, w, fx, fy, cx, cy, near, far, depth, rgb, normal);
  return check_launch("um_tsdf_raycast");
}

}  // namespace um
