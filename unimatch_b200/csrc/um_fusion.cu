// TSDF fusion of posed depth maps into a dense voxel volume (um_tsdf_integrate) and the zero-crossing points of the fused
// surface (um_tsdf_surface_count, um_tsdf_surface_points).  Semantics and the fp32 order of operations:
// include/unimatch_sm100.h; the float32 and float64 statements are tests/refops_fusion.py.
#include "um_common.cuh"

namespace {

constexpr int FUSE_THREADS = UM_TSDF_THREADS;
constexpr int FUSE_WARPS = FUSE_THREADS / 32;

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
  const float px = centre(ii, vol.vs, vol.ox), py = centre(j, vol.vs, vol.oy), pz = centre(k, vol.vs, vol.oz);
  const long long plane = (long long)h * w;
  bool loaded = false;
  float F = 0.f, Wt = 0.f, R = 0.f, G = 0.f, B = 0.f;
  for (int t = 0; t < nv; ++t) {
    const float* m = w2c + 12 * t;
    const float czz = __fmaf_rn(__ldg(m + 10), pz, __fmaf_rn(__ldg(m + 9), py, __fmaf_rn(__ldg(m + 8), px, __ldg(m + 11))));
    if (!(czz > 0.f)) continue;
    const float cxx = __fmaf_rn(__ldg(m + 2), pz, __fmaf_rn(__ldg(m + 1), py, __fmaf_rn(__ldg(m + 0), px, __ldg(m + 3))));
    const float cyy = __fmaf_rn(__ldg(m + 6), pz, __fmaf_rn(__ldg(m + 5), py, __fmaf_rn(__ldg(m + 4), px, __ldg(m + 7))));
    const float u = __fmaf_rn(fx, __fdiv_rn(cxx, czz), cx), v = __fmaf_rn(fy, __fdiv_rn(cyy, czz), cy);
    const float xf = floorf(__fadd_rn(u, 0.5f)), yf = floorf(__fadd_rn(v, 0.5f));
    if (!(xf >= 0.f && xf < (float)w && yf >= 0.f && yf < (float)h)) continue;      // NaN fails too
    const long long pix = (long long)yf * w + (long long)xf;
    const float d = __ldg(depth + t * plane + pix);
    if (!(isfinite(d) && d > 0.f)) continue;
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

// Block-wide exclusive sum of one int per thread, in thread order; also returns the block's total.
__device__ __forceinline__ int block_exclusive_sum(int x, int* total) {
  __shared__ int warp_sums[FUSE_WARPS];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int incl = x;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += y;
  }
  if (lane == 31) warp_sums[wid] = incl;
  __syncthreads();
  int before = 0, all = 0;
#pragma unroll
  for (int q = 0; q < FUSE_WARPS; ++q) {
    const int s = warp_sums[q];
    before += q < wid ? s : 0;
    all += s;
  }
  *total = all;
  return before + incl - x;
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

// Pass 2: one CTA turns the block counts into exclusive offsets in place, FUSE_THREADS at a time, in order; the total
// follows them at offsets[nb].
__global__ void __launch_bounds__(FUSE_THREADS) tsdf_scan_kernel(long long* __restrict__ offsets, long long nb) {
  __shared__ long long warp_sums[FUSE_WARPS];
  __shared__ long long carry;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (long long base = 0; base < nb; base += FUSE_THREADS) {
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
    for (int q = 0; q < FUSE_WARPS; ++q) {
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

// Pass 3: every voxel writes its points at its block's offset plus the points of the voxels before it in the block.
__global__ void __launch_bounds__(FUSE_THREADS)
tsdf_points_kernel(const float* __restrict__ tsdf, const float* __restrict__ weight, const float* __restrict__ color,
                   Volume vol, long long total, const long long* __restrict__ offsets, float* __restrict__ points,
                   uint8_t* __restrict__ colors) {
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
    ++o;
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
  tsdf_scan_kernel<<<1, FUSE_THREADS, 0, st>>>(offsets, (long long)nb);
  return check_launch("um_tsdf_surface_count");
}

int tsdf_surface_points_launch(const float* tsdf, const float* weight, const float* color, int X, int Y, int Z,
                               const float* origin, float voxel_size, const long long* offsets, float* points,
                               uint8_t* colors, cudaStream_t st) {
  tsdf_points_kernel<<<volume_blocks(X, Y, Z), FUSE_THREADS, 0, st>>>(
      tsdf, weight, color, make_volume(X, Y, Z, origin, voxel_size), (long long)X * Y * Z, offsets, points, colors);
  return check_launch("um_tsdf_surface_points");
}

}  // namespace um
