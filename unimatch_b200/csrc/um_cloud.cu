// Point-cloud ops for scoring reconstructions: cell keys (um_cloud_keys), the dense cell table and cell-ordered points
// of an indexed set (um_cloud_ranges), voxel down-sampling (um_cloud_down_sample_count, um_cloud_down_sample), exact
// nearest neighbours by a ring search over the table (um_cloud_nearest) and the fixed-order reduction of its block
// partials (um_cloud_stats).  Semantics and the pruning proof: include/unimatch_sm100.h; the numpy statement is
// tests/refops_recon.py.
#include <limits.h>

#include "um_geometry.cuh"

namespace {

constexpr int CLOUD_THREADS = COMPACT_THREADS, CLOUD_WARPS = CLOUD_THREADS / 32;

struct CloudGrid {
  double o[3], cell;
  int g[3];
};

// The cell of coordinate p along one axis: floor(((double)p - o) / cell), clamped to [0, g - 1].
__device__ __forceinline__ double cell_coord(float p, double o, double cell) {
  return __ddiv_rn(__dsub_rn((double)p, o), cell);
}
__device__ __forceinline__ int cell_index(double t, int g) {
  return t < 0.0 ? 0 : (t >= (double)(g - 1) ? g - 1 : (int)floor(t));
}

__global__ void __launch_bounds__(CLOUD_THREADS)
cloud_keys_kernel(const float* __restrict__ p, long long n, CloudGrid gr, long long* __restrict__ keys) {
  const long long i = (long long)blockIdx.x * CLOUD_THREADS + threadIdx.x;
  if (i >= n) return;
  int k[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) k[a] = cell_index(cell_coord(__ldg(p + 3 * i + a), gr.o[a], gr.cell), gr.g[a]);
  keys[i] = ((long long)k[2] * gr.g[1] + k[1]) * gr.g[0] + k[0];
}

// One thread per sorted position: the first and one-past-last position of each run of equal keys into the zeroed
// start / end tables, and the point at that position (x, y, z, its input index as int bits).
__global__ void __launch_bounds__(CLOUD_THREADS)
cloud_ranges_kernel(const long long* __restrict__ keys, const long long* __restrict__ order, const float* __restrict__ p,
                    long long n, long long n_cells, int* __restrict__ start, int* __restrict__ end,
                    float4* __restrict__ sorted) {
  const long long i = (long long)blockIdx.x * CLOUD_THREADS + threadIdx.x;
  if (i >= n) return;
  const long long key = __ldg(keys + i), j = __ldg(order + i);
  if (key >= 0 && key < n_cells) mark_run(keys, i, n, key, start, end);
  sorted[i] = make_float4(__ldg(p + 3 * j), __ldg(p + 3 * j + 1), __ldg(p + 3 * j + 2), __int_as_float((int)j));
}

__device__ __forceinline__ bool run_head(const long long* __restrict__ keys, long long i, long long n) {
  return i < n && (i == 0 || __ldg(keys + i - 1) != __ldg(keys + i));
}

// Pass 1 of down-sampling: the number of runs (occupied cells) that start in each block of CLOUD_THREADS positions.
__global__ void __launch_bounds__(CLOUD_THREADS)
cloud_heads_kernel(const long long* __restrict__ keys, long long n, long long* __restrict__ block_counts) {
  const long long i = (long long)blockIdx.x * CLOUD_THREADS + threadIdx.x;
  int all;
  block_rank(run_head(keys, i, n), &all);
  if (threadIdx.x == 0) block_counts[blockIdx.x] = all;
}

// Pass 3: the thread at the head of each run writes the run's mean, summed in fp64 in sorted (= input) order, to output
// row offsets[block] + the heads before it in the block.
__global__ void __launch_bounds__(CLOUD_THREADS)
cloud_down_sample_kernel(const long long* __restrict__ keys, const long long* __restrict__ order,
                         const float* __restrict__ p, long long n, const long long* __restrict__ offsets,
                         float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * CLOUD_THREADS + threadIdx.x;
  const bool head = run_head(keys, i, n);
  int all;
  const int before = block_rank(head, &all);
  if (!head) return;
  const long long m = __ldg(offsets + blockIdx.x) + before;
  const long long key = __ldg(keys + i);
  double s[3] = {0.0, 0.0, 0.0};
  long long c = 0;
  for (long long r = i; r < n && __ldg(keys + r) == key; ++r, ++c) {
    const long long j = __ldg(order + r);
#pragma unroll
    for (int a = 0; a < 3; ++a) s[a] = __dadd_rn(s[a], (double)__ldg(p + 3 * j + a));
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) out[3 * m + a] = __double2float_rn(__ddiv_rn(s[a], (double)c));
}

// A lower bound, in metres, on |Q - P| along one axis for every point P of cell k, where t is the query's computed cell
// coordinate: the gap from t to [k, k + 1], less 2^-20 cells and 2^-45 |t| for the rounding of both cell coordinates.
__device__ __forceinline__ double axis_gap(double t, int k, double cell) {
  const double d = fmax(fmax(__dsub_rn((double)k, t), __dsub_rn(t, (double)k + 1.0)), 0.0);
  return __dmul_rn(fmax(__dsub_rn(d, __dadd_rn(0x1p-20, __dmul_rn(0x1p-45, fabs(t)))), 0.0), cell);
}

// The fp32 s of every point of a region whose exact squared distance is at least lb exceeds best when this holds: the
// fp32 s is at least (1 - 2^-21) of the exact value less 2^-147, and the fp64 bound's own rounding is far below 2^-21.
__device__ __forceinline__ bool beyond(double lb, float best) {
  return __dsub_rn(__dmul_rn(lb, 1.0 - 0x1p-20), 0x1p-140) > (double)best;
}

__device__ __forceinline__ double sq(double x) { return __dmul_rn(x, x); }

// The points of cell (kx, ky, kz) into (best, bi), unless the cell is empty or its bound (yz: the y and z gaps squared and
// summed) proves that none reaches s <= best.
__device__ __forceinline__ void visit_cell(const float4* __restrict__ pts, const int* __restrict__ start,
                                           const int* __restrict__ end, const CloudGrid& gr, int kx, int ky, int kz,
                                           double yz, double tx, float qx, float qy, float qz, float& best, int& bi) {
  const long long c = ((long long)kz * gr.g[1] + ky) * gr.g[0] + kx;
  const int b = __ldg(start + c), e = __ldg(end + c);
  if (b == e || beyond(__dadd_rn(yz, sq(axis_gap(tx, kx, gr.cell))), best)) return;
  for (int r = b; r < e; ++r) {
    const float4 p = __ldg(pts + r);
    const float dx = __fsub_rn(qx, p.x), dy = __fsub_rn(qy, p.y), dz = __fsub_rn(qz, p.z);
    const float s = __fmaf_rn(dz, dz, __fmaf_rn(dy, dy, __fmul_rn(dx, dx)));
    const int pi = __float_as_int(p.w);
    if (s < best || (s == best && pi < bi)) best = s, bi = pi;
  }
}

// One query per thread.  Visits the cells of Chebyshev rings r = 0, 1, ... around the query's (clamped) cell, skipping
// cells and stopping at the first ring whose bound proves that nothing beyond it can reach s <= best, or when the rings
// cover the table.  Writes the distance and index, or only the block's partials (sum of d, count of d < threshold).
__global__ void __launch_bounds__(CLOUD_THREADS)
cloud_nearest_kernel(const float* __restrict__ queries, long long nq, const float4* __restrict__ pts,
                     const int* __restrict__ start, const int* __restrict__ end, CloudGrid gr, float threshold,
                     float* __restrict__ distance, long long* __restrict__ index, double* __restrict__ partial_sum,
                     long long* __restrict__ partial_count) {
  const long long i = (long long)blockIdx.x * CLOUD_THREADS + threadIdx.x;
  float d = 0.f;
  if (i < nq) {
    float q[3];
    double t[3], own[3];
    int j[3];
    const double inv_cell = __drcp_rn(gr.cell);      // the query's t only has to be within 2^-51 |t| of exact
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      q[a] = __ldg(queries + 3 * i + a);
      t[a] = __dmul_rn(__dsub_rn((double)q[a], gr.o[a]), inv_cell);
      j[a] = cell_index(t[a], gr.g[a]);
      own[a] = sq(axis_gap(t[a], j[a], gr.cell));
    }
    float best = __int_as_float(0x7f800000);
    int bi = INT_MAX;
    const int gx = gr.g[0], gy = gr.g[1];
#define UM_VISIT(kx) visit_cell(pts, start, end, gr, kx, ky, kz, yz, t[0], q[0], q[1], q[2], best, bi)
    for (int r = 0;; ++r) {
      if (r > 0) {             // the bound beyond ring r - 1: one axis at offset +-r, the others at their own cells
        bool any = false;
        double lb = 0.0;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          const double rest = __dadd_rn(own[(a + 1) % 3], own[(a + 2) % 3]);
#pragma unroll
          for (int side = -1; side <= 1; side += 2) {
            const int k = j[a] + side * r;
            if (k < 0 || k >= gr.g[a]) continue;
            const double v = __dadd_rn(sq(axis_gap(t[a], k, gr.cell)), rest);
            lb = any ? fmin(lb, v) : v;
            any = true;
          }
        }
        if (!any || beyond(lb, best)) break;
      }
      for (int kz = max(j[2] - r, 0); kz <= j[2] + r && kz < gr.g[2]; ++kz) {
        const bool fz = abs(kz - j[2]) == r;
        const double gz = sq(axis_gap(t[2], kz, gr.cell));
        for (int ky = max(j[1] - r, 0); ky <= j[1] + r && ky < gy; ++ky) {
          const double yz = __dadd_rn(sq(axis_gap(t[1], ky, gr.cell)), gz);
          if (fz || abs(ky - j[1]) == r) {
            for (int kx = max(j[0] - r, 0); kx <= min(j[0] + r, gx - 1); ++kx) UM_VISIT(kx);
          } else {
            if (j[0] - r >= 0) UM_VISIT(j[0] - r);
            if (j[0] + r < gx) UM_VISIT(j[0] + r);
          }
        }
      }
    }
#undef UM_VISIT
    d = __fsqrt_rn(best);
    if (distance) distance[i] = d, index[i] = bi;
  }
  if (!partial_sum) return;
  // the block's partials: a shfl_down tree per warp, then the warps in order; counts are exact
  __shared__ double warp_sum[CLOUD_WARPS];
  __shared__ int warp_count[CLOUD_WARPS];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const double v = warp_sum_ordered(i < nq ? (double)d : 0.0);
  const unsigned below = __ballot_sync(0xffffffffu, i < nq && d < threshold);
  if (lane == 0) warp_sum[wid] = v, warp_count[wid] = __popc(below);
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = warp_sum[0];
    long long c = warp_count[0];
    for (int q = 1; q < CLOUD_WARPS; ++q) s = __dadd_rn(s, warp_sum[q]), c += warp_count[q];
    partial_sum[blockIdx.x] = s;
    partial_count[blockIdx.x] = c;
  }
}

// One warp: lane l adds the partials of blocks l, l + 32, ... in order from 0, then a shfl_down tree (16, 8, 4, 2, 1).
__global__ void __launch_bounds__(32)
cloud_stats_kernel(const double* __restrict__ partial_sum, const long long* __restrict__ partial_count, long long nb,
                   double* __restrict__ out) {
  const int lane = threadIdx.x;
  const double s = partials_sum_ordered(partial_sum, nb, 1);
  long long c = 0;
  for (long long b = lane; b < nb; b += 32) c += __ldg(partial_count + b);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_down_sync(0xffffffffu, c, o);
  if (lane == 0) out[0] = s, out[1] = (double)c;
}

}  // namespace

namespace um {

static unsigned cloud_blocks(long long n) { return (unsigned)((n + CLOUD_THREADS - 1) / CLOUD_THREADS); }

static CloudGrid cloud_grid(const double* o, double cell, const int* g) {
  CloudGrid gr;
  for (int a = 0; a < 3; ++a) gr.o[a] = o[a], gr.g[a] = g[a];
  gr.cell = cell;
  return gr;
}

int cloud_keys_launch(const float* points, long long n, const double* origin, double cell, const int* dims,
                      long long* keys, cudaStream_t st) {
  cloud_keys_kernel<<<cloud_blocks(n), CLOUD_THREADS, 0, st>>>(points, n, cloud_grid(origin, cell, dims), keys);
  return check_launch("um_cloud_keys");
}

int cloud_ranges_launch(const long long* keys, const long long* order, const float* points, long long n, long long n_cells,
                        int* start, int* end, float* sorted, cudaStream_t st) {
  if (int rc = zero_runs(start, end, n_cells, "um_cloud_ranges", st)) return rc;
  cloud_ranges_kernel<<<cloud_blocks(n), CLOUD_THREADS, 0, st>>>(keys, order, points, n, n_cells, start, end,
                                                                 reinterpret_cast<float4*>(sorted));
  return check_launch("um_cloud_ranges");
}

int cloud_down_sample_count_launch(const long long* keys, long long n, long long* offsets, cudaStream_t st) {
  const unsigned nb = cloud_blocks(n);
  cloud_heads_kernel<<<nb, CLOUD_THREADS, 0, st>>>(keys, n, offsets);
  if (int rc = check_launch("um_cloud_down_sample_count (heads)")) return rc;
  return offsets_scan_launch(offsets, nb, "um_cloud_down_sample_count (scan)", st);
}

int cloud_down_sample_launch(const long long* keys, const long long* order, const float* points, long long n,
                             const long long* offsets, float* out, cudaStream_t st) {
  cloud_down_sample_kernel<<<cloud_blocks(n), CLOUD_THREADS, 0, st>>>(keys, order, points, n, offsets, out);
  return check_launch("um_cloud_down_sample");
}

int cloud_nearest_launch(const float* queries, long long nq, const float* sorted, const int* start, const int* end,
                         const double* origin, double cell, const int* dims, float threshold, float* distance,
                         long long* index, double* partial_sum, long long* partial_count, cudaStream_t st) {
  cloud_nearest_kernel<<<cloud_blocks(nq), CLOUD_THREADS, 0, st>>>(
      queries, nq, reinterpret_cast<const float4*>(sorted), start, end, cloud_grid(origin, cell, dims), threshold, distance,
      index, partial_sum, partial_count);
  return check_launch("um_cloud_nearest");
}

int cloud_stats_launch(const double* partial_sum, const long long* partial_count, long long nb, double* out,
                       cudaStream_t st) {
  cloud_stats_kernel<<<1, 32, 0, st>>>(partial_sum, partial_count, nb, out);
  return check_launch("um_cloud_stats");
}

}  // namespace um
