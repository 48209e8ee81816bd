// Frame-to-model point-to-plane ICP against the fused TSDF volume (KinectFusion's tracking): the depth pyramid
// (um_icp_downsample), live normals (um_icp_normals), the pose state and reference rows (um_icp_init), projective
// association with the per-block normal equations (um_icp_reduce), the Gauss-Newton step (um_icp_solve) and acceptance
// (um_icp_accept).  The model maps come from um_tsdf_raycast (um_fusion.cu), unchanged.
// Semantics and the order of operations: include/unimatch_sm100.h; the numpy statement is tests/refops_icp.py.
#include "um_geometry.cuh"

namespace {

constexpr int ICP_TX = 16, ICP_TY = 8, ICP_THREADS = ICP_TX * ICP_TY, ICP_WARPS = ICP_THREADS / 32;
constexpr int TERMS = UM_ICP_TERMS;
constexpr int STATE = UM_ICP_STATE;
constexpr int PIXEL_THREADS = 256;

__device__ __forceinline__ int frames_valid(const int* __restrict__ n_valid, int n) {
  return min(max(__ldg(n_valid), 0), n);
}

// One thread per output pixel: the mean of the 2 x 2 block's valid depths within trunc of its smallest valid depth.
__global__ void __launch_bounds__(PIXEL_THREADS)
icp_downsample_kernel(const float* __restrict__ src, float* __restrict__ dst, int n, int h, int w, int h2, int w2,
                      float trunc) {
  const long long i = (long long)blockIdx.x * PIXEL_THREADS + threadIdx.x;
  if (i >= (long long)n * h2 * w2) return;
  const int f = (int)(i / ((long long)h2 * w2));
  const int r = (int)(i - (long long)f * h2 * w2), y = r / w2, x = r - y * w2;
  const float* s = src + (long long)f * h * w + (long long)(2 * y) * w + 2 * x;
  const float d[4] = {__ldg(s), __ldg(s + 1), __ldg(s + w), __ldg(s + w + 1)};
  float lo = 0.f;
  bool any = false;
#pragma unroll
  for (int q = 0; q < 4; ++q)
    if (valid_depth(d[q])) lo = any ? fminf(lo, d[q]) : d[q], any = true;
  float sum = 0.f;
  int c = 0;
#pragma unroll
  for (int q = 0; q < 4; ++q)
    if (valid_depth(d[q]) && __fsub_rn(d[q], lo) <= trunc) sum = __fadd_rn(sum, d[q]), ++c;
  dst[i] = any ? __fdiv_rn(sum, (float)c) : 0.f;
}

// One thread per pixel: the unit normal (v(x+1, y) - v) x (v(x, y+1) - v) facing the camera, 0 where not all three
// depths are valid or the cross product vanishes.
__global__ void __launch_bounds__(PIXEL_THREADS)
icp_normals_kernel(const float* __restrict__ depth, float* __restrict__ normal, int n, int h, int w, float fx, float fy,
                   float cx, float cy) {
  const long long i = (long long)blockIdx.x * PIXEL_THREADS + threadIdx.x;
  if (i >= (long long)n * h * w) return;
  const int r = (int)(i % ((long long)h * w)), y = r / w, x = r - y * w;
  float out[3] = {0.f, 0.f, 0.f};
  if (x + 1 < w && y + 1 < h) {
    const float d = __ldg(depth + i), dx = __ldg(depth + i + 1), dy = __ldg(depth + i + w);
    if (valid_depth(d) && valid_depth(dx) && valid_depth(dy)) {
      const Pinhole k = {fx, fy, cx, cy};
      const float3 v = back_project(k, (float)x, (float)y, d), vx = back_project(k, (float)(x + 1), (float)y, dx),
                   vy = back_project(k, (float)x, (float)(y + 1), dy);
      const float e1[3] = {__fsub_rn(vx.x, v.x), __fsub_rn(vx.y, v.y), __fsub_rn(vx.z, v.z)};
      const float e2[3] = {__fsub_rn(vy.x, v.x), __fsub_rn(vy.y, v.y), __fsub_rn(vy.z, v.z)};
      float c[3];
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        const int b = (a + 1) % 3, e = (a + 2) % 3;
        c[a] = __fsub_rn(__fmul_rn(e1[b], e2[e]), __fmul_rn(e1[e], e2[b]));
      }
      const float len = __fsqrt_rn(__fmaf_rn(c[2], c[2], __fmaf_rn(c[1], c[1], __fmul_rn(c[0], c[0]))));
      const float facing = __fmaf_rn(c[2], v.z, __fmaf_rn(c[1], v.y, __fmul_rn(c[0], v.x)));
      if (len > 0.f && isfinite(len)) {
        const float s = facing > 0.f ? -len : len;
#pragma unroll
        for (int a = 0; a < 3; ++a) out[a] = __fdiv_rn(c[a], s);
      }
    }
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) normal[3 * i + a] = out[a];
}

__device__ __forceinline__ double dm(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double da(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double ds(double a, double b) { return __dsub_rn(a, b); }

// The rigid inverse (R^T, -R^T t) of the [3, 4] rows m, rounded to fp32 rows.
__device__ __forceinline__ void rigid_inverse_rows(const double* m, float* out) {
#pragma unroll
  for (int i = 0; i < 3; ++i) {
#pragma unroll
    for (int j = 0; j < 3; ++j) out[4 * i + j] = (float)m[4 * j + i];
    out[4 * i + 3] = (float)-da(da(dm(m[i], m[3]), dm(m[4 + i], m[7])), dm(m[8 + i], m[11]));
  }
}

// Per frame f < n_valid: T_ref = C P (C the [4, 4] correction, or P itself without one), T = T_ref, no degenerate
// solve, and T_ref's fp32 camera-to-world and world-to-camera rows.
__global__ void icp_init_kernel(const double* __restrict__ poses, const double* __restrict__ correction, int n,
                                const int* __restrict__ n_valid, double* __restrict__ state, float* __restrict__ c2w,
                                float* __restrict__ w2c) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= frames_valid(n_valid, n)) return;
  const double* P = poses + 16 * f;
  double ref[12];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (correction) {
        const double* C = correction + 4 * i;
        double v = da(da(dm(C[0], P[j]), dm(C[1], P[4 + j])), dm(C[2], P[8 + j]));
        ref[4 * i + j] = j == 3 ? da(v, C[3]) : v;
      } else {
        ref[4 * i + j] = P[4 * i + j];
      }
    }
  }
  double* s = state + (long long)STATE * f;
#pragma unroll
  for (int q = 0; q < 12; ++q) {
    s[q] = ref[q], s[12 + q] = ref[q];
    c2w[12 * f + q] = (float)ref[q];
  }
  s[24] = 0.0;
  rigid_inverse_rows(ref, w2c + 12 * f);
}

// The per-pixel terms of one live pixel: a (6), r and whether it is an inlier and a valid live pixel.
struct PixelTerms {
  float a[6], r;
  bool inlier, valid;
};

__device__ __forceinline__ PixelTerms pixel_terms(const float* __restrict__ depth, const float* __restrict__ live_normal,
                                                  const float* __restrict__ model_depth,
                                                  const float* __restrict__ model_normal, const float T[12],
                                                  const float* __restrict__ M, const float* __restrict__ V, int f, int x,
                                                  int y, int h, int w, float fx, float fy, float cx, float cy,
                                                  float max_distance, float cos_max_angle) {
  PixelTerms t = {{0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, 0.f, false, false};
  if (x >= w || y >= h) return t;
  const long long plane = (long long)h * w, i = (long long)f * plane + (long long)y * w + x;
  const float d = __ldg(depth + i);
  const float n[3] = {__ldg(live_normal + 3 * i), __ldg(live_normal + 3 * i + 1), __ldg(live_normal + 3 * i + 2)};
  if (!valid_depth(d) || (n[0] == 0.f && n[1] == 0.f && n[2] == 0.f)) return t;
  t.valid = true;
  const Pinhole k = {fx, fy, cx, cy};
  const float3 v = back_project(k, (float)x, (float)y, d);
  float p[3], nw[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    p[a] = apply_row(T, a, v);
    nw[a] = __fmaf_rn(T[4 * a + 2], n[2], __fmaf_rn(T[4 * a + 1], n[1], __fmul_rn(T[4 * a], n[0])));
  }
  // projective association in the reference camera (world-to-camera rows V), integration's nearest-pixel rule
  const float3 c = apply_rows(V, make_float3(p[0], p[1], p[2]));
  if (!(c.z > 0.f)) return t;
  float xf, yf;
  if (!nearest_pixel(project(k, c), w, h, xf, yf)) return t;
  const long long j = (long long)f * plane + (long long)yf * w + (long long)xf;
  const float D = __ldg(model_depth + j);
  const float m[3] = {__ldg(model_normal + 3 * j), __ldg(model_normal + 3 * j + 1), __ldg(model_normal + 3 * j + 2)};
  if (!(D > 0.f) || (m[0] == 0.f && m[1] == 0.f && m[2] == 0.f)) return t;
  // the model vertex: the ray cast's direction through the pixel centre, at its depth, from the reference camera
  const float xc = __fdiv_rn(__fsub_rn(xf, cx), fx), yc = __fdiv_rn(__fsub_rn(yf, cy), fy);
  float diff[3], pc[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float dir = __fmaf_rn(M[4 * a], xc, __fmaf_rn(M[4 * a + 1], yc, M[4 * a + 2]));
    diff[a] = __fsub_rn(p[a], __fmaf_rn(D, dir, M[4 * a + 3]));
    pc[a] = __fsub_rn(p[a], M[4 * a + 3]);
  }
  const float dist = __fsqrt_rn(__fmaf_rn(diff[2], diff[2], __fmaf_rn(diff[1], diff[1], __fmul_rn(diff[0], diff[0]))));
  const float cosang = __fmaf_rn(nw[2], m[2], __fmaf_rn(nw[1], m[1], __fmul_rn(nw[0], m[0])));
  if (!(dist <= max_distance && cosang >= cos_max_angle)) return t;
  t.inlier = true;
  t.r = __fmaf_rn(m[2], diff[2], __fmaf_rn(m[1], diff[1], __fmul_rn(m[0], diff[0])));
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const int b = (a + 1) % 3, e = (a + 2) % 3;
    t.a[a] = __fsub_rn(__fmul_rn(pc[b], m[e]), __fmul_rn(pc[e], m[b]));
    t.a[3 + a] = m[a];
  }
  return t;
}

// One term of every thread's pixel summed over the warp (lane 0 holds the sum) into warp_sums[k].
__device__ __forceinline__ void warp_term(double v, int k, int lane, double* warp_sums) {
  v = warp_sum_ordered(v);
  if (lane == 0) warp_sums[k] = v;
}

// One thread per live pixel of 16 x 8 tiles; per block, the 30 sums over its pixels: a warp shuffle tree, then the warps
// in order, written to partials[f, block].
__global__ void __launch_bounds__(ICP_THREADS)
icp_reduce_kernel(const float* __restrict__ depth, const float* __restrict__ live_normal,
                  const float* __restrict__ model_depth, const float* __restrict__ model_normal,
                  const double* __restrict__ state, const float* __restrict__ c2w, const float* __restrict__ w2c, int n,
                  int h, int w, float fx, float fy, float cx, float cy, float max_distance, float cos_max_angle,
                  const int* __restrict__ n_valid, double* __restrict__ partials) {
  const int f = blockIdx.z;
  if (f >= frames_valid(n_valid, n)) return;
  __shared__ double warp_sums[ICP_WARPS][TERMS];
  __shared__ float rows[3][12];
  const int tid = threadIdx.y * ICP_TX + threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid < 12) {
    rows[0][tid] = (float)__ldg(state + (long long)STATE * f + tid);
    rows[1][tid] = __ldg(c2w + 12 * f + tid);
    rows[2][tid] = __ldg(w2c + 12 * f + tid);
  }
  __syncthreads();
  const PixelTerms t = pixel_terms(depth, live_normal, model_depth, model_normal, rows[0], rows[1], rows[2], f,
                                   blockIdx.x * ICP_TX + threadIdx.x, blockIdx.y * ICP_TY + threadIdx.y, h, w, fx, fy, cx,
                                   cy, max_distance, cos_max_angle);
  // terms: k < 21 the upper triangle of a a^T row by row, 21..26 a r, 27 r^2, 28 inlier, 29 valid (0 unless an inlier,
  // but for 29); fp32 products, converted to fp64
  double* ws = warp_sums[wid];
  int k = 0;
#pragma unroll
  for (int i = 0; i < 6; ++i)
#pragma unroll
    for (int j = i; j < 6; ++j, ++k) warp_term(t.inlier ? (double)__fmul_rn(t.a[i], t.a[j]) : 0.0, k, lane, ws);
#pragma unroll
  for (int i = 0; i < 6; ++i) warp_term(t.inlier ? (double)__fmul_rn(t.a[i], t.r) : 0.0, 21 + i, lane, ws);
  warp_term(t.inlier ? (double)__fmul_rn(t.r, t.r) : 0.0, 27, lane, ws);
  warp_term(t.inlier ? 1.0 : 0.0, 28, lane, ws);
  warp_term(t.valid ? 1.0 : 0.0, 29, lane, ws);
  __syncthreads();
  if (tid < TERMS) {
    double s = warp_sums[0][tid];
#pragma unroll
    for (int q = 1; q < ICP_WARPS; ++q) s = da(s, warp_sums[q][tid]);
    const long long nb = (long long)gridDim.x * gridDim.y, b = (long long)blockIdx.y * gridDim.x + blockIdx.x;
    partials[((long long)f * nb + b) * TERMS + tid] = s;
  }
}

// The 30 sums of frame f, one warp per term (warp q takes terms q and q + 15, so the solve keeps 128 registers): lane l
// sums the partials of blocks l, l + 32, ... in order from 0, then a shfl_down tree (16, 8, 4, 2, 1) adds the lanes.
// No atomics: the same result from run to run.
constexpr int SUM_THREADS = 32 * (TERMS / 2);

__device__ __forceinline__ void sum_partials(const double* __restrict__ partials, int nb, int f, double* sums) {
  const int lane = threadIdx.x & 31;
  for (int k = threadIdx.x >> 5; k < TERMS; k += TERMS / 2) {
    const double s = partials_sum_ordered(partials + (long long)f * nb * TERMS + k, nb, TERMS);
    if (lane == 0) sums[k] = s;
  }
  __syncthreads();
}

// The Gauss-Newton step of frame blockIdx.x: the Jacobi-scaled Cholesky solve, then T <- dT T.
__global__ void __launch_bounds__(SUM_THREADS)
icp_solve_kernel(const double* __restrict__ partials, int nb, int n, const int* __restrict__ n_valid, double min_inliers,
                 double min_pivot, int record, double* __restrict__ state) {
  const int f = blockIdx.x;
  if (f >= frames_valid(n_valid, n)) return;
  __shared__ double S[TERMS];
  sum_partials(partials, nb, f, S);
  if (threadIdx.x != 0) return;
  double* st = state + (long long)STATE * f;
  double A[6][6], b[6], sc[6], L[6][6], x[6];
  for (int i = 0, k = 0; i < 6; ++i)
    for (int j = i; j < 6; ++j, ++k) A[i][j] = A[j][i] = S[k];
  bool ok = S[28] >= min_inliers;
  for (int i = 0; i < 6; ++i) {                                 // an unconstrained unknown (A_ii = 0) keeps a zero pivot
    b[i] = S[21 + i];
    sc[i] = A[i][i] > 0.0 ? __drcp_rn(__dsqrt_rn(A[i][i])) : 1.0;
  }
  for (int j = 0; ok && j < 6; ++j) {
    double d = dm(dm(A[j][j], sc[j]), sc[j]);
    for (int k = 0; k < j; ++k) d = ds(d, dm(L[j][k], L[j][k]));
    ok &= d >= min_pivot;                                      // NaN fails too
    if (!ok) break;
    L[j][j] = __dsqrt_rn(d);
    for (int i = j + 1; i < 6; ++i) {
      double e = dm(dm(A[i][j], sc[i]), sc[j]);
      for (int k = 0; k < j; ++k) e = ds(e, dm(L[i][k], L[j][k]));
      L[i][j] = __ddiv_rn(e, L[j][j]);
    }
  }
  if (!ok) {
    if (record) st[24] = da(st[24], 1.0);
    return;
  }
  for (int i = 0; i < 6; ++i) {                                 // L z = -S b
    double e = -dm(b[i], sc[i]);
    for (int k = 0; k < i; ++k) e = ds(e, dm(L[i][k], x[k]));
    x[i] = __ddiv_rn(e, L[i][i]);
  }
  for (int i = 5; i >= 0; --i) {                                // L^T y = z
    double e = x[i];
    for (int k = i + 1; k < 6; ++k) e = ds(e, dm(L[k][i], x[k]));
    x[i] = __ddiv_rn(e, L[i][i]);
  }
  for (int i = 0; i < 6; ++i) x[i] = dm(x[i], sc[i]);
  // dT: the rotation exp(w) (Rodrigues) about the reference centre c, then the translation tau
  const double th = __dsqrt_rn(da(da(dm(x[0], x[0]), dm(x[1], x[1])), dm(x[2], x[2])));
  double R[3][3] = {{1.0, 0.0, 0.0}, {0.0, 1.0, 0.0}, {0.0, 0.0, 1.0}};
  if (th > 0.0) {
    const double k[3] = {__ddiv_rn(x[0], th), __ddiv_rn(x[1], th), __ddiv_rn(x[2], th)};
    const double c = cos(th), s = sin(th), v = ds(1.0, c);
    const double K[3][3] = {{0.0, -k[2], k[1]}, {k[2], 0.0, -k[0]}, {-k[1], k[0], 0.0}};
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) R[i][j] = da(da(i == j ? c : 0.0, dm(s, K[i][j])), dm(dm(v, k[i]), k[j]));
  }
  double T[12], u[3];
  for (int q = 0; q < 12; ++q) T[q] = st[q];
  for (int a = 0; a < 3; ++a) u[a] = ds(T[4 * a + 3], st[12 + 4 * a + 3]);
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) st[4 * i + j] = da(da(dm(R[i][0], T[j]), dm(R[i][1], T[4 + j])), dm(R[i][2], T[8 + j]));
    const double ru = da(da(dm(R[i][0], u[0]), dm(R[i][1], u[1])), dm(R[i][2], u[2]));
    st[4 * i + 3] = da(da(ru, st[12 + 4 * i + 3]), x[3 + i]);
  }
}

// Acceptance of frame blockIdx.x from the last association pass: the outputs, T_ref back when not tracked, and the
// correction C = T P^-1 when tracked (n == 1).
__global__ void __launch_bounds__(SUM_THREADS)
icp_accept_kernel(const double* __restrict__ partials, int nb, int n, const int* __restrict__ n_valid,
                  double min_inlier_fraction, const double* __restrict__ poses, double* __restrict__ correction,
                  double* __restrict__ state, float* __restrict__ pose_out, uint8_t* __restrict__ tracked,
                  int64_t* __restrict__ inliers, float* __restrict__ rmse, float* __restrict__ w2c) {
  const int f = blockIdx.x;
  if (f >= frames_valid(n_valid, n)) return;
  __shared__ double S[TERMS];
  sum_partials(partials, nb, f, S);
  if (threadIdx.x != 0) return;
  double* st = state + (long long)STATE * f;
  const bool ok = st[24] == 0.0 && S[28] >= dm(min_inlier_fraction, S[29]);
  if (!ok)
    for (int q = 0; q < 12; ++q) st[q] = st[12 + q];
  tracked[f] = ok;
  inliers[f] = (int64_t)S[28];
  rmse[f] = S[28] > 0.0 ? (float)__dsqrt_rn(__ddiv_rn(S[27], S[28])) : 0.f;
  float* po = pose_out + 16 * f;
  for (int q = 0; q < 12; ++q) po[q] = (float)st[q];
  po[12] = po[13] = po[14] = 0.f, po[15] = 1.f;
  rigid_inverse_rows(st, w2c + 12 * f);
  if (ok && correction) {                        // C = T P^-1, P^-1 = (P_R^T, -P_R^T P_t)
    const double* P = poses + 16 * f;
    double Pi[12];
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) Pi[4 * i + j] = P[4 * j + i];
      Pi[4 * i + 3] = -da(da(dm(P[i], P[3]), dm(P[4 + i], P[7])), dm(P[8 + i], P[11]));
    }
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 4; ++j) {
        const double v = da(da(dm(st[4 * i], Pi[j]), dm(st[4 * i + 1], Pi[4 + j])), dm(st[4 * i + 2], Pi[8 + j]));
        correction[4 * i + j] = j == 3 ? da(v, st[4 * i + 3]) : v;
      }
  }
}

}  // namespace

namespace um {

static unsigned pixel_blocks(long long n) { return (unsigned)((n + PIXEL_THREADS - 1) / PIXEL_THREADS); }

int icp_downsample_launch(const float* src, float* dst, int n, int h, int w, float trunc, cudaStream_t st) {
  const int h2 = h / 2, w2 = w / 2;
  icp_downsample_kernel<<<pixel_blocks((long long)n * h2 * w2), PIXEL_THREADS, 0, st>>>(src, dst, n, h, w, h2, w2, trunc);
  return check_launch("um_icp_downsample");
}

int icp_normals_launch(const float* depth, float* normal, int n, int h, int w, float fx, float fy, float cx, float cy,
                       cudaStream_t st) {
  icp_normals_kernel<<<pixel_blocks((long long)n * h * w), PIXEL_THREADS, 0, st>>>(depth, normal, n, h, w, fx, fy, cx, cy);
  return check_launch("um_icp_normals");
}

int icp_init_launch(const double* poses, const double* correction, int n, const int* n_valid, double* state, float* c2w,
                    float* w2c, cudaStream_t st) {
  icp_init_kernel<<<(unsigned)((n + 63) / 64), 64, 0, st>>>(poses, correction, n, n_valid, state, c2w, w2c);
  return check_launch("um_icp_init");
}

int icp_reduce_launch(const float* depth, const float* live_normal, const float* model_depth, const float* model_normal,
                      const double* state, const float* c2w, const float* w2c, int n, int h, int w, float fx, float fy,
                      float cx, float cy, float max_distance, float cos_max_angle, const int* n_valid, double* partials,
                      cudaStream_t st) {
  const dim3 grid((unsigned)((w + ICP_TX - 1) / ICP_TX), (unsigned)((h + ICP_TY - 1) / ICP_TY), (unsigned)n);
  icp_reduce_kernel<<<grid, dim3(ICP_TX, ICP_TY), 0, st>>>(depth, live_normal, model_depth, model_normal, state, c2w, w2c,
                                                          n, h, w, fx, fy, cx, cy, max_distance, cos_max_angle, n_valid,
                                                          partials);
  return check_launch("um_icp_reduce");
}

int icp_solve_launch(const double* partials, int nb, int n, const int* n_valid, double min_inliers, double min_pivot,
                     int record, double* state, cudaStream_t st) {
  icp_solve_kernel<<<(unsigned)n, SUM_THREADS, 0, st>>>(partials, nb, n, n_valid, min_inliers, min_pivot, record, state);
  return check_launch("um_icp_solve");
}

int icp_accept_launch(const double* partials, int nb, int n, const int* n_valid, double min_inlier_fraction,
                      const double* poses, double* correction, double* state, float* pose_out, uint8_t* tracked,
                      int64_t* inliers, float* rmse, float* w2c, cudaStream_t st) {
  icp_accept_kernel<<<(unsigned)n, SUM_THREADS, 0, st>>>(partials, nb, n, n_valid, min_inlier_fraction, poses, correction, state,
                                               pose_out, tracked, inliers, rmse, w2c);
  return check_launch("um_icp_accept");
}

}  // namespace um
