// Point tracks chained through the flows of consecutive pairs.  Dense: the forward flows from every pixel of a first frame,
// with the forward occlusion masks deciding visibility (um_chain_tracks).  Sparse: query points, each given at its own
// frame, chained forward through the forward flows and backward through the backward flows (um_track_points_forward /
// um_track_points_backward).  Multi-flow: every pixel of a first frame, each new frame reached from several earlier
// frames, keeping the most certain visible candidate (um_multi_flow_tracks).  Semantics and the fp32 order of operations:
// include/unimatch_sm100.h; the float64 statements are tests/refops_tracks.py, tests/refops_points.py and
// tests/refops_multiflow.py.  Scene flow: the second disparity warped through the flow with the same bilinear
// (um_warp_disparity; statement tests/refops_sceneflow.py).
#include "um_common.cuh"

namespace {

constexpr int TRACK_THREADS = 256;
constexpr int POINT_THREADS = 128;

// Bilinear taps of one axis at pixel coordinate c (align_corners=True): corners i0 = floor(c) and i0 + 1 with weights
// (1 - f, f), f = c - i0 (exact in fp32); in0 / in1 tell which corners lie inside [0, n-1].
struct Axis {
  int i0;
  bool in0, in1;
  float w0, w1;
};
__device__ __forceinline__ Axis axis_taps(float c, int n) {
  Axis a;
  const float f0 = floorf(c);
  a.i0 = (int)f0;
  a.w1 = __fsub_rn(c, f0);
  a.w0 = __fsub_rn(1.f, a.w1);
  a.in0 = a.i0 >= 0 && a.i0 < n;
  a.in1 = a.i0 + 1 >= 0 && a.i0 + 1 < n;
  return a;
}

// s = wy0 (wx0 v00 + wx1 v01) + wy1 (wx0 v10 + wx1 v11), each product and sum rounded on its own (no FMA); a corner outside
// the image is not read and counts as 0 (zero padding).
__device__ __forceinline__ float lerp2(const float* img, int w, const Axis& ax, const Axis& ay) {
  auto at = [&](bool in, int dy, int dx) { return in ? __ldg(img + (long long)(ay.i0 + dy) * w + (ax.i0 + dx)) : 0.f; };
  const float top = __fadd_rn(__fmul_rn(ax.w0, at(ay.in0 && ax.in0, 0, 0)), __fmul_rn(ax.w1, at(ay.in0 && ax.in1, 0, 1)));
  const float bot = __fadd_rn(__fmul_rn(ax.w0, at(ay.in1 && ax.in0, 1, 0)), __fmul_rn(ax.w1, at(ay.in1 && ax.in1, 1, 1)));
  return __fadd_rn(__fmul_rn(ay.w0, top), __fmul_rn(ay.w1, bot));
}

// One step of a track through flow f (planar [2, h, w]) and mask o ([h, w] or NULL): the step every entry shares.
__device__ __forceinline__ void track_step(float2& p, bool& v, const float* f, const float* o, int h, int w) {
  const long long plane = (long long)h * w;
  float dx = 0.f, dy = 0.f, m = 0.f;
  // a track at least a pixel outside (or NaN) has no corner inside: the zero-padded samples are 0
  if (p.x > -1.f && p.x < (float)w && p.y > -1.f && p.y < (float)h) {
    const Axis ax = axis_taps(p.x, w), ay = axis_taps(p.y, h);
    dx = lerp2(f, w, ax, ay);
    dy = lerp2(f + plane, w, ax, ay);
    if (o) m = lerp2(o, w, ax, ay);
  }
  p.x = __fadd_rn(p.x, dx);
  p.y = __fadd_rn(p.y, dy);
  v = v && m < 0.5f && p.x >= 0.f && p.x <= (float)(w - 1) && p.y >= 0.f && p.y <= (float)(h - 1);
}

// One thread owns track `pix` and advances it through the n flows in order; the state is read once and written once.
__global__ void __launch_bounds__(TRACK_THREADS)
chain_tracks_kernel(const float* __restrict__ flow, const float* __restrict__ occ, int n, int h, int w,
                    float2* __restrict__ pos, uint8_t* __restrict__ vis, float2* __restrict__ pos_out,
                    uint8_t* __restrict__ vis_out) {
  const long long plane = (long long)h * w;
  const long long pix = (long long)blockIdx.x * TRACK_THREADS + threadIdx.x;
  if (pix >= plane) return;
  float2 p = pos[pix];
  bool v = vis[pix] != 0;
  for (int t = 0; t < n; ++t) {
    track_step(p, v, flow + (long long)t * 2 * plane, occ ? occ + (long long)t * plane : nullptr, h, w);
    pos_out[(long long)t * plane + pix] = p;
    vis_out[(long long)t * plane + pix] = v ? 1 : 0;
  }
  pos[pix] = p;
  vis[pix] = v ? 1 : 0;
}

// The query's frame t_q if it is an integer in [0, limit), else -1.
__device__ __forceinline__ int query_frame(float t, int limit) {
  return (t >= 0.f && t < (float)limit && t == floorf(t)) ? (int)t : -1;
}

// One thread owns query q and advances it through the launch's pairs t0 .. t0+n-1 that follow its frame: it joins at pair
// t_q (from the query itself) or continues from the state an earlier launch left.
__global__ void __launch_bounds__(POINT_THREADS)
track_points_forward_kernel(const float* __restrict__ flow, const float* __restrict__ occ, int n, int h, int w, int t0,
                            const float* __restrict__ queries, int nq, int nt, float2* __restrict__ pos,
                            uint8_t* __restrict__ vis, float2* __restrict__ tracks, uint8_t* __restrict__ visible) {
  const int q = blockIdx.x * POINT_THREADS + threadIdx.x;
  if (q >= nq) return;
  const int tq = query_frame(queries[3 * q], nt);
  if (tq < 0 || tq >= t0 + n) return;
  const long long plane = (long long)h * w, row = (long long)q * nt;
  float2 p;
  bool v;
  int j = t0;
  if (tq >= t0) {
    p = make_float2(queries[3 * q + 2], queries[3 * q + 1]);
    v = true;
    j = tq;
  } else {
    p = pos[q];
    v = vis[q] != 0;
  }
  for (; j < t0 + n; ++j) {
    const long long i = j - t0;
    track_step(p, v, flow + i * 2 * plane, occ ? occ + i * plane : nullptr, h, w);
    tracks[row + j + 1] = p;
    visible[row + j + 1] = v ? 1 : 0;
  }
  pos[q] = p;
  vis[q] = v ? 1 : 0;
}

// One thread owns query q: frame t_q is the query itself, then pairs t_q-1 .. 0 of the backward flows in turn.  A query
// that cannot be served (t_q not an integer in [0, nt) or past the n stored pairs) gets a NaN, invisible row.
__global__ void __launch_bounds__(POINT_THREADS)
track_points_backward_kernel(const float* __restrict__ flow, const float* __restrict__ occ, int n, int h, int w,
                             const float* __restrict__ queries, int nq, int nt, float2* __restrict__ tracks,
                             uint8_t* __restrict__ visible) {
  const int q = blockIdx.x * POINT_THREADS + threadIdx.x;
  if (q >= nq) return;
  const int tq = query_frame(queries[3 * q], min(nt, n + 1));
  const long long plane = (long long)h * w, row = (long long)q * nt;
  if (tq < 0) {
    for (int t = 0; t < nt; ++t) {
      tracks[row + t] = make_float2(__int_as_float(0x7fffffff), __int_as_float(0x7fffffff));
      visible[row + t] = 0;
    }
    return;
  }
  float2 p = make_float2(queries[3 * q + 2], queries[3 * q + 1]);
  bool v = true;
  tracks[row + tq] = p;
  visible[row + tq] = 1;
  for (int j = tq - 1; j >= 0; --j) {
    track_step(p, v, flow + (long long)j * 2 * plane, occ ? occ + (long long)j * plane : nullptr, h, w);
    tracks[row + j] = p;
    visible[row + j] = v ? 1 : 0;
  }
}

// One thread owns pixel `pix` of the first frame and walks the launch's n frames in order.  Frame t's candidates extend the
// states in slots src[t][j] by the flow, mask and residual of pair (t, j); the choice goes to slot dst[t] and to the
// outputs.  Only this thread touches pixel `pix` of any slot, so a later frame may read a slot an earlier one wrote.
__global__ void __launch_bounds__(TRACK_THREADS)
multi_flow_tracks_kernel(const float* __restrict__ flow, const float* __restrict__ occ, const float* __restrict__ err,
                         const int* __restrict__ src, const int* __restrict__ dst, int n, int k, int h, int w, int r,
                         float2* pos, float* sig, uint8_t* vis, float2* __restrict__ tracks,
                         uint8_t* __restrict__ visible, float* __restrict__ sigma) {
  const long long plane = (long long)h * w;
  const long long pix = (long long)blockIdx.x * TRACK_THREADS + threadIdx.x;
  if (pix >= plane) return;
  const float nan = __int_as_float(0x7fffffff);
  for (int t = 0; t < n; ++t) {
    bool any = false, any_valid = false;
    float2 bp = make_float2(nan, nan), vp = bp;
    float bs = nan, vs = nan;
    for (int j = 0; j < k; ++j) {
      const int s = __ldg(src + t * k + j);
      if (s < 0 || s >= r) continue;
      const long long at = (long long)s * plane + pix, c = (long long)t * k + j;
      float2 p = pos[at];
      float s2 = sig[at];
      bool v = vis[at] != 0;
      float e = 0.f;                                 // the residual at the source position, sampled as track_step samples
      if (p.x > -1.f && p.x < (float)w && p.y > -1.f && p.y < (float)h)
        e = lerp2(err + c * plane, w, axis_taps(p.x, w), axis_taps(p.y, h));
      track_step(p, v, flow + c * 2 * plane, occ + c * plane, h, w);
      s2 = __fadd_rn(s2, __fmul_rn(e, e));
      if (v && (!any_valid || s2 < vs)) {
        any_valid = true;
        vp = p;
        vs = s2;
      }
      if (!any || s2 < bs) {
        any = true;
        bp = p;
        bs = s2;
      }
    }
    const float2 p = any_valid ? vp : bp;
    const float s2 = any_valid ? vs : bs;
    const int d = __ldg(dst + t);
    if (d >= 0 && d < r) {
      const long long at = (long long)d * plane + pix;
      pos[at] = p;
      sig[at] = s2;
      vis[at] = any_valid ? 1 : 0;
    }
    tracks[(long long)t * plane + pix] = p;
    sigma[(long long)t * plane + pix] = s2;
    visible[(long long)t * plane + pix] = any_valid ? 1 : 0;
  }
}

// One thread per pixel of the B frames: q = p + flow(p), then the bilinear sample of disp_next at q clamped into the frame
// (grid_sample's border padding).  The clamped coordinate always lies inside, so only the weight-0 corner at x0 + 1 = w or
// y0 + 1 = h can fall outside, and lerp2 reads 0 there.
__global__ void __launch_bounds__(TRACK_THREADS)
warp_disparity_kernel(const float* __restrict__ disp_next, const float* __restrict__ flow, float* __restrict__ disp1,
                      uint8_t* __restrict__ in_frame, int h, int w, long long total) {
  const long long i = (long long)blockIdx.x * TRACK_THREADS + threadIdx.x;
  if (i >= total) return;
  const long long plane = (long long)h * w;
  const long long b = i / plane, pix = i - b * plane;
  const int y = (int)(pix / w), x = (int)(pix - (long long)y * w);
  const float* f = flow + 2 * b * plane + pix;
  const float qx = __fadd_rn((float)x, __ldg(f)), qy = __fadd_rn((float)y, __ldg(f + plane));
  const float mw = (float)(w - 1), mh = (float)(h - 1);
  in_frame[i] = (qx >= 0.f && qx <= mw && qy >= 0.f && qy <= mh) ? 1 : 0;
  const float cx = fminf(fmaxf(qx, 0.f), mw), cy = fminf(fmaxf(qy, 0.f), mh);
  disp1[i] = lerp2(disp_next + b * plane, w, axis_taps(cx, w), axis_taps(cy, h));
}

}  // namespace

namespace um {

// Arguments are checked by um_chain_tracks (um_api.cu).
int chain_tracks_launch(const float* flow, const float* occ, int n, int h, int w, float* pos, uint8_t* vis, float* pos_out,
                        uint8_t* vis_out, cudaStream_t st) {
  const long long hw = (long long)h * w;
  chain_tracks_kernel<<<(unsigned)((hw + TRACK_THREADS - 1) / TRACK_THREADS), TRACK_THREADS, 0, st>>>(
      flow, occ, n, h, w, reinterpret_cast<float2*>(pos), vis, reinterpret_cast<float2*>(pos_out), vis_out);
  return check_launch("um_chain_tracks");
}

// Arguments are checked by um_track_points_forward / um_track_points_backward (um_api.cu).
int track_points_forward_launch(const float* flow, const float* occ, int n, int h, int w, int t0, const float* queries,
                                int nq, int nt, float* pos, uint8_t* vis, float* tracks, uint8_t* visible, cudaStream_t st) {
  track_points_forward_kernel<<<(unsigned)((nq + POINT_THREADS - 1) / POINT_THREADS), POINT_THREADS, 0, st>>>(
      flow, occ, n, h, w, t0, queries, nq, nt, reinterpret_cast<float2*>(pos), vis, reinterpret_cast<float2*>(tracks),
      visible);
  return check_launch("um_track_points_forward");
}

// Arguments are checked by um_multi_flow_tracks (um_api.cu).
int multi_flow_tracks_launch(const float* flow, const float* occ, const float* err, const int* src, const int* dst, int n,
                             int k, int h, int w, int r, float* pos, float* sig, uint8_t* vis, float* tracks,
                             uint8_t* visible, float* sigma, cudaStream_t st) {
  const long long hw = (long long)h * w;
  multi_flow_tracks_kernel<<<(unsigned)((hw + TRACK_THREADS - 1) / TRACK_THREADS), TRACK_THREADS, 0, st>>>(
      flow, occ, err, src, dst, n, k, h, w, r, reinterpret_cast<float2*>(pos), sig, vis,
      reinterpret_cast<float2*>(tracks), visible, sigma);
  return check_launch("um_multi_flow_tracks");
}

// Arguments are checked by um_warp_disparity (um_api.cu).
int warp_disparity_launch(const float* disp_next, const float* flow, float* disp1, uint8_t* in_frame, int batch, int h, int w,
                          cudaStream_t st) {
  const long long total = (long long)batch * h * w;
  warp_disparity_kernel<<<(unsigned)((total + TRACK_THREADS - 1) / TRACK_THREADS), TRACK_THREADS, 0, st>>>(
      disp_next, flow, disp1, in_frame, h, w, total);
  return check_launch("um_warp_disparity");
}

int track_points_backward_launch(const float* flow, const float* occ, int n, int h, int w, const float* queries, int nq,
                                 int nt, float* tracks, uint8_t* visible, cudaStream_t st) {
  track_points_backward_kernel<<<(unsigned)((nq + POINT_THREADS - 1) / POINT_THREADS), POINT_THREADS, 0, st>>>(
      flow, occ, n, h, w, queries, nq, nt, reinterpret_cast<float2*>(tracks), visible);
  return check_launch("um_track_points_backward");
}

}  // namespace um
