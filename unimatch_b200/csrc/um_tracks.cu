// Dense point tracks: the forward flows of consecutive pairs chained from every pixel of a first frame, with the forward
// occlusion masks deciding visibility.  Semantics and the fp32 order of operations: include/unimatch_sm100.h
// (um_chain_tracks); the float64 statement is tests/refops_tracks.py.
#include "um_common.cuh"

namespace {

constexpr int TRACK_THREADS = 256;

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
  const float xmax = (float)(w - 1), ymax = (float)(h - 1);
  for (int t = 0; t < n; ++t) {
    const float* f = flow + (long long)t * 2 * plane;
    float dx = 0.f, dy = 0.f, o = 0.f;
    // a track at least a pixel outside (or NaN) has no corner inside: the zero-padded samples are 0
    if (p.x > -1.f && p.x < (float)w && p.y > -1.f && p.y < (float)h) {
      const Axis ax = axis_taps(p.x, w), ay = axis_taps(p.y, h);
      dx = lerp2(f, w, ax, ay);
      dy = lerp2(f + plane, w, ax, ay);
      if (occ) o = lerp2(occ + (long long)t * plane, w, ax, ay);
    }
    p.x = __fadd_rn(p.x, dx);
    p.y = __fadd_rn(p.y, dy);
    v = v && o < 0.5f && p.x >= 0.f && p.x <= xmax && p.y >= 0.f && p.y <= ymax;
    pos_out[(long long)t * plane + pix] = p;
    vis_out[(long long)t * plane + pix] = v ? 1 : 0;
  }
  pos[pix] = p;
  vis[pix] = v ? 1 : 0;
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

}  // namespace um
