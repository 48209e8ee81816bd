// Shared helpers for libunimatch_sm100 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "unimatch_sm100.h"

#define UM_STR2(x) #x
#define UM_STR(x) UM_STR2(x)
#define UM_C 128                      // feature channels (main_flow.py:73 --feature_channels 128)

namespace um {

void set_error(const char* fmt, ...);
void count_launch(int n = 1);

inline int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: %s", what, cudaGetErrorString(e));
    return UM_ECUDA;
  }
  count_launch();
  return UM_OK;
}

// ---- per-device launch configuration --------------------------------------------------------------------
// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) and the SM count belong to a DEVICE, not to the process: a process
// that runs the module on a second GPU (e.g. the reference's nn.DataParallel branch, main_flow.py:194-198) must
// configure every kernel there too and size its persistent grids for that device.
constexpr int kMaxDevices = 64;
inline int current_device() {
  int d = 0;
  cudaGetDevice(&d);
  return (d >= 0 && d < kMaxDevices) ? d : 0;
}
struct PerDeviceBytes { size_t bytes[kMaxDevices] = {}; };
// raise the dynamic shared-memory limit of `kernel` to `smem` bytes on the current device (once per device and size)
template <typename K>
inline int ensure_smem(PerDeviceBytes& st, K kernel, size_t smem, const char* what) {
  const int d = current_device();
  if (smem <= st.bytes[d]) return UM_OK;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) {
    set_error("cudaFuncSetAttribute(%s): %s", what, cudaGetErrorString(e));
    return UM_ECUDA;
  }
  st.bytes[d] = smem;
  return UM_OK;
}
inline int device_sm_count() {
  static int sms[kMaxDevices] = {};
  const int d = current_device();
  if (!sms[d]) {
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, d);
    sms[d] = n > 0 ? n : 132;
  }
  return sms[d];
}

// The per-image driver kernels put the image on grid y, which holds at most 65535 CTAs.  A batch of n images is launched
// in chunks of at most that many: launch(first, count) launches images first .. first + count - 1, and each launch is
// checked.  Every batch the drivers run is one chunk.
constexpr long long kMaxGridY = 65535;
template <class Launch>
inline int launch_image_chunks(long long n, const char* what, Launch launch) {
  for (long long first = 0; first < n; first += kMaxGridY) {
    launch(first, (unsigned)(n - first < kMaxGridY ? n - first : kMaxGridY));
    if (int rc = check_launch(what)) return rc;
  }
  return UM_OK;
}

// Runs body() in both arms of `if (ragged)`.  A driver kernel reads an image's geometry from a table or derives it from a
// uniform shape; inlined into each arm, its body is compiled with the layout known, so the one instantiation holds a
// uniform and a ragged version, and a thread outside its ragged image leaves without running the uniform version's
// index arithmetic first (most CTAs of a grid sized by the capacity have no pixel).
template <class Body>
__device__ __forceinline__ void by_layout(bool ragged, Body body) {
  if (ragged) body();
  else body();
}

#define UM_REQUIRE(cond, ...)             \
  do {                                    \
    if (!(cond)) {                        \
      um::set_error(__VA_ARGS__);         \
      return UM_EINVAL;                   \
    }                                     \
  } while (0)

// ---- window geometry (attention.py:45-104 / :107-163 as pure index arithmetic) -------------------------
struct Geom {
  int h, w, kh, kw, wh, ww, sh, sw, mask_mode, lw, nwin;
};

inline bool make_geom(const um_attn_geom* g, Geom* o) {
  if (!g || g->h <= 0 || g->w <= 0 || g->kh <= 0 || g->kw <= 0) return false;
  if (g->h % g->kh || g->w % g->kw) return false;
  o->h = g->h; o->w = g->w; o->kh = g->kh; o->kw = g->kw;
  o->wh = g->h / g->kh; o->ww = g->w / g->kw;
  o->sh = g->sh; o->sw = g->sw; o->mask_mode = g->mask_mode;
  o->lw = o->wh * o->ww; o->nwin = g->kh * g->kw;
  if (o->sh < 0 || o->sh >= o->h || o->sw < 0 || o->sw >= o->w) return false;
  return true;
}

// token t of window `win` -> index into the (unrolled) h*w grid
__device__ __forceinline__ int window_token(const Geom& g, int win, int t, int* yr_out = nullptr, int* xr_out = nullptr) {
  int wy = win / g.kw, wx = win - wy * g.kw;
  int i = t / g.ww, j = t - i * g.ww;
  int yr = wy * g.wh + i, xr = wx * g.ww + j;          // coordinates in the rolled frame
  if (yr_out) *yr_out = yr;
  if (xr_out) *xr_out = xr;
  int y = yr + g.sh; if (y >= g.h) y -= g.h;           // rolled[y,x] = orig[(y+sh)%h, (x+sw)%w]
  int x = xr + g.sw; if (x >= g.w) x -= g.w;
  return y * g.w + x;
}

// Swin shift-region id in the rolled frame (utils.py:84-108): 3 bands per axis.
__device__ __forceinline__ int shift_region(const Geom& g, int yr, int xr) {
  int ry = (g.sh > 0) ? ((yr < g.h - g.wh) ? 0 : ((yr < g.h - g.sh) ? 1 : 2)) : 0;
  int rx = (g.sw > 0) ? ((xr < g.w - g.ww) ? 0 : ((xr < g.w - g.sw) ? 1 : 2)) : 0;
  return ry * 3 + rx;
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Per-image geometry of the ragged entries (um_ragged_item, read from device memory): an item is used only if it lies
// inside the capacity and inside the packed buffer; otherwise its threads read and write nothing.
__device__ __forceinline__ bool ragged_ok(const um_ragged_item& it, int h_max, int w_max, long long elems_per_pixel,
                                          long long numel) {
  return it.h > 0 && it.w > 0 && it.h <= h_max && it.w <= w_max && it.offset >= 0 &&
         it.offset + elems_per_pixel * it.h * it.w <= numel;
}

}  // namespace um
