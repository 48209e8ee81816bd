// Small fused glue kernels on the matching path: position add, convex upsampling, x2 bilinear flow upsampling.
// All channel-last, all bandwidth-bound, all vectorised (float4).
#include "um_common.cuh"

namespace {

// ---- feature_add_position (utils.py:111-131): x + table[y mod wh, x mod ww, :] ---------------------------
__global__ void __launch_bounds__(256) add_position_kernel(const float4* __restrict__ x, const float4* __restrict__ table,
                                                           float4* __restrict__ out, int h, int w, int wh, int ww,
                                                           long long total4) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < total4; i += stride) {
    const int c4 = (int)(i & 31);
    const long long tok = i >> 5;
    const int xx = (int)(tok % w);
    const int yy = (int)((tok / w) % h);
    const float4 p = __ldg(table + ((long long)(yy % wh) * ww + (xx % ww)) * 32 + c4);
    float4 v = __ldg(x + i);
    v.x += p.x; v.y += p.y; v.z += p.z; v.w += p.w;
    out[i] = v;
  }
}

// ---- convex upsampling (utils.py:134-152) ---------------------------------------------------------------
// thread = (low-res pixel, sub-pixel ky*F+kx); mask reads are coalesced over the sub-pixel index.
__global__ void __launch_bounds__(256) convex_upsample_kernel(const float* __restrict__ flow, const float* __restrict__ mask,
                                                              float* __restrict__ up, int h, int w, int fd, int F,
                                                              float mult, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int FF = F * F;
  const int sp = (int)(i % FF);
  const long long pix = i / FF;
  const int x = (int)(pix % w);
  const int y = (int)((pix / w) % h);
  const long long b = pix / ((long long)h * w);
  const float* mrow = mask + pix * (9LL * FF) + sp;
  float lg[9], mx = -3.4e38f;
#pragma unroll
  for (int t = 0; t < 9; ++t) { lg[t] = __ldg(mrow + t * FF); mx = fmaxf(mx, lg[t]); }
  float den = 0.f;
#pragma unroll
  for (int t = 0; t < 9; ++t) { lg[t] = expf(lg[t] - mx); den += lg[t]; }
  float a0 = 0.f, a1 = 0.f;
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    const int yy = y + t / 3 - 1, xx = x + t % 3 - 1;
    if (yy < 0 || yy >= h || xx < 0 || xx >= w) continue;
    const float p = lg[t] / den;
    const float* fp = flow + ((b * h + yy) * (long long)w + xx) * fd;
    a0 = fmaf(p, mult * __ldg(fp), a0);
    if (fd > 1) a1 = fmaf(p, mult * __ldg(fp + 1), a1);
  }
  const int ky = sp / F, kx = sp - ky * F;
  const long long H = (long long)h * F, W = (long long)w * F;
  const long long o = ((b * fd) * H + (long long)y * F + ky) * W + (long long)x * F + kx;
  up[o] = a0;
  if (fd > 1) up[o + H * W] = a1;
}

// ---- F.interpolate(scale_factor=2, bilinear, align_corners=True) * mult (unimatch.py:154) -----------------
__global__ void __launch_bounds__(256) upsample2x_kernel(const float* __restrict__ in, float* __restrict__ out, int h,
                                                         int w, int fd, float mult, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int H = 2 * h, W = 2 * w;
  const int c = (int)(i % fd);
  const long long p = i / fd;
  const int X = (int)(p % W);
  const int Y = (int)((p / W) % H);
  const long long b = p / ((long long)H * W);
  // ATen area_pixel_compute_source_index, align_corners: src = dst * (in-1)/(out-1)
  const float sy = (H > 1) ? (float)(h - 1) / (float)(H - 1) : 0.f;
  const float sx = (W > 1) ? (float)(w - 1) / (float)(W - 1) : 0.f;
  const float fy = sy * (float)Y, fx = sx * (float)X;
  const int y0 = (int)fy, x0 = (int)fx;
  const int y1 = y0 + ((y0 < h - 1) ? 1 : 0), x1 = x0 + ((x0 < w - 1) ? 1 : 0);
  const float ly = fy - (float)y0, lx = fx - (float)x0;
  const float hy = 1.0f - ly, hx = 1.0f - lx;
  const float* base = in + b * (long long)h * w * fd + c;
  const float v00 = __ldg(base + ((long long)y0 * w + x0) * fd), v01 = __ldg(base + ((long long)y0 * w + x1) * fd);
  const float v10 = __ldg(base + ((long long)y1 * w + x0) * fd), v11 = __ldg(base + ((long long)y1 * w + x1) * fd);
  out[i] = (hy * (hx * v00 + lx * v01) + ly * (hx * v10 + lx * v11)) * mult;
}

// ---- planar bilinear resize, align_corners=True (the drivers' F.interpolate before / after the model) -------------------
// Sample (Y, X) of an (hi, wi) -> (ho, wo) resize: bilinear(src, Y (hi-1)/(ho-1), X (wi-1)/(wo-1)), ATen's
// upsample_bilinear2d arithmetic (area_pixel_compute_source_index with align_corners, lambda weights, the same order of
// operations).  `load(y, x)` reads the source, so every caller -- fp32 planes, uint8 channel-last frames, transposed or
// not -- runs the same instructions and gets the same bits for the same source values.  Every rounding step is an explicit
// intrinsic, so the compiler cannot contract the blend differently in different kernels; the FMAs are the ones the
// original `hy * (hx*v00 + lx*v01) + ly * (hx*v10 + lx*v11)` compiled to.  At equal sizes the weights are exactly (1, 0)
// and the result is the source value.
template <class Load>
__device__ __forceinline__ float bilinear_align_corners(const Load& load, int hi, int wi, int ho, int wo, int Y, int X) {
  const float sy = (ho > 1) ? __fdiv_rn((float)(hi - 1), (float)(ho - 1)) : 0.f;
  const float sx = (wo > 1) ? __fdiv_rn((float)(wi - 1), (float)(wo - 1)) : 0.f;
  const float fy = __fmul_rn(sy, (float)Y), fx = __fmul_rn(sx, (float)X);
  const int y0 = (int)fy, x0 = (int)fx;
  const int y1 = y0 + ((y0 < hi - 1) ? 1 : 0), x1 = x0 + ((x0 < wi - 1) ? 1 : 0);
  const float ly = __fsub_rn(fy, (float)y0), lx = __fsub_rn(fx, (float)x0);
  const float hy = __fsub_rn(1.0f, ly), hx = __fsub_rn(1.0f, lx);
  const float v00 = load(y0, x0), v01 = load(y0, x1);
  const float v10 = load(y1, x0), v11 = load(y1, x1);
  const float row0 = __fmaf_rn(lx, v01, __fmul_rn(hx, v00));
  const float row1 = __fmaf_rn(hx, v10, __fmul_rn(lx, v11));
  return __fmaf_rn(hy, row0, __fmul_rn(ly, row1));
}

// out[b,c,Y,X] = scale[c] * bilinear(in[b,c], ...).  `flip_x`: the OUTPUT is mirrored horizontally (torchvision hflip of
// evaluate_stereo.py:789-796 folded into the same pass).
__global__ void __launch_bounds__(256) resize_bilinear_kernel(const float* __restrict__ in, float* __restrict__ out, int C,
                                                              int hi, int wi, int ho, int wo, float s0, float s1, float s2,
                                                              int flip_x, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int X = (int)(i % wo);
  const int Y = (int)((i / wo) % ho);
  const long long bc = i / ((long long)ho * wo);
  const int c = (int)(bc % C);
  const float* base = in + bc * (long long)hi * wi;
  const float v = bilinear_align_corners([&](int y, int x) { return __ldg(base + (long long)y * wi + x); }, hi, wi, ho, wo, Y, X);
  const float sc = c == 0 ? s0 : (c == 1 ? s1 : s2);
  const int Xo = flip_x ? wo - 1 - X : X;
  out[(bc * ho + Y) * (long long)wo + Xo] = sc == 1.0f ? v : v * sc;
}

// ---- video frames -> model input: uint8 [T,H,W,3] channel-last -> fp32 planar [T,3,ho,wo] -------------------------------
// = resize_bilinear(frames.permute(0,3,1,2).float()), with the portrait transpose of evaluate_flow.py:713-717 (the source
// is read as [3, W, H]) folded into the load.  One thread per output pixel, three planes written.
__global__ void __launch_bounds__(256) frames_to_planar_kernel(const uint8_t* __restrict__ frames, float* __restrict__ out,
                                                               int H, int W, int transpose, int ho, int wo, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int X = (int)(i % wo);
  const int Y = (int)((i / wo) % ho);
  const long long t = i / ((long long)ho * wo);
  const int hs = transpose ? W : H, ws = transpose ? H : W;     // source size as the resize sees it
  const uint8_t* base = frames + t * (long long)H * W * 3;
  const long long plane = (long long)ho * wo;
  float* o = out + t * 3 * plane + (long long)Y * wo + X;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const auto load = [&](int y, int x) {
      const long long pix = transpose ? (long long)x * W + y : (long long)y * W + x;
      return (float)__ldg(base + pix * 3 + c);
    };
    o[c * plane] = bilinear_align_corners(load, hs, ws, ho, wo, Y, X);
  }
}

// ---- depth frames -> model input: uint8 [T,H,W,3] -> ImageNet-normalised fp32 planar [T,3,ho,wo] ----------------------
// = resize_bilinear of the frames normalised the way the depth data pipeline does it on the host
// (dataloader/depth/augmentation.py:30, 56-61): every SOURCE sample is x / 255, then - mean_c, then / std_c, each one
// correctly rounded fp32 operation in that order, and the normalised samples are resampled.  No transpose: the depth
// drivers have no portrait rule.
__global__ void __launch_bounds__(256) frames_to_planar_normalized_kernel(const uint8_t* __restrict__ frames,
                                                                          float* __restrict__ out, int H, int W, int ho, int wo,
                                                                          float m0, float m1, float m2, float s0, float s1,
                                                                          float s2, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int X = (int)(i % wo);
  const int Y = (int)((i / wo) % ho);
  const long long t = i / ((long long)ho * wo);
  const uint8_t* base = frames + t * (long long)H * W * 3;
  const long long plane = (long long)ho * wo;
  float* o = out + t * 3 * plane + (long long)Y * wo + X;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float mean = c == 0 ? m0 : (c == 1 ? m1 : m2), std = c == 0 ? s0 : (c == 1 ? s1 : s2);
    const auto load = [&](int y, int x) {
      const float v = (float)__ldg(base + ((long long)y * W + x) * 3 + c);
      return __fdiv_rn(__fsub_rn(__fdiv_rn(v, 255.0f), mean), std);
    };
    o[c * plane] = bilinear_align_corners(load, H, W, ho, wo, Y, X);
  }
}

// ---- Middlebury flow colouring: flow_to_image of utils/flow_viz.py:240-275 (the VCN variant) --------------------------
// Precision follows numpy on float32 flow: |u| or |v| > 1e7 (UNKNOWN_FLOW_THRESH, :140) -> zeroed and painted black;
// rad = sqrt(u*u + v*v) and its per-image maximum in FLOAT32 (:264-265); everything after that in FLOAT64, because
// `maxrad + np.finfo(float).eps` is a float64 scalar (:267-268) and compute_color (:195-236) works on the float64 result.
// The build contracts a*b+c into FMAs, which numpy does not: every step below is an explicitly rounded intrinsic.
// NaN components are treated like unknown flow (excluded from the maximum, painted black).
__device__ __forceinline__ bool flow_unknown(float u, float v) {
  return !(fabsf(u) <= 1e7f) || !(fabsf(v) <= 1e7f);        // also true for NaN
}

__global__ void __launch_bounds__(256) flow_maxrad_kernel(const float* __restrict__ flow, unsigned* __restrict__ maxbits,
                                                          long long hw) {
  const int n = blockIdx.y;
  const float* u = flow + (long long)n * 2 * hw;
  const float* v = u + hw;
  float m = 0.f;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < hw; p += (long long)gridDim.x * blockDim.x) {
    const float a = __ldg(u + p), b = __ldg(v + p);
    if (flow_unknown(a, b)) continue;
    m = fmaxf(m, __fsqrt_rn(__fadd_rn(__fmul_rn(a, a), __fmul_rn(b, b))));
  }
  m = um::warp_max(m);
  __shared__ float part[8];
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < 8; ++i) m = fmaxf(m, part[i]);
    atomicMax(maxbits + n, __float_as_uint(m));              // m >= 0: the bit patterns order like the values
  }
}

// Middlebury colour wheel (make_color_wheel, flow_viz.py:145-192): 55 hues, RY 15, YG 6, GC 4, CB 11, BM 13, MR 6.
__device__ __forceinline__ int wheel(int k, int ch) {
  const int r0 = 255, g0 = 255, b0 = 255;
  if (k < 15) { const int s = 255 * k / 15; return ch == 0 ? r0 : ch == 1 ? s : 0; }
  k -= 15;
  if (k < 6) { const int s = 255 * k / 6; return ch == 0 ? 255 - s : ch == 1 ? g0 : 0; }
  k -= 6;
  if (k < 4) { const int s = 255 * k / 4; return ch == 0 ? 0 : ch == 1 ? g0 : s; }
  k -= 4;
  if (k < 11) { const int s = 255 * k / 11; return ch == 0 ? 0 : ch == 1 ? 255 - s : b0; }
  k -= 11;
  if (k < 13) { const int s = 255 * k / 13; return ch == 0 ? s : ch == 1 ? 0 : b0; }
  k -= 13;
  const int s = 255 * k / 6;
  return ch == 0 ? r0 : ch == 1 ? 0 : 255 - s;
}

__global__ void __launch_bounds__(256) flow_color_kernel(const float* __restrict__ flow, const unsigned* __restrict__ maxbits,
                                                         uint8_t* __restrict__ out, int w, long long hw, long long row_stride,
                                                         long long image_stride, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long n = i / hw, p = i - n * hw;
  const float uf = __ldg(flow + n * 2 * hw + p), vf = __ldg(flow + n * 2 * hw + hw + p);
  uint8_t* o = out + n * image_stride + (p / w) * row_stride + (p % w) * 3;
  if (flow_unknown(uf, vf)) { o[0] = o[1] = o[2] = 0; return; }
  const double den = __dadd_rn((double)__uint_as_float(__ldg(maxbits + n)), 2.220446049250313e-16);   // maxrad + eps
  const double u = __ddiv_rn((double)uf, den), v = __ddiv_rn((double)vf, den);
  const double rad = __dsqrt_rn(__dadd_rn(__dmul_rn(u, u), __dmul_rn(v, v)));
  const double a = __ddiv_rn(atan2(-v, -u), 3.141592653589793);
  const double fk = __dadd_rn(__dmul_rn(__ddiv_rn(__dadd_rn(a, 1.0), 2.0), 54.0), 1.0);        // (a+1)/2*(ncols-1)+1
  const int k0 = (int)floor(fk);
  const int k1 = k0 + 1 == 56 ? 1 : k0 + 1;
  const double f = __dsub_rn(fk, (double)k0);
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const double c0 = __ddiv_rn((double)wheel(k0 - 1, ch), 255.0), c1 = __ddiv_rn((double)wheel(k1 - 1, ch), 255.0);
    double col = __dadd_rn(__dmul_rn(__dsub_rn(1.0, f), c0), __dmul_rn(f, c1));
    col = rad <= 1.0 ? __dsub_rn(1.0, __dmul_rn(rad, __dsub_rn(1.0, col))) : __dmul_rn(col, 0.75);
    o[ch] = (uint8_t)(int)floor(__dmul_rn(255.0, col));
  }
}

// ---- disparity colouring: vis_disparity of utils/visualization.py:11-16 ------------------------------------------------
// numpy on a float32 disparity: g = uint8(((d - min) / (max - min)) * 255) per image, three separately rounded fp32
// operations (the build would otherwise contract and reorder them), truncated; a NaN result gives 0 (what numpy's cast
// gives on x86-64), which covers constant images, NaN anywhere in the image (min / max propagate it) and +-inf.  The
// picture is cv2's COLORMAP_INFERNO LUT at g, in cv2's BGR channel order (what cv2.imwrite writes).
// Per-image min / max live in 2n words as order-preserving keys of the floats, so that unsigned atomicMax orders like the
// values, negatives included: lo[i] = max of ~key (= ~min key), hi[i] = max of key.  A NaN sets hi[i] to 0xFFFFFFFF, the
// key of a NaN that no other value has, and that flag paints the whole image INFERNO[0].  Both start at 0 (one memset).
__device__ __forceinline__ unsigned float_key(float f) {
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_float(unsigned k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
constexpr unsigned kNanKey = 0xffffffffu;

// cv2.applyColorMap(np.arange(256, dtype=np.uint8)[:, None], cv2.COLORMAP_INFERNO): 256 x (B, G, R)
__device__ const uint8_t kInferno[768] = {
    4, 0, 0, 5, 0, 1, 6, 1, 1, 8, 1, 1, 10, 1, 2, 12, 2, 2, 14, 2, 2, 16, 2, 3,
    18, 3, 4, 20, 3, 4, 23, 4, 5, 25, 4, 6, 27, 5, 7, 29, 5, 8, 31, 6, 9, 34, 7, 10,
    36, 7, 11, 38, 8, 12, 41, 8, 13, 43, 9, 14, 45, 9, 16, 48, 10, 17, 50, 10, 18, 52, 11, 20,
    55, 11, 21, 57, 11, 22, 60, 12, 24, 62, 12, 25, 65, 12, 27, 67, 12, 28, 69, 12, 30, 72, 12, 31,
    74, 12, 33, 76, 12, 35, 79, 12, 36, 81, 12, 38, 83, 11, 40, 85, 11, 41, 87, 11, 43, 89, 11, 45,
    91, 10, 47, 92, 10, 49, 94, 10, 50, 95, 10, 52, 97, 9, 54, 98, 9, 56, 99, 9, 57, 100, 9, 59,
    101, 9, 61, 102, 9, 62, 103, 10, 64, 104, 10, 66, 104, 10, 68, 105, 10, 69, 106, 11, 71, 106, 11, 73,
    107, 12, 74, 107, 12, 76, 108, 13, 77, 108, 13, 79, 108, 14, 81, 109, 14, 82, 109, 15, 84, 109, 15, 85,
    110, 16, 87, 110, 16, 89, 110, 17, 90, 110, 18, 92, 110, 18, 93, 110, 19, 95, 110, 19, 97, 110, 20, 98,
    110, 21, 100, 110, 21, 101, 110, 22, 103, 110, 22, 105, 110, 23, 106, 110, 24, 108, 110, 24, 109, 110, 25, 111,
    110, 25, 113, 110, 26, 114, 110, 26, 116, 110, 27, 117, 109, 28, 119, 109, 28, 120, 109, 29, 122, 109, 29, 124,
    109, 30, 125, 108, 30, 127, 108, 31, 128, 108, 32, 130, 107, 32, 132, 107, 33, 133, 107, 33, 135, 106, 34, 136,
    106, 34, 138, 105, 35, 140, 105, 35, 141, 105, 36, 143, 104, 37, 144, 104, 37, 146, 103, 38, 147, 103, 38, 149,
    102, 39, 151, 102, 39, 152, 101, 40, 154, 100, 41, 155, 100, 41, 157, 99, 42, 159, 99, 42, 160, 98, 43, 162,
    97, 44, 163, 96, 44, 165, 96, 45, 166, 95, 46, 168, 94, 46, 169, 94, 47, 171, 93, 48, 173, 92, 48, 174,
    91, 49, 176, 90, 50, 177, 90, 50, 179, 89, 51, 180, 88, 52, 182, 87, 53, 183, 86, 53, 185, 85, 54, 186,
    84, 55, 188, 83, 56, 189, 82, 57, 191, 81, 58, 192, 80, 58, 193, 79, 59, 195, 78, 60, 196, 77, 61, 198,
    76, 62, 199, 75, 63, 200, 74, 64, 202, 73, 65, 203, 72, 66, 204, 71, 67, 206, 70, 68, 207, 69, 69, 208,
    68, 70, 210, 67, 71, 211, 66, 72, 212, 65, 74, 213, 63, 75, 215, 62, 76, 216, 61, 77, 217, 60, 78, 218,
    59, 80, 219, 58, 81, 221, 56, 82, 222, 55, 83, 223, 54, 85, 224, 53, 86, 225, 52, 87, 226, 51, 89, 227,
    49, 90, 228, 48, 92, 229, 47, 93, 230, 46, 94, 231, 45, 96, 232, 43, 97, 233, 42, 99, 234, 41, 100, 235,
    40, 102, 235, 38, 103, 236, 37, 105, 237, 36, 106, 238, 35, 108, 239, 33, 110, 239, 32, 111, 240, 31, 113, 241,
    29, 115, 241, 28, 116, 242, 27, 118, 243, 25, 120, 243, 24, 121, 244, 23, 123, 245, 21, 125, 245, 20, 126, 246,
    19, 128, 246, 18, 130, 247, 16, 132, 247, 15, 133, 248, 14, 135, 248, 12, 137, 248, 11, 139, 249, 10, 140, 249,
    9, 142, 249, 8, 144, 250, 7, 146, 250, 7, 148, 250, 6, 150, 251, 6, 151, 251, 6, 153, 251, 6, 155, 251,
    7, 157, 251, 7, 159, 252, 8, 161, 252, 9, 163, 252, 10, 165, 252, 12, 166, 252, 13, 168, 252, 15, 170, 252,
    17, 172, 252, 18, 174, 252, 20, 176, 252, 22, 178, 252, 24, 180, 252, 26, 182, 251, 29, 184, 251, 31, 186, 251,
    33, 188, 251, 35, 190, 251, 38, 192, 250, 40, 194, 250, 42, 196, 250, 45, 198, 250, 47, 199, 249, 50, 201, 249,
    53, 203, 249, 55, 205, 248, 58, 207, 248, 61, 209, 247, 64, 211, 247, 67, 213, 246, 70, 215, 246, 73, 217, 245,
    76, 219, 245, 79, 221, 244, 83, 223, 244, 86, 225, 244, 90, 227, 243, 93, 229, 243, 97, 230, 242, 101, 232, 242,
    105, 234, 242, 109, 236, 241, 113, 237, 241, 117, 239, 241, 121, 241, 241, 125, 242, 242, 130, 244, 242, 134, 245, 243,
    138, 246, 243, 142, 248, 244, 146, 249, 245, 150, 250, 246, 154, 251, 248, 157, 252, 249, 161, 253, 250, 164, 255, 252,
};

// grid (x: CTAs over the pixels of one image, y: image); 4 loads in flight per thread and step
__global__ void __launch_bounds__(256) disp_minmax_kernel(const float* __restrict__ disp, unsigned* __restrict__ lo,
                                                          unsigned* __restrict__ hi, int hw) {
  const int n = blockIdx.y;
  const float* d = disp + (long long)n * hw;
  unsigned l = 0, m = 0;
  bool nan = false;
  const int stride = gridDim.x * blockDim.x;
  for (long long p0 = blockIdx.x * blockDim.x + threadIdx.x; p0 < hw; p0 += 4LL * stride) {
    float v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const long long p = p0 + (long long)k * stride;
      v[k] = p < hw ? __ldg(d + p) : __ldg(d + p0);     // out of range: repeat a value of this thread's, no effect
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      nan |= v[k] != v[k];
      const unsigned key = float_key(v[k]);
      l = max(l, ~key);
      m = max(m, key);
    }
  }
  if (nan) m = kNanKey;
  l = __reduce_max_sync(0xffffffffu, l);
  m = __reduce_max_sync(0xffffffffu, m);
  __shared__ unsigned part[2][8];
  if ((threadIdx.x & 31) == 0) { part[0][threadIdx.x >> 5] = l; part[1][threadIdx.x >> 5] = m; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < 8; ++i) { l = max(l, part[0][i]); m = max(m, part[1][i]); }
    atomicMax(lo + n, l);
    atomicMax(hi + n, m);
  }
}

// grid (x: CTAs over the pixels of one image, y: image); the LUT is staged in shared memory once per CTA, because every
// warp indexes it divergently (a __constant__ table would serialise those reads)
__global__ void __launch_bounds__(256) disp_color_kernel(const float* __restrict__ disp, const unsigned* __restrict__ lo,
                                                         const unsigned* __restrict__ hi, uint8_t* __restrict__ out, int w,
                                                         int hw, long long row_stride, long long image_stride) {
  __shared__ uint8_t lut[768];
  for (int i = threadIdx.x; i < 768; i += blockDim.x) lut[i] = kInferno[i];
  __syncthreads();
  const int n = blockIdx.y;
  const unsigned hkey = __ldg(hi + n);
  const bool flagged = hkey == kNanKey;
  const float mn = key_float(~__ldg(lo + n)), mx = key_float(hkey);
  const float range = __fsub_rn(mx, mn);
  const float* d = disp + (long long)n * hw;
  uint8_t* img = out + n * image_stride;
  for (long long p = blockIdx.x * blockDim.x + threadIdx.x; p < hw; p += (long long)gridDim.x * blockDim.x) {
    const float q = __fmul_rn(__fdiv_rn(__fsub_rn(__ldg(d + p), mn), range), 255.0f);
    const int g = (flagged || !(q >= 0.f)) ? 0 : min((int)q, 255);          // NaN -> 0; (int) truncates, as numpy's cast
    const int y = (int)p / w, x = (int)p - y * w;
    uint8_t* o = img + y * row_stride + 3LL * x;
    o[0] = lut[3 * g]; o[1] = lut[3 * g + 1]; o[2] = lut[3 * g + 2];
  }
}

// ---- depth colouring: viz_depth_tensor(1. / depth) of utils/visualization.py:92-107 ----------------------------------
// Per image of N pixels, as numpy 1.19 / matplotlib 3.5.1 evaluate it (oracle/depth_viz.py states it step by step):
// inv = 1 / depth (correctly rounded fp32); vmin = min(inv); vmax = a * (1 - g) + b * g in float64, where a and b are the
// sorted inv at ranks k and min(k + 1, N - 1), k = floor(0.95 * (N - 1)) and g its fraction; t = (inv - vmin) /
// fp32(vmax - vmin) in fp32; x = t * 256 indexes the plasma table, below 0 -> first colour, 255 and above -> last colour,
// NaN -> black.  vmin == vmax (and vmin > vmax, where matplotlib raises; only float64 rounding with a = vmin gets there)
// gives t = 0 everywhere; a NaN anywhere in the image (or a NaN vmax, +inf * 0 when b = +inf and g = 0) paints it black.
// a and b are found exactly by a radix select on the order-preserving keys of inv, one byte per pass from the top: pass 0
// fuses the reciprocal, the minimum and the NaN flag with the histogram of the top byte; passes 1-3 histogram the next
// byte of the keys under rank k's prefix and, where it differs, rank k+1's.  Per image the scratch holds one 2 x 256-bin
// histogram per pass and kDvState words of state, all zeroed by one memset; the launch count does not depend on the data.
constexpr int kDvBins = 256;
constexpr int kDvHistWords = 4 * 2 * kDvBins;
enum : int { kDvLo, kDvNan, kDvPrefA, kDvPrefB, kDvRankA, kDvRankB, kDvRange, kDvMode, kDvState };
constexpr int kDvWords = kDvHistWords + kDvState;          // = 2056, the per-image scratch size the header states
enum : unsigned { kDvNormal = 0, kDvFlat = 1, kDvBlack = 2 };
constexpr unsigned kNoBin = 0xffffffffu;

// matplotlib's _plasma_data (CC0) as uint8(floor(float64(c) * 255)): 256 x (R, G, B)
__device__ const uint8_t kPlasma[768] = {
    12, 7, 134, 16, 7, 135, 19, 6, 137, 21, 6, 138, 24, 6, 139, 27, 6, 140, 29, 6, 141, 31, 5, 142,
    33, 5, 143, 35, 5, 144, 37, 5, 145, 39, 5, 146, 41, 5, 147, 43, 5, 148, 45, 4, 148, 47, 4, 149,
    49, 4, 150, 51, 4, 151, 52, 4, 152, 54, 4, 152, 56, 4, 153, 58, 4, 154, 59, 3, 154, 61, 3, 155,
    63, 3, 156, 64, 3, 156, 66, 3, 157, 68, 3, 158, 69, 3, 158, 71, 2, 159, 73, 2, 159, 74, 2, 160,
    76, 2, 161, 78, 2, 161, 79, 2, 162, 81, 1, 162, 82, 1, 163, 84, 1, 163, 86, 1, 163, 87, 1, 164,
    89, 1, 164, 90, 0, 165, 92, 0, 165, 94, 0, 165, 95, 0, 166, 97, 0, 166, 98, 0, 166, 100, 0, 167,
    101, 0, 167, 103, 0, 167, 104, 0, 167, 106, 0, 167, 108, 0, 168, 109, 0, 168, 111, 0, 168, 112, 0, 168,
    114, 0, 168, 115, 0, 168, 117, 0, 168, 118, 1, 168, 120, 1, 168, 121, 1, 168, 123, 2, 168, 124, 2, 167,
    126, 3, 167, 127, 3, 167, 129, 4, 167, 130, 4, 167, 132, 5, 166, 133, 6, 166, 134, 7, 166, 136, 7, 165,
    137, 8, 165, 139, 9, 164, 140, 10, 164, 142, 12, 164, 143, 13, 163, 144, 14, 163, 146, 15, 162, 147, 16, 161,
    149, 17, 161, 150, 18, 160, 151, 19, 160, 153, 20, 159, 154, 21, 158, 155, 23, 158, 157, 24, 157, 158, 25, 156,
    159, 26, 155, 160, 27, 155, 162, 28, 154, 163, 29, 153, 164, 30, 152, 165, 31, 151, 167, 33, 151, 168, 34, 150,
    169, 35, 149, 170, 36, 148, 172, 37, 147, 173, 38, 146, 174, 39, 145, 175, 40, 144, 176, 42, 143, 177, 43, 143,
    178, 44, 142, 180, 45, 141, 181, 46, 140, 182, 47, 139, 183, 48, 138, 184, 50, 137, 185, 51, 136, 186, 52, 135,
    187, 53, 134, 188, 54, 133, 189, 55, 132, 190, 56, 131, 191, 57, 130, 192, 59, 129, 193, 60, 128, 194, 61, 128,
    195, 62, 127, 196, 63, 126, 197, 64, 125, 198, 65, 124, 199, 66, 123, 200, 68, 122, 201, 69, 121, 202, 70, 120,
    203, 71, 119, 204, 72, 118, 205, 73, 117, 206, 74, 117, 207, 75, 116, 208, 77, 115, 209, 78, 114, 209, 79, 113,
    210, 80, 112, 211, 81, 111, 212, 82, 110, 213, 83, 109, 214, 85, 109, 215, 86, 108, 215, 87, 107, 216, 88, 106,
    217, 89, 105, 218, 90, 104, 219, 91, 103, 220, 93, 102, 220, 94, 102, 221, 95, 101, 222, 96, 100, 223, 97, 99,
    223, 98, 98, 224, 100, 97, 225, 101, 96, 226, 102, 96, 227, 103, 95, 227, 104, 94, 228, 106, 93, 229, 107, 92,
    229, 108, 91, 230, 109, 90, 231, 110, 90, 232, 112, 89, 232, 113, 88, 233, 114, 87, 234, 115, 86, 234, 116, 85,
    235, 118, 84, 236, 119, 84, 236, 120, 83, 237, 121, 82, 237, 123, 81, 238, 124, 80, 239, 125, 79, 239, 126, 78,
    240, 128, 77, 240, 129, 77, 241, 130, 76, 242, 132, 75, 242, 133, 74, 243, 134, 73, 243, 135, 72, 244, 137, 71,
    244, 138, 71, 245, 139, 70, 245, 141, 69, 246, 142, 68, 246, 143, 67, 246, 145, 66, 247, 146, 65, 247, 147, 65,
    248, 149, 64, 248, 150, 63, 248, 152, 62, 249, 153, 61, 249, 154, 60, 250, 156, 59, 250, 157, 58, 250, 159, 58,
    250, 160, 57, 251, 162, 56, 251, 163, 55, 251, 164, 54, 252, 166, 53, 252, 167, 53, 252, 169, 52, 252, 170, 51,
    252, 172, 50, 252, 173, 49, 253, 175, 49, 253, 176, 48, 253, 178, 47, 253, 179, 46, 253, 181, 45, 253, 182, 45,
    253, 184, 44, 253, 185, 43, 253, 187, 43, 253, 188, 42, 253, 190, 41, 253, 192, 41, 253, 193, 40, 253, 195, 40,
    253, 196, 39, 253, 198, 38, 252, 199, 38, 252, 201, 38, 252, 203, 37, 252, 204, 37, 252, 206, 37, 251, 208, 36,
    251, 209, 36, 251, 211, 36, 250, 213, 36, 250, 214, 36, 250, 216, 36, 249, 217, 36, 249, 219, 36, 248, 221, 36,
    248, 223, 36, 247, 224, 36, 247, 226, 37, 246, 228, 37, 246, 229, 37, 245, 231, 38, 245, 233, 38, 244, 234, 38,
    243, 236, 38, 243, 238, 38, 242, 240, 38, 242, 241, 38, 241, 243, 38, 240, 245, 37, 240, 246, 35, 239, 248, 33,
};

// 0.95 * (N - 1) in float64, as numpy 1.19's percentile forms the index of q = 95 / 100
__device__ __forceinline__ double p95_index(int hw) { return __dmul_rn(0.95, (double)(hw - 1)); }

// grid (x: CTAs over the pixels of one image, y: image).  Pass 0 histograms the top byte of every key (bins 0-255); pass
// p > 0 histograms byte 3 - p of the keys whose top p bytes equal rank k's prefix (bins 0-255) or else rank k+1's (bins
// 256-511).  The loop bound is warp-uniform, so that a warp's equal bins are counted by one shared atomic
// (__match_any_sync): a smooth depth map puts most of a warp into one bin, which would otherwise serialise the atomics.
template <bool kFirst>
__global__ void __launch_bounds__(256) depth_hist_kernel(const float* __restrict__ depth, unsigned* __restrict__ scratch,
                                                         int hw, int pass) {
  __shared__ unsigned hist[2 * kDvBins];
  for (int i = threadIdx.x; i < 2 * kDvBins; i += blockDim.x) hist[i] = 0;
  const int n = blockIdx.y, lane = threadIdx.x & 31;
  unsigned* img = scratch + (long long)n * kDvWords;
  unsigned* st = img + kDvHistWords;
  const float* d = depth + (long long)n * hw;
  const int shift = 32 - 8 * pass;                           // pass > 0: the prefix is the key's top 8 * pass bits
  const unsigned pa = kFirst ? 0u : st[kDvPrefA], pb = kFirst ? 0u : st[kDvPrefB];
  __syncthreads();
  unsigned lo = 0;
  bool nan = false;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long base = (long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31); base < hw; base += 4 * stride) {
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long long p = base + lane + j * stride;
      v[j] = p < hw ? __ldg(d + p) : 0.f;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      unsigned bin = kNoBin;
      if (base + lane + j * stride < hw) {
        const float inv = __frcp_rn(v[j]);
        const unsigned key = float_key(inv);
        if (kFirst) {
          nan |= inv != inv;
          if (inv == inv) lo = max(lo, ~key);
          bin = key >> 24;
        } else {
          const unsigned top = key >> shift, digit = (key >> (shift - 8)) & 255u;
          bin = top == pa ? digit : top == pb ? kDvBins + digit : kNoBin;
        }
      }
      const unsigned peers = __match_any_sync(0xffffffffu, bin);
      if (bin != kNoBin && lane == __ffs(peers) - 1) atomicAdd(hist + bin, (unsigned)__popc(peers));
    }
  }
  __syncthreads();
  unsigned* gh = img + pass * 2 * kDvBins;
  for (int i = threadIdx.x; i < 2 * kDvBins; i += blockDim.x)
    if (hist[i]) atomicAdd(gh + i, hist[i]);
  if (kFirst) {
    lo = __reduce_max_sync(0xffffffffu, lo);
    nan = __any_sync(0xffffffffu, nan);
    if (lane == 0) {
      if (lo) atomicMax(st + kDvLo, lo);
      if (nan) atomicOr(st + kDvNan, 1u);
    }
  }
}

// one CTA of 256 threads per image, thread t owning bin t: a block-wide scan of the pass's histogram finds the bins that
// hold ranks k and k+1 and appends them to both prefixes.  After the last pass the prefixes are the keys a and b, and
// thread 0 forms vmax, the fp32 divisor and the image's mode, each float64 / fp32 operation rounded on its own.
__global__ void __launch_bounds__(256) depth_select_kernel(unsigned* __restrict__ scratch, int hw, int pass) {
  unsigned* img = scratch + (long long)blockIdx.x * kDvWords;
  unsigned* st = img + kDvHistWords;
  const unsigned* h = img + pass * 2 * kDvBins;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  unsigned pa = 0, pb = 0, ra, rb;
  if (pass == 0) {
    ra = (unsigned)(int)p95_index(hw);                         // floor of a non-negative index
    rb = min(ra + 1, (unsigned)hw - 1);
  } else {
    pa = st[kDvPrefA]; pb = st[kDvPrefB]; ra = st[kDvRankA]; rb = st[kDvRankB];
  }
  const unsigned ca = h[t], cb = (pass == 0 || pa == pb) ? ca : h[kDvBins + t];
  unsigned ia = ca, ib = cb;                                   // inclusive prefix sums over the bins
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned xa = __shfl_up_sync(0xffffffffu, ia, o), xb = __shfl_up_sync(0xffffffffu, ib, o);
    if (lane >= o) { ia += xa; ib += xb; }
  }
  __shared__ unsigned wsum[2][8], sel[4];
  if (lane == 31) { wsum[0][warp] = ia; wsum[1][warp] = ib; }
  __syncthreads();
  for (int i = 0; i < warp; ++i) { ia += wsum[0][i]; ib += wsum[1][i]; }
  if (ia - ca <= ra && ra < ia) { sel[0] = (pa << 8) | t; sel[1] = ra - (ia - ca); }
  if (ib - cb <= rb && rb < ib) { sel[2] = (pb << 8) | t; sel[3] = rb - (ib - cb); }
  __syncthreads();
  if (t != 0) return;
  if (pass < 3) {
    st[kDvPrefA] = sel[0]; st[kDvRankA] = sel[1]; st[kDvPrefB] = sel[2]; st[kDvRankB] = sel[3];
    return;
  }
  const double idx = p95_index(hw), g = __dsub_rn(idx, (double)(int)idx);
  const double a = key_float(sel[0]), b = key_float(sel[2]);
  const double vmax = __dadd_rn(__dmul_rn(a, __dsub_rn(1.0, g)), __dmul_rn(b, g));
  const double vmin = key_float(~st[kDvLo]);
  unsigned mode = kDvNormal;
  if (st[kDvNan] || vmax != vmax) mode = kDvBlack;
  else if (!(vmin < vmax)) mode = kDvFlat;
  else st[kDvRange] = __float_as_uint(__double2float_rn(__dsub_rn(vmax, vmin)));
  st[kDvMode] = mode;
}

// grid (x: CTAs over the pixels of one image, y: image); the floor table is staged in shared memory as in disp_color_kernel
__global__ void __launch_bounds__(256) depth_color_kernel(const float* __restrict__ depth, const unsigned* __restrict__ scratch,
                                                          uint8_t* __restrict__ out, int w, int hw, long long row_stride,
                                                          long long image_stride) {
  __shared__ uint8_t lut[768];
  for (int i = threadIdx.x; i < 768; i += blockDim.x) lut[i] = kPlasma[i];
  __syncthreads();
  const int n = blockIdx.y;
  const unsigned* st = scratch + (long long)n * kDvWords + kDvHistWords;
  const unsigned mode = __ldg(st + kDvMode);
  const float vmin = key_float(~__ldg(st + kDvLo)), range = __uint_as_float(__ldg(st + kDvRange));
  const float* d = depth + (long long)n * hw;
  uint8_t* img = out + n * image_stride;
  for (long long p = blockIdx.x * blockDim.x + threadIdx.x; p < hw; p += (long long)gridDim.x * blockDim.x) {
    int i = mode == kDvFlat ? 0 : -1;                          // colour index, -1 = black
    if (mode == kDvNormal) {
      const float x = __fmul_rn(__fdiv_rn(__fsub_rn(__frcp_rn(__ldg(d + p)), vmin), range), 256.0f);
      i = x != x ? -1 : x < 0.f ? 0 : x >= 255.f ? 255 : (int)x;
    }
    const int y = (int)p / w, xx = (int)p - y * w;
    uint8_t* o = img + y * row_stride + 3LL * xx;
    if (i < 0) {
      o[0] = o[1] = o[2] = 0;
    } else {
      o[0] = lut[3 * i]; o[1] = lut[3 * i + 1]; o[2] = lut[3 * i + 2];
    }
  }
}

// ---- leaderboard submission payloads (evaluate_flow.py:19-156, evaluate_stereo.py:28-298) ---------------------------------
struct SubmitGeom {
  const float* pred;
  int C, h, w, H, W, top, left, resize;
};

// Value of channel c at payload pixel (Y, X): the unpad crop, or the align-corners resize with the reference's two-step
// rescale ((x * ori) / inf, two roundings; not x * (ori / inf)).
__device__ __forceinline__ float submit_value(const SubmitGeom& g, long long b, int c, int Y, int X) {
  const float* plane = g.pred + (b * g.C + c) * (long long)g.h * g.w;
  if (!g.resize) return __ldg(plane + (long long)(Y + g.top) * g.w + (X + g.left));
  const float v = bilinear_align_corners([&](int y, int x) { return __ldg(plane + (long long)y * g.w + x); }, g.h, g.w, g.H, g.W,
                                         Y, X);
  return c == 0 ? __fdiv_rn(__fmul_rn(v, (float)g.W), (float)g.w) : __fdiv_rn(__fmul_rn(v, (float)g.H), (float)g.h);
}

// numpy's float -> uint16 cast on x86-64 (cvttss2si, then the low 16 bits): truncation toward zero where the result fits
// int32, INT32_MIN (low half 0) for NaN, +-inf and everything else.  __float2int_rz saturates instead, so the range test
// comes first and the conversion only sees values it converts exactly.
__device__ __forceinline__ unsigned numpy_u16(float x) {
  const int t = (x >= -2147483648.0f && x < 2147483648.0f) ? __float2int_rz(x) : (-2147483647 - 1);
  return (unsigned)t & 0xffffu;
}

// The uint16 samples of payload pixel (Y, X): 3 for KITTI flow (R, G, B), 1 for KITTI disparity.
template <int FMT>
__device__ __forceinline__ void submit_png_samples(const SubmitGeom& g, long long b, int Y, int X, unsigned* s) {
  if (FMT == UM_SUBMIT_KITTI_FLOW_PNG) {
    s[0] = numpy_u16(__fadd_rn(__fmul_rn(64.0f, submit_value(g, b, 0, Y, X)), 32768.0f));
    s[1] = numpy_u16(__fadd_rn(__fmul_rn(64.0f, submit_value(g, b, 1, Y, X)), 32768.0f));
    s[2] = 1u;
  } else {
    s[0] = numpy_u16(__fmul_rn(submit_value(g, b, 0, Y, X), 256.0f));
  }
}

// One thread per payload pixel.  PNG formats: the pixel's big-endian bytes minus those of the pixel above (the "Up" filter),
// which the thread recomputes, so rows stay independent; thread X = 0 writes the row's filter byte.
template <int FMT>
__global__ void __launch_bounds__(256) encode_submission_kernel(SubmitGeom g, uint8_t* __restrict__ out, long long sample_stride,
                                                                long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int X = (int)(i % g.W);
  const int Y = (int)((i / g.W) % g.H);
  const long long b = i / ((long long)g.H * g.W);
  uint8_t* dst = out + b * sample_stride;
  if (FMT == UM_SUBMIT_FLO) {
    reinterpret_cast<float2*>(dst)[(long long)Y * g.W + X] = make_float2(submit_value(g, b, 0, Y, X), submit_value(g, b, 1, Y, X));
  } else if (FMT == UM_SUBMIT_PFM) {
    reinterpret_cast<float*>(dst)[(long long)(g.H - 1 - Y) * g.W + X] = submit_value(g, b, 0, Y, X);
  } else {
    constexpr int NS = FMT == UM_SUBMIT_KITTI_FLOW_PNG ? 3 : 1;
    unsigned cur[NS], up[NS];
    submit_png_samples<FMT>(g, b, Y, X, cur);
    if (Y > 0) submit_png_samples<FMT>(g, b, Y - 1, X, up);
    uint8_t* row = dst + (long long)Y * (1 + 2 * NS * (long long)g.W);
    if (X == 0) row[0] = Y > 0 ? 2 : 0;
    uint8_t* px = row + 1 + 2 * NS * (long long)X;
#pragma unroll
    for (int k = 0; k < NS; ++k) {
      unsigned hi = cur[k] >> 8, lo = cur[k] & 0xffu;
      if (Y > 0) { hi -= up[k] >> 8; lo -= up[k] & 0xffu; }
      px[2 * k] = (uint8_t)hi;
      px[2 * k + 1] = (uint8_t)lo;
    }
  }
}

inline int ew_grid(long long n, int block = 256) {
  long long g = (n + block - 1) / block;
  const long long cap = 132LL * 16;      // 132 SMs (H100 SXM) x 16 resident CTAs, grid-stride beyond that
  return (int)(g < cap ? (g > 0 ? g : 1) : cap);
}

}  // namespace

extern "C" {

int um_add_position(const float* x, const float* table, float* out, int32_t n_streams, int32_t h, int32_t w,
                    int32_t wh, int32_t ww, void* stream) {
  UM_REQUIRE(x && table && out && n_streams > 0 && h > 0 && w > 0 && wh > 0 && ww > 0 && h % wh == 0 && w % ww == 0,
             "um_add_position: bad arguments");
  const long long total4 = (long long)n_streams * h * w * 32;
  add_position_kernel<<<ew_grid(total4), 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const float4*>(x), reinterpret_cast<const float4*>(table), reinterpret_cast<float4*>(out), h, w,
      wh, ww, total4);
  return um::check_launch("um_add_position");
}

int um_convex_upsample(const float* flow, const float* mask, float* up, int32_t batch, int32_t h, int32_t w,
                       int32_t flow_dim, int32_t factor, float mult, void* stream) {
  UM_REQUIRE(flow && mask && up && batch > 0 && h > 0 && w > 0 && factor > 0, "um_convex_upsample: bad arguments");
  UM_REQUIRE(flow_dim == 1 || flow_dim == 2, "um_convex_upsample: flow_dim must be 1 or 2");
  const long long total = (long long)batch * h * w * factor * factor;
  convex_upsample_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(flow, mask, up, h, w, flow_dim,
                                                                                          factor, mult, total);
  return um::check_launch("um_convex_upsample");
}

int um_upsample2x(const float* flow, float* out, int32_t batch, int32_t h, int32_t w, int32_t flow_dim, float mult,
                  void* stream) {
  UM_REQUIRE(flow && out && batch > 0 && h > 0 && w > 0 && flow_dim > 0, "um_upsample2x: bad arguments");
  const long long total = (long long)batch * 4 * h * w * flow_dim;
  upsample2x_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(flow, out, h, w, flow_dim, mult, total);
  return um::check_launch("um_upsample2x");
}

int um_resize_bilinear(const float* in, float* out, int32_t batch, int32_t channels, int32_t h_in, int32_t w_in,
                       int32_t h_out, int32_t w_out, const float* scale, int32_t flip_x, void* stream) {
  UM_REQUIRE(in && out && batch > 0 && channels > 0 && channels <= 3 && h_in > 0 && w_in > 0 && h_out > 0 && w_out > 0,
             "um_resize_bilinear: bad arguments (1-3 channels, positive sizes)");
  const long long total = (long long)batch * channels * h_out * w_out;
  const float s0 = scale ? scale[0] : 1.0f, s1 = (scale && channels > 1) ? scale[1] : 1.0f,
              s2 = (scale && channels > 2) ? scale[2] : 1.0f;
  resize_bilinear_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(in, out, channels, h_in, w_in, h_out,
                                                                                          w_out, s0, s1, s2, flip_x, total);
  return um::check_launch("um_resize_bilinear");
}

int um_frames_to_planar(const uint8_t* frames, float* out, int32_t n, int32_t h, int32_t w, int32_t transpose,
                        int32_t h_out, int32_t w_out, void* stream) {
  UM_REQUIRE(frames && out && n > 0 && h > 0 && w > 0 && h_out > 0 && w_out > 0,
             "um_frames_to_planar: bad arguments (positive sizes, non-null buffers)");
  const long long total = (long long)n * h_out * w_out;
  frames_to_planar_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(frames, out, h, w, transpose ? 1 : 0,
                                                                                           h_out, w_out, total);
  return um::check_launch("um_frames_to_planar");
}

int um_frames_to_planar_normalized(const uint8_t* frames, float* out, int32_t n, int32_t h, int32_t w, int32_t h_out,
                                   int32_t w_out, const float* mean, const float* std, void* stream) {
  UM_REQUIRE(frames && out && mean && std && n > 0 && h > 0 && w > 0 && h_out > 0 && w_out > 0,
             "um_frames_to_planar_normalized: bad arguments (positive sizes, non-null buffers, 3 means and stds)");
  const long long total = (long long)n * h_out * w_out;
  frames_to_planar_normalized_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      frames, out, h, w, h_out, w_out, mean[0], mean[1], mean[2], std[0], std[1], std[2], total);
  return um::check_launch("um_frames_to_planar_normalized");
}

int um_flow_to_image(const float* flow, uint8_t* out, int64_t row_stride, int64_t image_stride, float* max_scratch,
                     int32_t n, int32_t h, int32_t w, void* stream) {
  UM_REQUIRE(flow && out && max_scratch && n > 0 && h > 0 && w > 0, "um_flow_to_image: bad arguments");
  UM_REQUIRE(row_stride >= 3LL * w && image_stride >= row_stride * h,
             "um_flow_to_image: row_stride must cover 3*w bytes and image_stride h rows");
  cudaStream_t st = (cudaStream_t)stream;
  const long long hw = (long long)h * w;
  if (cudaMemsetAsync(max_scratch, 0, sizeof(float) * n, st) != cudaSuccess) return um::check_launch("um_flow_to_image");
  long long bx = (hw + 255) / 256;
  const long long cap = (132LL * 8 + n - 1) / n;          // about 8 CTAs per SM over the whole batch, grid-stride beyond
  bx = bx < cap ? bx : cap;
  flow_maxrad_kernel<<<dim3((unsigned)(bx > 0 ? bx : 1), (unsigned)n), 256, 0, st>>>(flow, reinterpret_cast<unsigned*>(max_scratch), hw);
  if (int rc = um::check_launch("um_flow_to_image")) return rc;
  const long long total = (long long)n * hw;
  flow_color_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(flow, reinterpret_cast<const unsigned*>(max_scratch), out, w,
                                                                     hw, row_stride, image_stride, total);
  return um::check_launch("um_flow_to_image");
}

int um_disparity_to_image(const float* disp, uint8_t* out, int64_t row_stride, int64_t image_stride, float* minmax_scratch,
                          int32_t n, int32_t h, int32_t w, void* stream) {
  UM_REQUIRE(disp && out && minmax_scratch && n > 0 && h > 0 && w > 0, "um_disparity_to_image: bad arguments");
  UM_REQUIRE((long long)h * w <= 0x7fffffffLL, "um_disparity_to_image: an image has at most 2^31 - 1 pixels");
  UM_REQUIRE(row_stride >= 3LL * w && image_stride >= row_stride * h,
             "um_disparity_to_image: row_stride must cover 3*w bytes and image_stride h rows");
  cudaStream_t st = (cudaStream_t)stream;
  const int hw = h * w;
  unsigned* lo = reinterpret_cast<unsigned*>(minmax_scratch);
  unsigned* hi = lo + n;
  if (cudaMemsetAsync(minmax_scratch, 0, sizeof(float) * 2 * n, st) != cudaSuccess)
    return um::check_launch("um_disparity_to_image");
  const long long per_image = ((long long)um::device_sm_count() * 8 + n - 1) / n;   // ~8 CTAs per SM over the batch
  long long bx = ((long long)hw + 1023) / 1024;                                     // 4 pixels per thread and pass
  bx = bx < per_image ? bx : per_image;
  disp_minmax_kernel<<<dim3((unsigned)(bx > 0 ? bx : 1), (unsigned)n), 256, 0, st>>>(disp, lo, hi, hw);
  if (int rc = um::check_launch("um_disparity_to_image")) return rc;
  long long cx = ((long long)hw + 255) / 256;
  cx = cx < 2 * per_image ? cx : 2 * per_image;
  disp_color_kernel<<<dim3((unsigned)cx, (unsigned)n), 256, 0, st>>>(disp, lo, hi, out, w, hw, row_stride, image_stride);
  return um::check_launch("um_disparity_to_image");
}

int um_depth_to_image(const float* depth, uint8_t* out, int64_t row_stride, int64_t image_stride, void* scratch, int32_t n,
                      int32_t h, int32_t w, void* stream) {
  UM_REQUIRE(depth && out && scratch && n > 0 && h > 0 && w > 0, "um_depth_to_image: bad arguments");
  UM_REQUIRE((long long)h * w <= 0x7fffffffLL, "um_depth_to_image: an image has at most 2^31 - 1 pixels");
  UM_REQUIRE(row_stride >= 3LL * w && image_stride >= row_stride * h,
             "um_depth_to_image: row_stride must cover 3*w bytes and image_stride h rows");
  static_assert(kDvWords == 2056, "the header states the scratch size");
  cudaStream_t st = (cudaStream_t)stream;
  const int hw = h * w;
  unsigned* words = reinterpret_cast<unsigned*>(scratch);
  if (cudaMemsetAsync(scratch, 0, sizeof(unsigned) * kDvWords * n, st) != cudaSuccess)
    return um::check_launch("um_depth_to_image");
  const long long per_image = ((long long)um::device_sm_count() * 8 + n - 1) / n;   // ~8 CTAs per SM over the batch
  long long bx = ((long long)hw + 1023) / 1024;                                     // 4 pixels per thread and pass
  bx = bx < per_image ? bx : per_image;
  const dim3 grid((unsigned)(bx > 0 ? bx : 1), (unsigned)n);
  for (int pass = 0; pass < 4; ++pass) {
    if (pass == 0) depth_hist_kernel<true><<<grid, 256, 0, st>>>(depth, words, hw, pass);
    else depth_hist_kernel<false><<<grid, 256, 0, st>>>(depth, words, hw, pass);
    if (int rc = um::check_launch("um_depth_to_image")) return rc;
    depth_select_kernel<<<(unsigned)n, 256, 0, st>>>(words, hw, pass);
    if (int rc = um::check_launch("um_depth_to_image")) return rc;
  }
  long long cx = ((long long)hw + 255) / 256;
  cx = cx < 2 * per_image ? cx : 2 * per_image;
  depth_color_kernel<<<dim3((unsigned)cx, (unsigned)n), 256, 0, st>>>(depth, words, out, w, hw, row_stride, image_stride);
  return um::check_launch("um_depth_to_image");
}

int um_encode_submission(const float* pred, int32_t batch, int32_t channels, int32_t h, int32_t w, int32_t geometry,
                         int32_t top, int32_t left, int32_t out_h, int32_t out_w, int32_t format, uint8_t* out,
                         int64_t sample_stride, void* stream) {
  UM_REQUIRE(pred && out && batch > 0 && h > 0 && w > 0 && out_h > 0 && out_w > 0, "um_encode_submission: bad arguments");
  UM_REQUIRE(format >= UM_SUBMIT_FLO && format <= UM_SUBMIT_PFM, "um_encode_submission: unknown format %d", format);
  const bool flow = format == UM_SUBMIT_FLO || format == UM_SUBMIT_KITTI_FLOW_PNG;
  UM_REQUIRE(channels == (flow ? 2 : 1), "um_encode_submission: format %d needs %d channels", format, flow ? 2 : 1);
  UM_REQUIRE(geometry == UM_SUBMIT_RESIZE ||
                 (geometry == UM_SUBMIT_CROP && top >= 0 && left >= 0 && top + out_h <= h && left + out_w <= w),
             "um_encode_submission: the crop must lie inside the prediction");
  const long long pixels = (long long)out_h * out_w;
  const long long bytes = format == UM_SUBMIT_FLO ? 8 * pixels
                        : format == UM_SUBMIT_PFM ? 4 * pixels
                        : (long long)out_h * (1 + (format == UM_SUBMIT_KITTI_FLOW_PNG ? 6LL : 2LL) * out_w);
  UM_REQUIRE(sample_stride >= bytes, "um_encode_submission: sample_stride must cover the %lld payload bytes", bytes);
  const int align = format == UM_SUBMIT_FLO ? 8 : (format == UM_SUBMIT_PFM ? 4 : 1);
  UM_REQUIRE((uintptr_t)out % align == 0 && sample_stride % align == 0,
             "um_encode_submission: out and sample_stride must be %d-byte aligned for this format", align);
  const SubmitGeom g{pred, channels, h, w, out_h, out_w, top, left, geometry == UM_SUBMIT_RESIZE ? 1 : 0};
  const long long total = (long long)batch * pixels;
  const unsigned grid = (unsigned)((total + 255) / 256);
  cudaStream_t st = (cudaStream_t)stream;
  switch (format) {
    case UM_SUBMIT_FLO: encode_submission_kernel<UM_SUBMIT_FLO><<<grid, 256, 0, st>>>(g, out, sample_stride, total); break;
    case UM_SUBMIT_KITTI_FLOW_PNG:
      encode_submission_kernel<UM_SUBMIT_KITTI_FLOW_PNG><<<grid, 256, 0, st>>>(g, out, sample_stride, total);
      break;
    case UM_SUBMIT_KITTI_DISP_PNG:
      encode_submission_kernel<UM_SUBMIT_KITTI_DISP_PNG><<<grid, 256, 0, st>>>(g, out, sample_stride, total);
      break;
    default: encode_submission_kernel<UM_SUBMIT_PFM><<<grid, 256, 0, st>>>(g, out, sample_stride, total); break;
  }
  return um::check_launch("um_encode_submission");
}

}  // extern "C"
