// Small fused glue kernels on the matching path: position add, LayerNorm(+residual), convex upsampling,
// x2 bilinear flow upsampling, GRU gate math.  All channel-last, all bandwidth-bound, all vectorised (float4).
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

// ---- LayerNorm over 128 channels + residual (transformer.py:137-144): one warp per row -------------------
__global__ void __launch_bounds__(256) layernorm_residual_kernel(const float* __restrict__ x, const float* __restrict__ res,
                                                                 const float* __restrict__ gamma, const float* __restrict__ beta,
                                                                 float* __restrict__ out, long long rows, long long ldx,
                                                                 long long ldr, long long ldo) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float4 v = __ldg(reinterpret_cast<const float4*>(x + row * ldx) + lane);
  float s = (v.x + v.y) + (v.z + v.w);
  s = um::warp_sum(s);
  const float mean = s * (1.0f / 128.0f);
  const float dx = v.x - mean, dy = v.y - mean, dz = v.z - mean, dw = v.w - mean;
  float q = (dx * dx + dy * dy) + (dz * dz + dw * dw);
  q = um::warp_sum(q);
  const float rstd = rsqrtf(q * (1.0f / 128.0f) + 1e-5f);
  const float4 g = __ldg(reinterpret_cast<const float4*>(gamma) + lane);
  const float4 b = __ldg(reinterpret_cast<const float4*>(beta) + lane);
  float4 o = make_float4(dx * rstd * g.x + b.x, dy * rstd * g.y + b.y, dz * rstd * g.z + b.z, dw * rstd * g.w + b.w);
  if (res) {
    const float4 r = __ldg(reinterpret_cast<const float4*>(res + row * ldr) + lane);
    o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
  }
  reinterpret_cast<float4*>(out + row * ldo)[lane] = o;
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

// ---- SepConvGRU gate math (reg_refine.py:37-52) -------------------------------------------------------------
__device__ __forceinline__ float sigmoidf(float x) { return 1.0f / (1.0f + expf(-x)); }

// rows of 128 channels with independent row strides (the z|r pre-activations come out of one fused conv)
__global__ void __launch_bounds__(256) gru_rh_kernel(const float* __restrict__ r, long long ldr, const float* __restrict__ hh,
                                                     long long ldh, float* __restrict__ rh, long long ldo, long long rows) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < rows * 32; i += stride) {
    const long long row = i >> 5; const int c4 = (int)(i & 31);
    const float4 a = __ldg(reinterpret_cast<const float4*>(r + row * ldr) + c4);
    const float4 b = __ldg(reinterpret_cast<const float4*>(hh + row * ldh) + c4);
    reinterpret_cast<float4*>(rh + row * ldo)[c4] =
        make_float4(sigmoidf(a.x) * b.x, sigmoidf(a.y) * b.y, sigmoidf(a.z) * b.z, sigmoidf(a.w) * b.w);
  }
}

__device__ __forceinline__ float gru_mix(float z, float q, float h) {
  const float s = sigmoidf(z);
  return (1.0f - s) * h + s * tanhf(q);
}

__global__ void __launch_bounds__(256) gru_update_kernel(const float* __restrict__ z, long long ldz, const float* __restrict__ q,
                                                         long long ldq, const float* __restrict__ hh, long long ldh,
                                                         float* __restrict__ out, long long ldo, long long rows) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < rows * 32; i += stride) {
    const long long row = i >> 5; const int c4 = (int)(i & 31);
    const float4 a = __ldg(reinterpret_cast<const float4*>(z + row * ldz) + c4);
    const float4 b = __ldg(reinterpret_cast<const float4*>(q + row * ldq) + c4);
    const float4 c = __ldg(reinterpret_cast<const float4*>(hh + row * ldh) + c4);
    reinterpret_cast<float4*>(out + row * ldo)[c4] =
        make_float4(gru_mix(a.x, b.x, c.x), gru_mix(a.y, b.y, c.y), gru_mix(a.z, b.z, c.z), gru_mix(a.w, b.w, c.w));
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

int um_layernorm_residual(const float* x, const float* residual, const float* gamma, const float* beta, float* out,
                          int64_t rows, int64_t ldx, int64_t ldr, int64_t ldo, void* stream) {
  UM_REQUIRE(x && gamma && beta && out && rows > 0, "um_layernorm_residual: bad arguments");
  UM_REQUIRE(ldx % 4 == 0 && ldo % 4 == 0 && (!residual || ldr % 4 == 0), "um_layernorm_residual: strides must be multiples of 4");
  layernorm_residual_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>(x, residual, gamma, beta, out,
                                                                                         rows, ldx, ldr, ldo);
  return um::check_launch("um_layernorm_residual");
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

int um_gru_rh(const float* r_pre, int64_t ldr, const float* h, int64_t ldh, float* rh, int64_t ldo, int64_t rows,
              void* stream) {
  UM_REQUIRE(r_pre && h && rh && rows > 0 && ldr % 4 == 0 && ldh % 4 == 0 && ldo % 4 == 0, "um_gru_rh: bad arguments");
  gru_rh_kernel<<<ew_grid(rows * 32), 256, 0, (cudaStream_t)stream>>>(r_pre, ldr, h, ldh, rh, ldo, rows);
  return um::check_launch("um_gru_rh");
}

int um_gru_update(const float* z_pre, int64_t ldz, const float* q_pre, int64_t ldq, const float* h, int64_t ldh,
                  float* h_out, int64_t ldo, int64_t rows, void* stream) {
  UM_REQUIRE(z_pre && q_pre && h && h_out && rows > 0 && ldz % 4 == 0 && ldq % 4 == 0 && ldh % 4 == 0 && ldo % 4 == 0,
             "um_gru_update: bad arguments");
  gru_update_kernel<<<ew_grid(rows * 32), 256, 0, (cudaStream_t)stream>>>(z_pre, ldz, q_pre, ldq, h, ldh, h_out, ldo, rows);
  return um::check_launch("um_gru_update");
}

}  // extern "C"
