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
// out[b,c,Y,X] = scale[c] * bilinear(in[b,c], Y (hi-1)/(ho-1), X (wi-1)/(wo-1)), ATen's upsample_bilinear2d arithmetic
// (area_pixel_compute_source_index with align_corners, lambda weights, the same order of operations).  `flip_x`: the
// OUTPUT is mirrored horizontally (torchvision hflip of evaluate_stereo.py:789-796 folded into the same pass).
__global__ void __launch_bounds__(256) resize_bilinear_kernel(const float* __restrict__ in, float* __restrict__ out, int C,
                                                              int hi, int wi, int ho, int wo, float s0, float s1, float s2,
                                                              int flip_x, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int X = (int)(i % wo);
  const int Y = (int)((i / wo) % ho);
  const long long bc = i / ((long long)ho * wo);
  const int c = (int)(bc % C);
  const float sy = (ho > 1) ? (float)(hi - 1) / (float)(ho - 1) : 0.f;
  const float sx = (wo > 1) ? (float)(wi - 1) / (float)(wo - 1) : 0.f;
  const float fy = sy * (float)Y, fx = sx * (float)X;
  const int y0 = (int)fy, x0 = (int)fx;
  const int y1 = y0 + ((y0 < hi - 1) ? 1 : 0), x1 = x0 + ((x0 < wi - 1) ? 1 : 0);
  const float ly = fy - (float)y0, lx = fx - (float)x0;
  const float hy = 1.0f - ly, hx = 1.0f - lx;
  const float* base = in + bc * (long long)hi * wi;
  const float v00 = __ldg(base + (long long)y0 * wi + x0), v01 = __ldg(base + (long long)y0 * wi + x1);
  const float v10 = __ldg(base + (long long)y1 * wi + x0), v11 = __ldg(base + (long long)y1 * wi + x1);
  const float sc = c == 0 ? s0 : (c == 1 ? s1 : s2);
  const float v = hy * (hx * v00 + lx * v01) + ly * (hx * v10 + lx * v11);
  const int Xo = flip_x ? wo - 1 - X : X;
  out[(bc * ho + Y) * (long long)wo + Xo] = sc == 1.0f ? v : v * sc;
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
