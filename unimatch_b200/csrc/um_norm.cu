// InstanceNorm2d (eps 1e-5, no affine, biased variance; backbone.py:7,41) on channel-last fp32 maps, as three
// bandwidth-bound passes: per-(image, channel) pivot-shifted partial sums -> mean / rstd -> fused normalise (+ReLU) (+residual,
// itself optionally normalised) (+ReLU) writing fp32 and/or the fp16 (hi, lo) planes the tensor-core convolution reads.
#include "um_common.cuh"
#include "um_tc.cuh"

namespace {

constexpr int CHUNKS = 64;

// Per-(image, channel) pivot: the fp32 mean of the first min(hw, 16) pixels, summed in pixel order.  The partial sums are
// of x - pivot, so E[x^2] - mean^2 no longer cancels when |mean| >> std (a channel with |mean| / std = 100 would otherwise
// lose ~1e-4 of rstd to the fp32 sums).  Both kernels form it with the same instructions, so they agree to the bit.
__device__ __forceinline__ float4 in_pivot(const float* __restrict__ x, long long ld, int hw, int n, int c4) {
  const int np = hw < 16 ? hw : 16;
  float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int r = 0; r < np; ++r) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(x + ((long long)n * hw + r) * ld) + c4);
    p.x += v.x; p.y += v.y; p.z += v.z; p.w += v.w;
  }
  const float inv = 1.0f / (float)np;
  return make_float4(p.x * inv, p.y * inv, p.z * inv, p.w * inv);
}

// grid (CHUNKS, N); 256 threads = (C/4 float4 lanes) x row lanes.  partial[n][chunk][2][C]: sums of x - pivot and of its square
__global__ void __launch_bounds__(256) in_partial_kernel(const float* __restrict__ x, long long ld, int hw, int C,
                                                         float* __restrict__ partial) {
  extern __shared__ float sm[];                 // [2][rows_per_iter][C]
  const int n = blockIdx.y, chunk = blockIdx.x;
  const int c4n = C >> 2;
  const int rlanes = 256 / c4n;
  const int c4 = threadIdx.x % c4n, rl = threadIdx.x / c4n;
  const int rows_per_chunk = (hw + CHUNKS - 1) / CHUNKS;
  const int r0 = chunk * rows_per_chunk, r1 = min(hw, r0 + rows_per_chunk);
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f), q = make_float4(0.f, 0.f, 0.f, 0.f);
  if (rl < rlanes) {
    const float4 pv = in_pivot(x, ld, hw, n, c4);
    for (int r = r0 + rl; r < r1; r += rlanes) {
      float4 v = __ldg(reinterpret_cast<const float4*>(x + ((long long)n * hw + r) * ld) + c4);
      v.x -= pv.x; v.y -= pv.y; v.z -= pv.z; v.w -= pv.w;
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
      q.x = fmaf(v.x, v.x, q.x); q.y = fmaf(v.y, v.y, q.y); q.z = fmaf(v.z, v.z, q.z); q.w = fmaf(v.w, v.w, q.w);
    }
  }
  float* ss = sm;
  float* qs = sm + rlanes * C;
  if (rl < rlanes) {
    reinterpret_cast<float4*>(ss + rl * C)[c4] = s;
    reinterpret_cast<float4*>(qs + rl * C)[c4] = q;
  }
  __syncthreads();
  if (threadIdx.x < C) {
    float a = 0.f, b = 0.f;
    for (int i = 0; i < rlanes; ++i) { a += ss[i * C + threadIdx.x]; b += qs[i * C + threadIdx.x]; }
    float* dst = partial + (((long long)n * CHUNKS + chunk) * 2) * C;
    dst[threadIdx.x] = a;
    dst[C + threadIdx.x] = b;
  }
}

// stats[n][0][c] = mean, stats[n][1][c] = rstd; final combination in double
__global__ void in_finalize_kernel(const float* __restrict__ x, long long ld, const float* __restrict__ partial,
                                   float* __restrict__ stats, int hw, int C, int total) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int n = i / C, c = i - n * C;
  const float4 pv = in_pivot(x, ld, hw, n, c >> 2);
  const float piv = (c & 3) == 0 ? pv.x : (c & 3) == 1 ? pv.y : (c & 3) == 2 ? pv.z : pv.w;
  double s = 0.0, q = 0.0;
  for (int k = 0; k < CHUNKS; ++k) {
    const float* p = partial + (((long long)n * CHUNKS + k) * 2) * C;
    s += (double)p[c]; q += (double)p[C + c];
  }
  const double dm = s / hw;                      // mean - pivot
  double var = q / hw - dm * dm;
  if (var < 0.0) var = 0.0;
  stats[((long long)n * 2) * C + c] = (float)((double)piv + dm);
  stats[((long long)n * 2 + 1) * C + c] = (float)(1.0 / sqrt(var + 1e-5));
}

struct ApplyParams {
  const float* a; long long ld_a; const float* st_a; int relu_a;
  const float* res; long long ld_res; const float* st_res; int relu_out;
  float* out; long long ld_o;
  __half* split; int cp, off; long long plane;
  int hw, C; long long total4;
};

__device__ __forceinline__ uint32_t pk(__half a, __half b) {
  return (uint32_t)__half_as_ushort(a) | ((uint32_t)__half_as_ushort(b) << 16);
}

__global__ void __launch_bounds__(256) in_apply_kernel(ApplyParams p) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const int c4n = p.C >> 2;
  for (; i < p.total4; i += stride) {
    const int c4 = (int)(i % c4n);
    const long long row = i / c4n;
    const int n = (int)(row / p.hw);
    float4 v = __ldg(reinterpret_cast<const float4*>(p.a + row * p.ld_a) + c4);
    if (p.st_a) {
      const float4 m = __ldg(reinterpret_cast<const float4*>(p.st_a + ((long long)n * 2) * p.C) + c4);
      const float4 r = __ldg(reinterpret_cast<const float4*>(p.st_a + ((long long)n * 2 + 1) * p.C) + c4);
      v.x = (v.x - m.x) * r.x; v.y = (v.y - m.y) * r.y; v.z = (v.z - m.z) * r.z; v.w = (v.w - m.w) * r.w;
    }
    if (p.relu_a) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
    if (p.res) {
      float4 u = __ldg(reinterpret_cast<const float4*>(p.res + row * p.ld_res) + c4);
      if (p.st_res) {
        const float4 m = __ldg(reinterpret_cast<const float4*>(p.st_res + ((long long)n * 2) * p.C) + c4);
        const float4 r = __ldg(reinterpret_cast<const float4*>(p.st_res + ((long long)n * 2 + 1) * p.C) + c4);
        u.x = (u.x - m.x) * r.x; u.y = (u.y - m.y) * r.y; u.z = (u.z - m.z) * r.z; u.w = (u.w - m.w) * r.w;
      }
      v.x += u.x; v.y += u.y; v.z += u.z; v.w += u.w;
    }
    if (p.relu_out) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
    if (p.out) reinterpret_cast<float4*>(p.out + row * p.ld_o)[c4] = v;
    if (p.split) {
      __half h[4], l[4];
      um::tc::split_f16(v.x, &h[0], &l[0]); um::tc::split_f16(v.y, &h[1], &l[1]);
      um::tc::split_f16(v.z, &h[2], &l[2]); um::tc::split_f16(v.w, &h[3], &l[3]);
      __half* d = p.split + row * p.cp + p.off + c4 * 4;
      *reinterpret_cast<uint2*>(d) = make_uint2(pk(h[0], h[1]), pk(h[2], h[3]));
      *reinterpret_cast<uint2*>(d + p.plane) = make_uint2(pk(l[0], l[1]), pk(l[2], l[3]));
    }
  }
}

}  // namespace

extern "C" {

int64_t um_instance_norm_scratch_floats(int32_t n, int32_t c) { return (int64_t)n * CHUNKS * 2 * c; }

int um_instance_norm_stats(const float* x, int64_t ld, int32_t n, int32_t hw, int32_t c, float* scratch, float* stats,
                           void* stream) {
  UM_REQUIRE(x && scratch && stats && n > 0 && hw > 0 && c > 0 && c % 4 == 0 && c <= 256 && ld % 4 == 0 && ld >= c,
             "um_instance_norm_stats: bad arguments (channels must be a multiple of 4, <= 256)");
  const int rlanes = 256 / (c / 4);
  UM_REQUIRE(rlanes >= 1, "um_instance_norm_stats: too many channels");
  cudaStream_t st = (cudaStream_t)stream;
  in_partial_kernel<<<dim3(CHUNKS, n), 256, 2 * rlanes * c * sizeof(float), st>>>(x, ld, hw, c, scratch);
  int rc = um::check_launch("um_instance_norm_stats(partial)");
  if (rc) return rc;
  const int total = n * c;
  in_finalize_kernel<<<(total + 127) / 128, 128, 0, st>>>(x, ld, scratch, stats, hw, c, total);
  return um::check_launch("um_instance_norm_stats(finalize)");
}

int um_instance_norm_apply(const float* a, int64_t ld_a, const float* stats_a, int32_t relu_a, const float* res,
                           int64_t ld_res, const float* stats_res, int32_t relu_out, float* out_f32, int64_t ld_o,
                           void* out_split, int32_t cp, int32_t off, int32_t n, int32_t hw, int32_t c, void* stream) {
  UM_REQUIRE(a && n > 0 && hw > 0 && c > 0 && c % 4 == 0 && ld_a % 4 == 0, "um_instance_norm_apply: bad arguments");
  UM_REQUIRE(out_f32 || out_split, "um_instance_norm_apply: no output");
  UM_REQUIRE(!res || ld_res % 4 == 0, "um_instance_norm_apply: bad residual stride");
  UM_REQUIRE(!out_f32 || ld_o % 4 == 0, "um_instance_norm_apply: bad output stride");
  UM_REQUIRE(!out_split || (cp % 4 == 0 && off % 4 == 0 && off + c <= cp), "um_instance_norm_apply: bad split layout");
  ApplyParams p{};
  p.a = a; p.ld_a = ld_a; p.st_a = stats_a; p.relu_a = relu_a;
  p.res = res; p.ld_res = ld_res; p.st_res = stats_res; p.relu_out = relu_out;
  p.out = out_f32; p.ld_o = ld_o;
  p.split = reinterpret_cast<__half*>(out_split); p.cp = cp; p.off = off; p.plane = (long long)n * hw * cp;
  p.hw = hw; p.C = c; p.total4 = (long long)n * hw * (c / 4);
  long long blocks = (p.total4 + 255) / 256;
  if (blocks > 132LL * 32) blocks = 132LL * 32;
  in_apply_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(p);
  return um::check_launch("um_instance_norm_apply");
}

}  // extern "C"
