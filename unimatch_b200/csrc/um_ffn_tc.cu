// Fused transformer FFN on the Hopper tensor cores (wgmma + TMA), fp32-faithful (fp16 hi/lo split operands):
//
//   out = residual + LayerNorm( GELU( [source | message] W1^T ) W2^T )            transformer.py:137-144
//
// Run as two GEMM launches (um_conv2d_tc: FFN1 256 -> 1024 + GELU, then FFN2 1024 -> 128 + LN), the 1024-wide hidden
// activation travels through HBM as fp16 (hi, lo) planes -- 4 KB per token row, 1.6 GB at 8 pairs of 480x832.  Here it
// never leaves the registers: one CTA per 128-row tile, warp-specialised:
//
//   warp 8          TMA producer: the tile's [source | message] planes (128 KB, resident for the tile), then a 5-slot ring
//                   of 16 KB weight tiles in the order the consumers use them: W1(c) as 4 K-slices, W2(c) as 2 row halves
//   warpgroups 0-1  consumers, 64 rows each, for every 64-wide hidden chunk c:
//                   H_c = X W1_c^T (48 wgmma 64x64x16, both operands in shared memory) into registers -> exact-erf GELU ->
//                   (hi, lo) fp16 pairs, which are already the register A operand of O += P_c W2_c^T (24 wgmma 64x64x16);
//                   after the last chunk: LayerNorm (two-pass statistics over the 4 threads of a row) + residual on O,
//                   fp32 rows and / or fp16 planes out.
#include "um_common.cuh"
#include "um_tc.cuh"

namespace um {

using namespace tc;

namespace {

constexpr int NTHREADS = 288;                        // 2 consumer warpgroups (warps 0-7) + one TMA producer warp (warp 8)
constexpr int PRODUCER = 8;
constexpr int HC = 64;                               // hidden channels per chunk
constexpr uint32_t X_BYTES = 4 * 32768;              // 4 K-slices x (hi, lo) x [128 rows x 64 ch]
constexpr uint32_t SLOT_BYTES = 16384;               // (hi, lo) x [64 weight rows x 64 k]
constexpr int NSLOT = 5;
constexpr uint32_t OFF_RING = X_BYTES;
constexpr uint32_t OFF_BAR = OFF_RING + NSLOT * SLOT_BYTES;        // 212992
constexpr uint32_t SMEM_BYTES = OFF_BAR + 256;
static_assert(SMEM_BYTES <= 232448, "shared memory budget");

struct FfnParams {
  int nchunk, hidden;
  const float* residual; long long ld_res;
  const float* gamma; const float* beta;
  float* out_f32; long long ld_f32;
  __half* out_split; long long split_plane;
};

__global__ void __launch_bounds__(NTHREADS, 1)
ffn_tc_kernel(const __grid_constant__ CUtensorMap map_x0, const __grid_constant__ CUtensorMap map_x1,
              const __grid_constant__ CUtensorMap map_w1, const __grid_constant__ CUtensorMap map_w2, FfnParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
  uint64_t* x_full = bars;
  uint64_t* full = bars + 1;                 // [NSLOT]
  uint64_t* empty = bars + 1 + NSLOT;        // [NSLOT]: one arrival per consumer warp
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = blockIdx.x;               // rows [128 tile, 128 tile + 128)

  if (threadIdx.x == 0) {
    mbar_init(x_full, 1);
    for (int i = 0; i < NSLOT; ++i) { mbar_init(full + i, 1); mbar_init(empty + i, 8); }
    fence_barrier_init();
  }
  if (warp == PRODUCER && lane == 0) {
    tma_prefetch_desc(&map_x0); tma_prefetch_desc(&map_x1); tma_prefetch_desc(&map_w1); tma_prefetch_desc(&map_w2);
  }
  __syncthreads();

  if (warp == PRODUCER) {
    if (elect_one()) {
      mbar_arrive_expect_tx(x_full, X_BYTES);
#pragma unroll
      for (int kc = 0; kc < 4; ++kc)                 // K slice kc: source kc / 2, channels 64 (kc % 2) ...
#pragma unroll
        for (int part = 0; part < 2; ++part)
          tma_load_4d(smem + (kc * 2 + part) * 16384, kc < 2 ? &map_x0 : &map_x1, x_full, (kc & 1) * 64, 0, tile * 8, part);
    }
    __syncwarp();
    int it = 0;
    for (int c = 0; c < p.nchunk; ++c)
      for (int q = 0; q < 6; ++q, ++it) {
        const int s = it % NSLOT;
        mbar_wait_inline(empty + s, ((it / NSLOT) & 1) ^ 1);
        uint8_t* slot = smem + OFF_RING + s * SLOT_BYTES;
        if (elect_one()) {
          mbar_arrive_expect_tx(full + s, SLOT_BYTES);
#pragma unroll
          for (int part = 0; part < 2; ++part) {
            if (q < 4) tma_load_2d(slot + part * 8192, &map_w1, full + s, q * 64, part * p.hidden + c * HC);
            else tma_load_2d(slot + part * 8192, &map_w2, full + s, c * HC, part * 128 + (q - 4) * 64);
          }
        }
        __syncwarp();
      }
    return;
  }

  // =============================== consumers ===============================
  const int wg = warp >> 2;
  const int fr = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's rows fr and fr + 8 (MMA fragment layout)
  const int fc = 2 * (lane & 3);                            // ... and columns 8 j + fc + {0, 1}
  const uint32_t x_base = smem_u32(smem) + wg * 8192;
  const int pa[3] = {1, 0, 0}, pb[3] = {0, 1, 0};          // lo*hi, hi*lo, hi*hi
  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  mbar_wait_inline(x_full, 0);
  int it = 0;
  for (int c = 0; c < p.nchunk; ++c) {
    // ---- H_c = X W1_c^T: 64 rows x 64 hidden channels, K = 256 in 4 slots ----
    float h[32];
    int sl[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      sl[q] = (it + q) % NSLOT;
      mbar_wait_inline(full + sl[q], ((it + q) / NSLOT) & 1);
    }
    fence_acc(h);
    wgmma_fence();
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint32_t sb = smem_u32(smem + OFF_RING + sl[q] * SLOT_BYTES);
#pragma unroll
      for (int cc = 0; cc < 3; ++cc)
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
          wgmma_ss<64>(h, desc_kmajor(x_base + (q * 2 + pa[cc]) * 16384 + ks * 32), desc_kmajor(sb + pb[cc] * 8192 + ks * 32),
                       (q | cc | ks) != 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_acc(h);
    __syncwarp();
    if (lane == 0)
#pragma unroll
      for (int q = 0; q < 4; ++q) mbar_arrive(empty + sl[q]);
    it += 4;
    // ---- GELU -> fp16 (hi, lo) pairs in the A-operand layout of the next MMA ----
    uint32_t ph[16], pl[16];
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
        split_f16x2(act_gelu(h[4 * jj + 2 * hh]), act_gelu(h[4 * jj + 2 * hh + 1]), &ph[2 * jj + hh], &pl[2 * jj + hh]);
    // ---- O += P_c W2_c^T: output channels [0, 64) and [64, 128) from one slot each ----
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      sl[q] = (it + q) % NSLOT;
      mbar_wait_inline(full + sl[q], ((it + q) / NSLOT) & 1);
    }
    fence_acc(o);
    wgmma_fence();
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const uint32_t sb = smem_u32(smem + OFF_RING + sl[q] * SLOT_BYTES);
      float (&oq)[32] = *reinterpret_cast<float (*)[32]>(o + 32 * q);
#pragma unroll
      for (int cc = 0; cc < 3; ++cc)
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
          const uint32_t* pp = cc == 0 ? pl : ph;
          const uint32_t a[4] = {pp[4 * ks], pp[4 * ks + 1], pp[4 * ks + 2], pp[4 * ks + 3]};
          wgmma_rs_n64(oq, a, desc_kmajor(sb + (cc == 1 ? 8192 : 0) + ks * 32), true);
        }
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_acc(o);
    __syncwarp();
    if (lane == 0) { mbar_arrive(empty + sl[0]); mbar_arrive(empty + sl[1]); }
    it += 2;
  }

  // ---- LayerNorm (+ residual) on the thread's two rows; a row's 128 channels are spread over 4 lanes ----
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const long long row = (long long)tile * 128 + fr + 8 * hh;
    float sum = 0.f;
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) sum += o[4 * jj + 2 * hh] + o[4 * jj + 2 * hh + 1];
    sum += __shfl_xor_sync(0xffffffffu, sum, 1);
    sum += __shfl_xor_sync(0xffffffffu, sum, 2);
    const float mean = sum * (1.0f / 128.0f);
    float sq = 0.f;
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
      const float d0 = o[4 * jj + 2 * hh] - mean, d1 = o[4 * jj + 2 * hh + 1] - mean;
      sq = fmaf(d0, d0, fmaf(d1, d1, sq));
    }
    sq += __shfl_xor_sync(0xffffffffu, sq, 1);
    sq += __shfl_xor_sync(0xffffffffu, sq, 2);
    const float rstd = rsqrtf(sq * (1.0f / 128.0f) + 1e-5f);
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
      const int col = 8 * jj + fc;
      float y0 = (o[4 * jj + 2 * hh] - mean) * rstd * __ldg(p.gamma + col) + __ldg(p.beta + col);
      float y1 = (o[4 * jj + 2 * hh + 1] - mean) * rstd * __ldg(p.gamma + col + 1) + __ldg(p.beta + col + 1);
      if (p.residual) {
        const float2 r = __ldg(reinterpret_cast<const float2*>(p.residual + row * p.ld_res + col));
        y0 += r.x; y1 += r.y;
      }
      if (p.out_f32) *reinterpret_cast<float2*>(p.out_f32 + row * p.ld_f32 + col) = make_float2(y0, y1);
      if (p.out_split) {
        uint32_t hi, lo;
        split_f16x2(y0, y1, &hi, &lo);
        *reinterpret_cast<uint32_t*>(p.out_split + row * 128 + col) = hi;
        *reinterpret_cast<uint32_t*>(p.out_split + p.split_plane + row * 128 + col) = lo;
      }
    }
  }
}

}  // namespace
}  // namespace um

extern "C" {

int um_ffn_tc(const um_ffn_desc* d, void* stream) {
  UM_REQUIRE(d && d->src[0] && d->src[1] && d->w1 && d->w2 && d->gamma && d->beta, "um_ffn_tc: null descriptor / operand");
  UM_REQUIRE(d->rows > 0 && d->rows % 256 == 0, "um_ffn_tc: rows must be a positive multiple of 256 (pairs of 128-row tiles)");
  UM_REQUIRE(d->hidden >= 128 && d->hidden % 128 == 0, "um_ffn_tc: hidden must be a multiple of 128");
  UM_REQUIRE(d->out_f32 || d->out_split, "um_ffn_tc: no output");
  UM_REQUIRE(d->src_plane_stride >= d->rows * 128 && d->src_plane_stride % 8 == 0,
             "um_ffn_tc: source plane stride must cover rows * 128 halves (multiple of 8)");
  if (d->residual)
    UM_REQUIRE(d->ld_res % 4 == 0 && d->ld_res >= 128 && (reinterpret_cast<uintptr_t>(d->residual) & 15) == 0,
               "um_ffn_tc: residual rows must be 16-byte aligned");
  if (d->out_f32)
    UM_REQUIRE(d->ld_f32 % 4 == 0 && d->ld_f32 >= 128 && (reinterpret_cast<uintptr_t>(d->out_f32) & 15) == 0,
               "um_ffn_tc: fp32 output rows must be 16-byte aligned");
  if (d->out_split)
    UM_REQUIRE(d->split_plane_stride >= d->rows * 128 && d->split_plane_stride % 8 == 0 &&
                   (reinterpret_cast<uintptr_t>(d->out_split) & 15) == 0,
               "um_ffn_tc: output plane stride must cover rows * 128 halves (multiple of 8), 16-byte aligned planes");
  using namespace um;
  const uint64_t gh = (uint64_t)d->rows / 16;                   // rows as a [rows/16, 16] pixel grid, 128 channels
  CUtensorMap mx0, mx1, mw1, mw2;
  int rc;
  if ((rc = make_map_4d_f16(&mx0, d->src[0], 128, 16, gh, 2, 1, (uint64_t)d->src_plane_stride))) return rc;
  if ((rc = make_map_4d_f16(&mx1, d->src[1], 128, 16, gh, 2, 1, (uint64_t)d->src_plane_stride))) return rc;
  if ((rc = make_map_2d_f16(&mw1, d->w1, 2ull * d->hidden, 256, 64))) return rc;
  if ((rc = make_map_2d_f16(&mw2, d->w2, 2ull * 128, (uint64_t)d->hidden, 64))) return rc;
  FfnParams p{};
  p.nchunk = d->hidden / HC; p.hidden = d->hidden;
  p.residual = d->residual; p.ld_res = d->ld_res; p.gamma = d->gamma; p.beta = d->beta;
  p.out_f32 = d->out_f32; p.ld_f32 = d->ld_f32;
  p.out_split = reinterpret_cast<__half*>(d->out_split); p.split_plane = d->split_plane_stride;
  static PerDeviceBytes configured;
  if ((rc = ensure_smem(configured, ffn_tc_kernel, SMEM_BYTES, "ffn_tc"))) return rc;
  ffn_tc_kernel<<<(unsigned)(d->rows / 128), NTHREADS, SMEM_BYTES, (cudaStream_t)stream>>>(mx0, mx1, mw1, mw2, p);
  return check_launch("um_ffn_tc");
}

}  // extern "C"
