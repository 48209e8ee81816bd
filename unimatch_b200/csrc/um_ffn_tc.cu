// Fused transformer FFN on the Hopper tensor cores (wgmma + TMA), fp32-faithful (fp16 hi/lo split operands):
//
//   out = residual + LayerNorm( GELU( [source | message] W1^T ) W2^T )            transformer.py:137-144
//
// Run as two GEMM launches (um_conv2d_tc: FFN1 256 -> 1024 + GELU, then FFN2 1024 -> 128 + LN), the 1024-wide hidden
// activation travels through HBM as fp16 (hi, lo) planes -- 4 KB per token row, 1.6 GB at 8 pairs of 480x832.  Here it
// never leaves the registers: one CTA per 128-row tile, warp-specialised:
//
//   warp 8          TMA producer: the tile's [source | message] planes (128 KB, resident for the tile), then a 3-slot ring
//                   of 32 KB weight tiles in the order the consumers use them: W1(c) as 4 K-slices of 128 hidden rows,
//                   W2(c) as 2 K-halves (64 hidden channels x 128 output rows); warps 9-11 only hand back their registers
//   warpgroups 0-1  consumers, 64 rows each, for every 128-wide hidden chunk c:
//                   H_c = X W1_c^T (48 wgmma 64x128x16, both operands in shared memory, one commit group per K-slice so
//                   a slice is released while the next ones run) into 64 registers -> exact-erf GELU -> (hi, lo) fp16
//                   pairs in the same registers, which are already the register A operand of O += P_c W2_c^T (24 wgmma
//                   64x128x16, K = 128 as 8 k-steps, one commit group per half: the GELU of the second half runs under
//                   the MMAs of the first); after the last chunk: LayerNorm (two-pass statistics over the 4 threads of a
//                   row) + residual on O, fp32 rows and / or fp16 planes out.
//                   The warpgroups take turns at issuing (named barriers 2 and 3), one slot's group per turn, so each
//                   group runs on the tensor pipe in one piece and the warpgroups stay a group apart: one's GELU and
//                   LayerNorm run under the other's MMAs.
// A chunk of 128 (not 64) hidden channels halves the shared-memory bytes per MMA of H_c: a 64x64x16 MMA reads 4 KB of
// operands in 32 tensor clocks, which with both warpgroups issuing is the whole 128 B/clk of the SM's shared memory.
// Every output element is summed in the same order as with 64-wide chunks (K-slice, split term, k-step for H; 64-wide
// hidden block, split term, k-step for O), so the result does not depend on the chunk width.
#include "um_common.cuh"
#include "um_tc.cuh"

namespace um {

using namespace tc;

namespace {

constexpr int NTHREADS = 384;                        // 2 consumer warpgroups (warps 0-7) + the TMA producer's warpgroup
constexpr int PRODUCER = 8;
// per-thread registers of each role (setmaxnreg): 128 x 40 + 256 x 232 <= the 64 K register file.  A consumer holds O and
// H_c / P_c (64 + 64) plus the operand addressing.
constexpr int REGS_PRODUCER = 40, REGS_CONSUMER = 232;
constexpr int TURN = 2;                              // named barriers 2 and 3: the consumer warpgroups' MMA turns
constexpr int HC = 128;                              // hidden channels per chunk
constexpr uint32_t X_BYTES = 4 * 32768;              // 4 K-slices x (hi, lo) x [128 rows x 64 ch]
constexpr uint32_t SLOT_BYTES = 32768;               // (hi, lo) x [128 weight rows x 64 k]
constexpr uint32_t PART_BYTES = SLOT_BYTES / 2;
constexpr int NSLOT = 3;
constexpr uint32_t OFF_RING = X_BYTES;
constexpr uint32_t OFF_BAR = OFF_RING + NSLOT * SLOT_BYTES;        // 229376
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

  if (warp >= PRODUCER) {
    setmaxnreg_dec<REGS_PRODUCER>();
    if (warp != PRODUCER) return;
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
            if (q < 4) tma_load_2d(slot + part * PART_BYTES, &map_w1, full + s, q * 64, part * p.hidden + c * HC);
            else tma_load_2d(slot + part * PART_BYTES, &map_w2, full + s, c * HC + (q - 4) * 64, part * 128);
          }
        }
        __syncwarp();
      }
    return;
  }

  // =============================== consumers ===============================
  setmaxnreg_inc<REGS_CONSUMER>();
  const int wg = warp >> 2;
  const int fr = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's rows fr and fr + 8 (MMA fragment layout)
  const int fc = 2 * (lane & 3);                            // ... and columns 8 j + fc + {0, 1}
  const uint32_t x_base = smem_u32(smem) + wg * 8192;
  const uint32_t ring = smem_u32(smem + OFF_RING);
  const int pa[3] = {1, 0, 0}, pb[3] = {0, 1, 0};          // lo*hi, hi*lo, hi*hi
  // the slot of the ring position `it` and the parity its fill completes with
  auto wait_full = [&](int it) {
    const int s = it % NSLOT;
    mbar_wait_inline(full + s, (it / NSLOT) & 1);
    return ring + s * SLOT_BYTES;
  };
  auto release = [&](int it) {
    __syncwarp();
    if (lane == 0) mbar_arrive(empty + it % NSLOT);
  };
  // The two warpgroups take turns at issuing MMAs, one weight slot's group per turn, warpgroup 0 first: named barrier
  // TURN + w is warpgroup w's turn.  Each group then runs on the tensor pipe in one piece, so the warpgroups stay a group
  // apart and one's GELU (or LayerNorm) runs under the other's MMAs.  Warpgroup 0 does not wait for its first turn and
  // warpgroup 1 does not pass on its last, so every arrive meets a sync.
  const int last_turn = 6 * p.nchunk - 1;
  auto turn_begin = [&](int it) {
    if (wg == 0) {
      if (it > 0) asm volatile("bar.sync %0, 256;" ::"n"(TURN) : "memory");
    } else {
      asm volatile("bar.sync %0, 256;" ::"n"(TURN + 1) : "memory");
    }
  };
  auto turn_end = [&](int it) {
    if (wg == 0) asm volatile("bar.arrive %0, 256;" ::"n"(TURN + 1) : "memory");
    else if (it < last_turn) asm volatile("bar.arrive %0, 256;" ::"n"(TURN) : "memory");
  };
  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  mbar_wait_inline(x_full, 0);
  int it = 0;
  for (int c = 0; c < p.nchunk; ++c) {
    // ---- H_c = X W1_c^T: 64 rows x 128 hidden channels, K = 256 in 4 slots.  A slot is released as soon as its
    //      group has retired (wait<1> after the next group is issued), so the ring keeps filling under the MMAs ----
    float h[64];
    fence_acc(h);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      turn_begin(it + q);
      const uint32_t sb = wait_full(it + q);
      wgmma_fence();
#pragma unroll
      for (int cc = 0; cc < 3; ++cc)
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
          wgmma_ss<128>(h, desc_kmajor(x_base + (q * 2 + pa[cc]) * 16384 + ks * 32),
                        desc_kmajor(sb + pb[cc] * PART_BYTES + ks * 32), (q | cc | ks) != 0);
      wgmma_commit();
      turn_end(it + q);
      if (q > 0) {
        wgmma_wait<1>();
        release(it + q - 1);
      }
    }
    wgmma_wait<0>();
    fence_acc(h);
    release(it + 3);
    it += 4;
    // ---- O += P_c W2_c^T, hidden channels [0, 64) and [64, 128) of the chunk from one slot each.  P_c is GELU(H_c) as
    //      fp16 (hi, lo) pairs in the A-operand layout, formed in place one half at a time: the second half's GELU runs
    //      under the first half's MMAs ----
    uint32_t ph[32], pl[32];
    fence_acc(o);
#pragma unroll
    for (int q = 0; q < 2; ++q) {
#pragma unroll
      for (int jj = 8 * q; jj < 8 * q + 8; ++jj)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
          split_f16x2(act_gelu(h[4 * jj + 2 * hh]), act_gelu(h[4 * jj + 2 * hh + 1]), &ph[2 * jj + hh], &pl[2 * jj + hh]);
      turn_begin(it + q);
      const uint32_t sb = wait_full(it + q);
      wgmma_fence();
#pragma unroll
      for (int cc = 0; cc < 3; ++cc)
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
          const uint32_t* pp = (cc == 0 ? pl : ph) + 16 * q + 4 * ks;
          const uint32_t a[4] = {pp[0], pp[1], pp[2], pp[3]};
          wgmma_rs_n128(o, a, desc_kmajor(sb + (cc == 1 ? PART_BYTES : 0) + ks * 32), true);
        }
      wgmma_commit();
      turn_end(it + q);
    }
    wgmma_wait<1>();
    release(it);
    wgmma_wait<0>();
    fence_acc(o);
    release(it + 1);
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
  if ((rc = make_map_2d_f16(&mw1, d->w1, 2ull * d->hidden, 256, HC))) return rc;
  if ((rc = make_map_2d_f16(&mw2, d->w2, 2ull * 128, (uint64_t)d->hidden, 128))) return rc;
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
