// Implicit-GEMM convolution / Linear layer on the Hopper tensor cores (wgmma), fp32-faithful (fp16 hi/lo split operands).
//
//   out[b,y,x,co] = post( bias[co] + sum_{src,ky,kx,ci} in_src[b, y+ky-ph, x+kx-pw, ci] * W[co, (src,ky,kx,ci)] )
//
// * Activations are channel-last fp16 (hi, lo) planes [2][B][H][W][Cp] (Cp multiple of 64).  One 4-D TMA box
//   (64 channels x 16 x 8 pixels) per filter tap lands directly in the 128B-swizzled K-major layout wgmma reads:
//   im2col is nothing but shifted box coordinates, and the zero padding of the convolution is TMA's out-of-bounds
//   fill.  Up to two input tensors are summed in the same accumulator, so torch.cat([h, x]) of the GRU never exists.
// * Weights are prepared once as [2][Cout_p][Ktot] fp16 planes, K ordered (src, tap, ci).
// * Persistent CTAs (one per SM) loop over tiles of 128 output pixels (16 x 8) x BN output channels (BN = 16 ... 128),
//   warp-specialised: one TMA producer warp (2-3 stage mbarrier ring that keeps running across tiles); two MMA
//   warpgroups, each running the MMAs of 64 of the tile's pixels (3 split terms x 4 K-steps of wgmma 64xBNx16 per stage)
//   into register accumulators, which they hand to the epilogue through a shared-memory tile (acc_full / acc_empty
//   mbarriers) before going on with the next tile's K loop; one epilogue warpgroup (thread = pixel): bias, activation,
//   fused GRU gate math or LayerNorm(+residual), fp32 and/or fp16-split channel-last bulk-tensor stores at a channel
//   offset of a wider buffer (free concatenation).  The epilogue of tile i thus runs under the MMAs of tile i + 1, and
//   neither role's registers count against the other's.
//
// Replaces the fp32 convolutions of BasicUpdateBlock (reg_refine.py:6-119), refine_proj (unimatch.py:315), the CNN
// encoder (backbone.py:49-86) and the transformer's Linear layers (1x1 "convolution" over a [rows/16, 16] pixel grid).
#include <stdlib.h>

#include "um_common.cuh"
#include "um_tc.cuh"

namespace um {

using namespace tc;

namespace {

constexpr int TW = 16, TH = 8;                 // spatial tile = 128 pixels
// operand ring depth: three stages, or two for the widest tiles (BN >= 96: 56-64 KB a stage next to their accumulator tile)
__host__ __device__ constexpr int stages_for(int bn) { return bn >= 96 ? 2 : 3; }
// 2 MMA warpgroups (warps 0-7) + one epilogue warpgroup (warps 8-11) + the TMA producer's warpgroup (warp 12 works,
// warps 13-15 leave at once)
constexpr int NTHREADS = 512;
constexpr int EPILOGUE = 8;
constexpr int PRODUCER = 12;
// per-thread registers of each role (setmaxnreg): 32 + 2 x 168 + 144 = 512 over the four warpgroups = the 64 K register
// file.  The MMA warpgroups hold acc and part (BN = 128, G > 1: 128 registers), the epilogue up to three 32-float
// arrays; the producer loop does not fit in 24.
constexpr int REGS_PRODUCER = 32, REGS_MMA = 168, REGS_EPI = 144;
constexpr uint32_t A_BYTES = 2 * 16384;        // hi + lo, [128 x 64] fp16 each
constexpr uint32_t STAGING_UNIT = 16384;       // one epilogue staging buffer: [128 rows x 32 floats]
constexpr uint32_t STAGING_BYTES = 2 * STAGING_UNIT;
constexpr uint32_t TAIL_BYTES = 256 + 2048;    // barriers, then bias[2][128] | gamma[128] | beta[128]
// accumulator tile handed from the MMA layout to the epilogue: [chunk of 32 channels][128 rows][32 floats]
__host__ __device__ constexpr uint32_t acc_bytes(int bn) { return (bn < 32 ? 32 : bn) * 128 * 4; }
__host__ __device__ constexpr uint32_t conv_smem_bytes(int bn) {
  return stages_for(bn) * (A_BYTES + 2 * bn * 128) + acc_bytes(bn) + STAGING_BYTES + TAIL_BYTES;
}

struct ConvParams {
  int B, H, W, tiles_x, tiles_y;
  int nsrc, cin_p[2];
  int KH, KW, PH, PW, stride;
  int cout, cout_p;
  const float* bias;
  int mode, act;
  float* out_f32; long long ld_f32; int off_f32;
  __half* out_split; int cp_split, off_split; long long plane_split;
  const float* aux0; long long ld_aux0;
  const float* aux1; long long ld_aux1;
  const float* gamma; const float* beta;
  const float* pre; long long ld_pre;   // optional fp32 [B,H,W,>=cout] added to the accumulator before the post-operation
  int ntiles, tiles_n;
  // window-major operand planes of the tensor-core attention (WIN instantiations): output channels [win_c0, win_c1)
  // are written as fp16 (hi, lo) rows of [op][part][stream][window][lp][128] at the row the attention kernel expects
  // (cyclic shift + window split of attention.py:72-83 done as address arithmetic), the others as usual
  __half* win_dst; long long win_plane;
  int win_c0, win_c1, win_lp;
  long long win_tokens, win_L;      // valid rows (streams * L) and tokens per stream
  Geom win_g;
};

// Epilogue math: fast-intrinsic sigmoid / tanh (absolute error at most 1.1e-7 / 2.3e-7 over every finite fp32
// argument, measured on an H100 by tests/test_epilogue_edges_gpu.py; well inside the parity tolerances); the rarely
// used exact-erf GELU stays out of line so that the epilogue's instruction footprint remains small.
__device__ __forceinline__ float sigmoid_fast(float y) { return __fdividef(1.0f, 1.0f + __expf(-y)); }
__device__ __forceinline__ float tanh_fast(float y) { return 1.0f - __fdividef(2.0f, 1.0f + __expf(2.0f * y)); }
__device__ __forceinline__ uint32_t pack_h2(__half a, __half b) {
  return (uint32_t)__half_as_ushort(a) | ((uint32_t)__half_as_ushort(b) << 16);
}

// 32 consecutive output channels [c0, c0 + 32) of accumulator row r (16-byte pieces XOR-swizzled by row)
__device__ __forceinline__ void load_acc32(const float* accs, int r, int c0, float* v) {
  const float* row = accs + (c0 >> 5) * 4096 + r * 32;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float4 x = *reinterpret_cast<const float4*>(row + ((i ^ (r & 7)) << 2));
    v[4 * i] = x.x; v[4 * i + 1] = x.y; v[4 * i + 2] = x.z; v[4 * i + 3] = x.w;
  }
}

// G > 1: every K stage (12 MMAs) is accumulated into a fresh register accumulator and added to the tile's running sum
// with ordinary round-to-nearest fp32 adds.  Tensor-core fp32 accumulation truncates at every accumulate step; the long-K
// convolutions (K >= 512) see one such step per stage instead of one per MMA.
// MODE / ACT >= 0 compile the epilogue for exactly that fused post-operation (a short straight-line loop instead of a
// run-time switch over every mode); -1 = decided at run time.
template <int BN, int G, int MODE, int ACT, bool WIN = false>
__global__ void __launch_bounds__(NTHREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap map_a0, const __grid_constant__ CUtensorMap map_a1,
               const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_of,
               const __grid_constant__ CUtensorMap map_os, ConvParams p) {
  static_assert(BN == 16 || BN == 64 || BN == 96 || BN == 128, "tile widths 16, 64, 96, 128");
  constexpr int NSB = 2;                                   // staging buffers of the epilogue's bulk-store ring
  constexpr uint32_t B_BYTES = 2 * BN * 128;               // hi + lo, [BN x 64] fp16 each
  constexpr uint32_t STAGE_BYTES = A_BYTES + B_BYTES;
  constexpr int STAGES = stages_for(BN);
  constexpr uint32_t ACC_BYTES = acc_bytes(BN);
  extern __shared__ __align__(1024) uint8_t smem[];
  float* accs = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES);
  float* stage_buf = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES + ACC_BYTES);   // 2 x [128 rows x 32 cols] fp32
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES + ACC_BYTES + STAGING_BYTES);
  uint64_t* full = bars;                  // [STAGES]
  uint64_t* empty = bars + STAGES;        // [STAGES]
  uint64_t* acc_full = bars + 2 * STAGES; // the tile's accumulators are in accs (one arrival per MMA thread)
  uint64_t* acc_empty = acc_full + 1;     // the epilogue has read accs (one arrival per epilogue thread)
  float* coef = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(bars) + 256);
  const int mode = MODE >= 0 ? MODE : p.mode;
  const int act = ACT >= 0 ? ACT : p.act;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // Work distribution: CTA `cid` of `ncid` walks the tiles cid, cid + ncid, ...  These and the number of K stages (64
  // input channels each) are formed by each role after its setmaxnreg: ptxas keeps a value that is live across that
  // instruction in local memory.
  auto k_stages = [&]() {
    int n = 0;
    for (int s = 0; s < p.nsrc; ++s) n += p.KH * p.KW * (p.cin_p[s] >> 6);
    return n;
  };

  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) { mbar_init(full + i, 1); mbar_init(empty + i, 8); }   // empty: one arrival per MMA warp
    mbar_init(acc_full, 256);
    mbar_init(acc_empty, 128);
    fence_barrier_init();
  }
  if (warp == PRODUCER && lane == 0) {
    tma_prefetch_desc(&map_a0); tma_prefetch_desc(&map_w);
    if (p.nsrc > 1) tma_prefetch_desc(&map_a1);
  }
  __syncthreads();

  if (warp >= PRODUCER) {
    setmaxnreg_dec<REGS_PRODUCER>();
    if (warp != PRODUCER) return;
    const int cid = (int)blockIdx.x, ncid = (int)gridDim.x;
    const int taps = p.KH * p.KW;
    const int nk = k_stages();
    // The producer warp runs CONVERGED (all 32 lanes execute the loops, one elected lane issues the TMA instructions):
    // addresses are then provably warp-uniform and live in uniform registers.
    int it = 0;
    for (int t = cid; t < p.ntiles; t += ncid) {
      const int n0 = (t % p.tiles_n) * BN;
      int tile = t / p.tiles_n;
      const int x0 = (tile % p.tiles_x) * TW; tile /= p.tiles_x;
      const int y0 = (tile % p.tiles_y) * TH;
      const int b = tile / p.tiles_y;
      // K stages are visited in a per-CTA rotated order: all CTAs need the same weight tiles, and walking them in
      // lock step makes every SM hit the same L2 lines at the same time
      const int chunks0 = p.cin_p[0] >> 6;
      const int nk0 = taps * chunks0;
      const int rot = (int)((unsigned)cid % (unsigned)nk);
      for (int kk = 0; kk < nk; ++kk, ++it) {
        int k = kk + rot; if (k >= nk) k -= nk;
        const int sidx = (k >= nk0) ? 1 : 0;
        const int kl = sidx ? k - nk0 : k;
        const int chunks = sidx ? (p.cin_p[1] >> 6) : chunks0;
        const int tap = kl / chunks, kc = kl - tap * chunks;
        const int ky = tap / p.KW, kx = tap - ky * p.KW;
        const CUtensorMap* ma = sidx ? &map_a1 : &map_a0;
        const int st = it % STAGES;
        mbar_wait_inline(empty + st, ((it / STAGES) & 1) ^ 1);
        uint8_t* sa = smem + st * STAGE_BYTES;
        uint8_t* sb = sa + A_BYTES;
        const int kcol = (sidx ? taps * p.cin_p[0] : 0) + tap * p.cin_p[sidx] + kc * 64;
        if (elect_one()) {
          mbar_arrive_expect_tx(full + st, STAGE_BYTES);
#pragma unroll
          for (int part = 0; part < 2; ++part) {
            tma_load_4d(sa + part * 16384, ma, full + st, kc * 64, x0 * p.stride + kx - p.PW, y0 * p.stride + ky - p.PH, part * p.B + b);
            tma_load_2d(sb + part * (BN * 128), &map_w, full + st, kcol, part * p.cout_p + n0);
          }
        }
        __syncwarp();
      }
    }
  } else if (warp < EPILOGUE) {
    // ---- MMA warpgroups: warpgroup grp computes pixels [64 grp, 64 grp + 64) of the tile, hands the accumulators to
    //      the epilogue through accs and goes on with the next tile's K loop ----
    setmaxnreg_inc<REGS_MMA>();
    const int cid = (int)blockIdx.x, ncid = (int)gridDim.x;
    const int nk = k_stages();
    const int quarter = warp & 3;
    const int grp = warp >> 2;
    const int frow = grp * 64 + quarter * 16 + (lane >> 2); // first accumulator row of this thread's MMA fragment (+ 8)
    const int fcol = 2 * (lane & 3);
    int lt = 0, it = 0;
    for (int t = cid; t < p.ntiles; t += ncid, ++lt) {
      float acc[BN / 2], part[BN / 2];
      for (int k = 0; k < nk; ++k, ++it) {
        const int st = it % STAGES;
        mbar_wait_inline(full + st, (it / STAGES) & 1);
        const uint32_t a_base = smem_u32(smem + st * STAGE_BYTES) + grp * 8192;
        const uint32_t b_base = smem_u32(smem + st * STAGE_BYTES) + A_BYTES;
        const int pa[3] = {1, 0, 0}, pb[3] = {0, 1, 0};        // lo*hi, hi*lo, hi*hi
        if (G > 1) fence_acc(part); else fence_acc(acc);
        wgmma_fence();
#pragma unroll
        for (int c = 0; c < 3; ++c)
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) {
            const uint64_t da = desc_kmajor(a_base + pa[c] * 16384 + ks * 32);
            const uint64_t db = desc_kmajor(b_base + pb[c] * (BN * 128) + ks * 32);
            if (G > 1) wgmma_ss<BN>(part, da, db, (c | ks) != 0);
            else wgmma_ss<BN>(acc, da, db, k > 0 || (c | ks) != 0);
          }
        wgmma_commit();
        wgmma_wait<0>();
        if (G > 1) fence_acc(part); else fence_acc(acc);
        __syncwarp();
        if (lane == 0) mbar_arrive(empty + st);                  // this warp is done with the stage
        if (G > 1) {
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) acc[i] = k ? acc[i] + part[i] : part[i];
        }
      }
      mbar_wait_inline(acc_empty, (lt & 1) ^ 1);               // the previous tile's epilogue has read accs
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = 8 * j + fcol;
        float* chunk = accs + (col >> 5) * 4096;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = frow + 8 * h;
          *reinterpret_cast<float2*>(chunk + row * 32 + ((((col & 31) >> 2) ^ (row & 7)) << 2) + (col & 3)) =
              make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        }
      }
      mbar_arrive(acc_full);
    }
  } else {
    // ---- epilogue warpgroup: thread = output pixel (accumulator row), walking the tile's 32-channel chunks.  Results
    //      are staged in shared memory in TMA box layout (a ring of two 16 KB buffers) and ONE thread issues bulk tensor
    //      stores, which overlap the next chunk's math. ----
    setmaxnreg_inc<REGS_EPI>();
    const int cid = (int)blockIdx.x, ncid = (int)gridDim.x;
    const int r = threadIdx.x - EPILOGUE * 32;
    const bool leader = r == 0;
    int sctr = 0;                                          // staging passes issued (buffer ring position)
    auto epi_sync = [&]() { asm volatile("bar.sync 1, 128;" ::: "memory"); };
    if (mode == UM_CONV_LN) { coef[256 + r] = __ldg(p.gamma + r); coef[384 + r] = __ldg(p.beta + r); }
    epi_sync();
    int lt = 0;
    for (int t = cid; t < p.ntiles; t += ncid, ++lt) {
      const int n0 = (t % p.tiles_n) * BN;
      int tile = t / p.tiles_n;
      const int x0 = (tile % p.tiles_x) * TW; tile /= p.tiles_x;
      const int y0 = (tile % p.tiles_y) * TH;
      const int b = tile / p.tiles_y;
      const long long pix_r = ((long long)b * p.H + (y0 + (r >> 4))) * p.W + x0 + (r & 15);
      const bool valid_r = (y0 + (r >> 4) < p.H) && (x0 + (r & 15) < p.W);

      // One 32-channel chunk of the tile -> global memory.  A staging buffer was last read by the bulk store issued two
      // passes earlier: that read must be over before anybody overwrites it (checking only after the writes, as an
      // earlier version did, let fast epilogues corrupt rows the TMA unit was still reading).
      auto emit = [&](const float (&v)[32], int co_out, bool to_f32, bool to_split, bool to_win = false) {
        if (WIN && to_win) {                                 // hi then lo rows staged like to_split, scattered row by row
          uint8_t* sbs = reinterpret_cast<uint8_t*>(stage_buf + (sctr % NSB) * 4096);
          ++sctr;
          if (leader) bulk_wait_read<0>();                   // this pass commits no bulk group: drain the ring
          epi_sync();
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            uint32_t hw[4], lw[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) split_f16x2(v[8 * i + 2 * e], v[8 * i + 2 * e + 1], &hw[e], &lw[e]);
            const int off = r * 64 + ((i ^ ((r >> 1) & 3)) << 4);
            *reinterpret_cast<uint4*>(sbs + off) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
            *reinterpret_cast<uint4*>(sbs + 8192 + off) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
          }
          epi_sync();
          const int wc = co_out - p.win_c0;                  // channel inside the window-plane range
          __half* obase = p.win_dst + (long long)(wc >> 7) * 2 * p.win_plane + (wc & 127);
          const int* rowdst = reinterpret_cast<const int*>(coef + 256) + (lt & 1) * 128;
          const int piece = r & 3;
#pragma unroll
          for (int itr = 0; itr < 4; ++itr) {
            const int row = itr * 32 + (r >> 2);
            const int drow = rowdst[row];
            if (drow < 0) continue;
            const int soff = row * 64 + ((piece ^ ((row >> 1) & 3)) << 4);
            const uint4 hv = *reinterpret_cast<const uint4*>(sbs + soff);
            const uint4 lv = *reinterpret_cast<const uint4*>(sbs + 8192 + soff);
            __half* d = obase + (long long)drow * 128 + piece * 8;
            *reinterpret_cast<uint4*>(d) = hv;
            *reinterpret_cast<uint4*>(d + p.win_plane) = lv;
          }
          return;
        }
        if (to_f32) {                                        // [128 rows][32 floats], 128B swizzle
          float* my_stage = stage_buf + (sctr % NSB) * 4096;
          ++sctr;
          if (leader) bulk_wait_read<NSB - 1>();
          epi_sync();
#pragma unroll
          for (int i = 0; i < 8; ++i)
            *reinterpret_cast<float4*>(my_stage + r * 32 + ((i ^ (r & 7)) << 2)) = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
          fence_proxy_async();
          epi_sync();
          if (leader) { tma_store_4d(&map_of, my_stage, co_out, x0, y0, b); bulk_commit(); }
        }
        if (to_split) {                                      // hi then lo: [128 rows][32 halves], 64-byte rows, 64B swizzle
          uint8_t* sbs = reinterpret_cast<uint8_t*>(stage_buf + (sctr % NSB) * 4096);
          ++sctr;
          if (leader) bulk_wait_read<NSB - 1>();
          epi_sync();
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            uint32_t hw[4], lw[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) split_f16x2(v[8 * i + 2 * e], v[8 * i + 2 * e + 1], &hw[e], &lw[e]);
            const int off = r * 64 + ((i ^ ((r >> 1) & 3)) << 4);
            *reinterpret_cast<uint4*>(sbs + off) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
            *reinterpret_cast<uint4*>(sbs + 8192 + off) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
          }
          fence_proxy_async();
          epi_sync();
          if (leader) {
            tma_store_4d(&map_os, sbs, co_out, x0, y0, b);
            tma_store_4d(&map_os, sbs + 8192, co_out, x0, y0, p.B + b);
            bulk_commit();
          }
        }
      };

      if constexpr (BN == 128) {
        if (mode == UM_CONV_LN) {
          // LayerNorm over the 128 channels of the row (+ residual), two-pass statistics like the reference's (mean first,
          // then the centred sum of squares, not E[x^2] - mean^2).  Each statistic is the sum of two partial sums, over
          // channels {0-31, 64-95} and {32-63, 96-127}, each accumulated in that channel order: the rounding the kernel
          // has always had.  The row is re-read from accs for every pass instead of being held in registers.
          mbar_wait_inline(acc_full, lt & 1);
          float sum0 = 0.f, sum1 = 0.f, sq0 = 0.f, sq1 = 0.f;
#pragma unroll 1
          for (int h = 0; h < 2; ++h) {
            float v0[32], v1[32];
            load_acc32(accs, r, 32 * h, v0);
            load_acc32(accs, r, 64 + 32 * h, v1);
            float sum = 0.f;
#pragma unroll
            for (int i = 0; i < 32; ++i) sum += v0[i];
#pragma unroll
            for (int i = 0; i < 32; ++i) sum += v1[i];
            if (h == 0) sum0 = sum; else sum1 = sum;
          }
          const float mean = (sum0 + sum1) * (1.0f / 128.0f);
#pragma unroll 1
          for (int h = 0; h < 2; ++h) {
            float v0[32], v1[32];
            load_acc32(accs, r, 32 * h, v0);
            load_acc32(accs, r, 64 + 32 * h, v1);
            float sq = 0.f;
#pragma unroll
            for (int i = 0; i < 32; ++i) { const float dd = v0[i] - mean; sq = fmaf(dd, dd, sq); }
#pragma unroll
            for (int i = 0; i < 32; ++i) { const float dd = v1[i] - mean; sq = fmaf(dd, dd, sq); }
            if (h == 0) sq0 = sq; else sq1 = sq;
          }
          const float rstd = rsqrtf((sq0 + sq1) * (1.0f / 128.0f) + 1e-5f);
          const bool need_a = valid_r && p.aux0;
#pragma unroll 1
          for (int c0 = 0; c0 < 128; c0 += 32) {
            float a[32];
            if (need_a) {                                    // residual
              const float4* pa = reinterpret_cast<const float4*>(p.aux0 + pix_r * p.ld_aux0 + c0);
#pragma unroll
              for (int i = 0; i < 8; ++i) { const float4 t4 = __ldg(pa + i); a[4 * i] = t4.x; a[4 * i + 1] = t4.y; a[4 * i + 2] = t4.z; a[4 * i + 3] = t4.w; }
            }
            float v[32];
            load_acc32(accs, r, c0, v);
            if (c0 == 96) mbar_arrive(acc_empty);            // the tile's last read of accs
            const float4* g4 = reinterpret_cast<const float4*>(coef + 256 + c0);
            const float4* b4 = reinterpret_cast<const float4*>(coef + 384 + c0);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const float4 g = g4[i], bb = b4[i];
              v[4 * i] = (v[4 * i] - mean) * rstd * g.x + bb.x;
              v[4 * i + 1] = (v[4 * i + 1] - mean) * rstd * g.y + bb.y;
              v[4 * i + 2] = (v[4 * i + 2] - mean) * rstd * g.z + bb.z;
              v[4 * i + 3] = (v[4 * i + 3] - mean) * rstd * g.w + bb.w;
            }
            if (need_a) {
#pragma unroll
              for (int i = 0; i < 32; ++i) v[i] += a[i];
            }
            emit(v, c0, p.out_f32 != nullptr, p.out_split != nullptr);
          }
          continue;
        }
      }

      // bias slice of this tile -> shared memory (read back as broadcast float4; double-buffered by tile parity)
      float* sbias = coef + (lt & 1) * 128;
      if (r < BN) sbias[r] = (p.bias && n0 + r < p.cout) ? __ldg(p.bias + n0 + r) : 0.f;
      if (WIN) {                                             // destination row of every token of this tile (r = row)
        const int yy = y0 + (r >> 4), xx = x0 + (r & 15);
        const long long token = ((long long)b * p.H + yy) * p.W + xx;
        int drow = -1;
        if (yy < p.H && xx < p.W && token < p.win_tokens) {
          const Geom& g = p.win_g;
          const int n = (int)(token / p.win_L);
          const int t = (int)(token - (long long)n * p.win_L);
          const int ty = t / g.w, tx = t - ty * g.w;
          int yr = ty - g.sh; if (yr < 0) yr += g.h;         // rolled[yr, xr] = orig[(yr + sh) % h, (xr + sw) % w]
          int xr = tx - g.sw; if (xr < 0) xr += g.w;
          const int wy = yr / g.wh, wx = xr / g.ww;
          drow = (n * g.nwin + wy * g.kw + wx) * p.win_lp + (yr - wy * g.wh) * g.ww + (xr - wx * g.ww);
        }
        reinterpret_cast<int*>(coef + 256)[(lt & 1) * 128 + r] = drow;
      }
      epi_sync();

      constexpr int CH = BN < 32 ? BN : 32;
#pragma unroll 1
      for (int c0 = 0; c0 < BN; c0 += 32) {
        const int co0 = n0 + c0;
        const bool live = co0 < p.cout;                      // warpgroup-uniform
        bool to_f32 = p.out_f32 != nullptr, to_split = p.out_split != nullptr;
        int co_out = co0;
        if (mode == UM_CONV_GRU_ZR) {                        // z -> fp32, r*h -> split planes
          to_f32 = co0 < 128; to_split = co0 >= 128;
          if (co0 >= 128) co_out = co0 - 128;
        }
        bool to_win = false;
        if (WIN && co0 >= p.win_c0 && co0 < p.win_c1) { to_win = true; to_f32 = to_split = false; }
        // the pre-accumulated part does not depend on the accumulator: fetched before waiting for it
        float px[32];
        const bool need_p = live && valid_r && p.pre;        // loop-invariant part of the convolution, computed once by the caller
        if (need_p) {
          const float4* pp = reinterpret_cast<const float4*>(p.pre + pix_r * p.ld_pre + co0);
#pragma unroll
          for (int i = 0; i < 8; ++i) { const float4 t4 = __ldg(pp + i); px[4 * i] = t4.x; px[4 * i + 1] = t4.y; px[4 * i + 2] = t4.z; px[4 * i + 3] = t4.w; }
        }
        float v[32];
        mbar_wait_inline(acc_full, lt & 1);
        load_acc32(accs, r, c0, v);                          // BN = 16: the upper 16 columns are unused
        if (c0 + 32 >= BN) mbar_arrive(acc_empty);           // the tile's last read of accs
        if (!live) continue;
        // ---- per-pixel math on the thread's own row ----
        if (p.bias) {
          const float4* s4 = reinterpret_cast<const float4*>(sbias + c0);
#pragma unroll
          for (int i = 0; i < CH / 4; ++i) {
            const float4 bb = s4[i];
            v[4 * i] += bb.x; v[4 * i + 1] += bb.y; v[4 * i + 2] += bb.z; v[4 * i + 3] += bb.w;
          }
        }
        if (need_p) {
#pragma unroll
          for (int i = 0; i < CH; ++i) v[i] += px[i];
        }
        // operands of the fused gate math, fetched once px is consumed: at most three 32-float arrays are live, which
        // keeps the epilogue inside its register budget
        float ax[32], bx[32];
        const bool need_a = valid_r && p.aux0 && (mode == UM_CONV_GRU_Q || (mode == UM_CONV_GRU_ZR && co0 >= 128));
        const bool need_b = valid_r && mode == UM_CONV_GRU_Q;
        if (need_a) {
          const float4* ap = reinterpret_cast<const float4*>(p.aux0 + pix_r * p.ld_aux0 + (mode == UM_CONV_GRU_ZR ? co0 - 128 : co0));
#pragma unroll
          for (int i = 0; i < 8; ++i) { const float4 t4 = __ldg(ap + i); ax[4 * i] = t4.x; ax[4 * i + 1] = t4.y; ax[4 * i + 2] = t4.z; ax[4 * i + 3] = t4.w; }
        }
        if (need_b) {
          const float4* bp = reinterpret_cast<const float4*>(p.aux1 + pix_r * p.ld_aux1 + co0);
#pragma unroll
          for (int i = 0; i < 8; ++i) { const float4 t4 = __ldg(bp + i); bx[4 * i] = t4.x; bx[4 * i + 1] = t4.y; bx[4 * i + 2] = t4.z; bx[4 * i + 3] = t4.w; }
        }
        if (mode == UM_CONV_GRU_ZR) {
#pragma unroll
          for (int i = 0; i < CH; ++i) v[i] = sigmoid_fast(v[i]);
          if (need_a) {
#pragma unroll
            for (int i = 0; i < CH; ++i) v[i] *= ax[i];
          }
        } else if (mode == UM_CONV_GRU_Q) {
          if (need_b) {
#pragma unroll
            for (int i = 0; i < CH; ++i) v[i] = (1.0f - bx[i]) * ax[i] + bx[i] * tanh_fast(v[i]);
          }
        } else if (act == UM_ACT_RELU) {
#pragma unroll
          for (int i = 0; i < CH; ++i) v[i] = fmaxf(v[i], 0.f);
        } else if (act == UM_ACT_TANH) {
#pragma unroll
          for (int i = 0; i < CH; ++i) v[i] = tanh_fast(v[i]);
        } else if (act == UM_ACT_SIGMOID) {
#pragma unroll
          for (int i = 0; i < CH; ++i) v[i] = sigmoid_fast(v[i]);
        } else if (act == UM_ACT_GELU) {
#pragma unroll
          for (int i = 0; i < CH; ++i) v[i] = act_gelu(v[i]);
        }
        if constexpr (BN >= 32) {
          emit(v, co_out, to_f32, to_split, to_win);
        } else {
          // BN = 16 (flow / disparity heads, 1-2 live channels): plain predicated stores through a staging transpose
          const int nvalid = min(CH, p.cout - co0);
          float* sb = stage_buf;
          epi_sync();                                        // the previous tile's readers are done with the buffer
#pragma unroll
          for (int i = 0; i < CH / 4; ++i)
            *reinterpret_cast<float4*>(sb + r * 32 + ((i ^ (r & 7)) << 2)) = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
          epi_sync();
          if (to_f32) {
#pragma unroll 1
            for (int itr = 0; itr < 8; ++itr) {
              const int row = itr * 16 + (r >> 3), piece = r & 7;
              const int yy = y0 + (row >> 4), xx = x0 + (row & 15);
              if (yy >= p.H || xx >= p.W || piece * 4 >= nvalid) continue;
              const float4 val = *reinterpret_cast<const float4*>(sb + row * 32 + ((piece ^ (row & 7)) << 2));
              float* dst = p.out_f32 + (((long long)b * p.H + yy) * p.W + xx) * p.ld_f32 + p.off_f32 + co_out + piece * 4;
              const float e[4] = {val.x, val.y, val.z, val.w};
              for (int k = 0; k < 4; ++k) if (piece * 4 + k < nvalid) dst[k] = e[k];
            }
          }
          if (to_split) {
#pragma unroll 1
            for (int itr = 0; itr < 4; ++itr) {
              const int row = itr * 32 + (r >> 2), piece = r & 3;            // piece = 8 channels
              const int yy = y0 + (row >> 4), xx = x0 + (row & 15);
              if (yy >= p.H || xx >= p.W || piece * 8 >= nvalid) continue;
              const float4 a4 = *reinterpret_cast<const float4*>(sb + row * 32 + (((2 * piece) ^ (row & 7)) << 2));
              const float4 c4 = *reinterpret_cast<const float4*>(sb + row * 32 + (((2 * piece + 1) ^ (row & 7)) << 2));
              const float e[8] = {a4.x, a4.y, a4.z, a4.w, c4.x, c4.y, c4.z, c4.w};
              __half* dh = p.out_split + (((long long)b * p.H + yy) * p.W + xx) * p.cp_split + p.off_split + co_out + piece * 8;
              __half* dl = dh + p.plane_split;
              for (int k = 0; k < 8; ++k)
                if (piece * 8 + k < nvalid) { __half h0, l0; split_f16(e[k], &h0, &l0); dh[k] = h0; dl[k] = l0; }
            }
          }
        }
      }
    }
    if (leader) bulk_wait_all();                             // shared memory must outlive the last bulk stores
  }
}

// fp32 rows [rows, C] (row stride ld) -> fp16 (hi, lo) planes at channel offset `off` of a [rows, cp] buffer
template <int VEC>
__global__ void __launch_bounds__(256) split_planes_kernel(const float* __restrict__ src, long long ld, int C,
                                                           __half* __restrict__ dst, int cp, int off, long long plane,
                                                           long long rows) {
  const int per_row = C / VEC;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * per_row) return;
  const long long row = i / per_row;
  const int c = (int)(i - row * per_row) * VEC;
  if (VEC == 4) {
    const float4 x = __ldg(reinterpret_cast<const float4*>(src + row * ld + c));
    __half h[4], l[4];
    split_f16(x.x, &h[0], &l[0]); split_f16(x.y, &h[1], &l[1]); split_f16(x.z, &h[2], &l[2]); split_f16(x.w, &h[3], &l[3]);
    *reinterpret_cast<uint2*>(dst + row * cp + off + c) = make_uint2(pack_h2(h[0], h[1]), pack_h2(h[2], h[3]));
    *reinterpret_cast<uint2*>(dst + plane + row * cp + off + c) = make_uint2(pack_h2(l[0], l[1]), pack_h2(l[2], l[3]));
  } else {
    __half h, l;
    split_f16(__ldg(src + row * ld + c), &h, &l);
    dst[row * cp + off + c] = h;
    dst[plane + row * cp + off + c] = l;
  }
}

}  // namespace

// plane_elems != 0 (batch 1 only): the (hi, lo) planes are `plane_elems` halves apart instead of densely stacked
int make_map_4d_f16(CUtensorMap* map, const void* base, uint64_t cp, uint64_t W, uint64_t H, uint64_t NB, uint32_t stride,
                    uint64_t plane_elems) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) { set_error("cuTensorMapEncodeTiled unavailable"); return UM_ECUDA; }
  cuuint64_t dims[4] = {cp, W, H, NB};
  cuuint64_t strides[3] = {cp * 2, cp * W * 2, (plane_elems ? plane_elems : cp * W * H) * 2};
  // stride s: the box traverses TW*s x TH*s input pixels and keeps every s-th one (16 x 8 land in shared memory)
  cuuint32_t box[4] = {64, 16 * stride, 8 * stride, 1};        // TW x TH
  cuuint32_t estr[4] = {1, stride, stride, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(4d) failed (%d)", (int)r); return UM_ECUDA; }
  return UM_OK;
}

// output tensor maps: channels [off, off + cout) of a channel-last buffer viewed as (c, W, H, N); TMA clips the box at the
// map's channel extent, so neighbouring channels of a wider buffer (free concatenation) are never touched
int make_map_out(CUtensorMap* map, void* base, int elem_bytes, uint64_t cout, uint64_t ld, uint64_t W, uint64_t H, uint64_t N,
                 uint64_t plane_elems) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) { set_error("cuTensorMapEncodeTiled unavailable"); return UM_ECUDA; }
  cuuint64_t dims[4] = {cout, W, H, N};
  cuuint64_t strides[3] = {ld * elem_bytes, ld * W * elem_bytes, (plane_elems ? plane_elems : ld * W * H) * elem_bytes};
  cuuint32_t box[4] = {32, 16, 8, 1};                          // TW x TH
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(map, elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, base, dims,
                   strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   elem_bytes == 4 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                   CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(out) failed (%d)", (int)r); return UM_ECUDA; }
  return UM_OK;
}

namespace {

template <int BN, int G, int MODE, int ACT, bool WIN = false>
int launch_conv(const CUtensorMap& m0, const CUtensorMap& m1, const CUtensorMap& mw, const CUtensorMap& mof,
                const CUtensorMap& mos, const ConvParams& p, cudaStream_t st) {
  constexpr uint32_t smem = conv_smem_bytes(BN);
  static_assert(smem <= 232448, "shared memory budget");
  static PerDeviceBytes configured;
  if (int rc = ensure_smem(configured, conv_tc_kernel<BN, G, MODE, ACT, WIN>, smem, "conv_tc")) return rc;
  const int num_sms = device_sm_count();
  const int grid = p.ntiles < num_sms ? p.ntiles : num_sms;      // persistent: one CTA per SM
  conv_tc_kernel<BN, G, MODE, ACT, WIN><<<grid, NTHREADS, smem, st>>>(m0, m1, mw, mof, mos, p);
  return check_launch("um_conv2d_tc");
}

}  // namespace
}  // namespace um

extern "C" {

int um_conv2d_tc(const um_conv_desc* d, void* stream) {
  using namespace um;
  UM_REQUIRE(d && d->src[0] && d->weights, "um_conv2d_tc: null descriptor / source / weights");
  UM_REQUIRE(d->batch > 0 && d->h > 0 && d->w > 0, "um_conv2d_tc: bad shape");
  UM_REQUIRE(d->nsrc == 1 || (d->nsrc == 2 && d->src[1]), "um_conv2d_tc: nsrc must be 1 or 2");
  for (int s = 0; s < d->nsrc; ++s)
    UM_REQUIRE(d->cin_p[s] > 0 && d->cin_p[s] % 64 == 0, "um_conv2d_tc: padded input channels must be multiples of 64");
  UM_REQUIRE(d->bn == 16 || d->bn == 64 || d->bn == 96 || d->bn == 128 || d->bn == 192 || d->bn == 256,
             "um_conv2d_tc: bn must be 16, 64, 96, 128, 192 or 256");
  UM_REQUIRE(d->cout > 0 && d->cout_p >= d->cout && d->cout_p % d->bn == 0, "um_conv2d_tc: bad output channel padding");
  UM_REQUIRE(d->kh > 0 && d->kw > 0 && d->kh * d->kw <= 49, "um_conv2d_tc: bad filter size");
  UM_REQUIRE(d->mode >= UM_CONV_LINEAR && d->mode <= UM_CONV_LN, "um_conv2d_tc: bad mode");
  if (d->mode == UM_CONV_LN)
    UM_REQUIRE(d->cout == 128 && d->cout_p == 128 && d->bn == 128 && d->gamma && d->beta && d->ld_f32 % 4 == 0 &&
                   d->off_f32 % 4 == 0 && d->cp_split % 8 == 0 && d->off_split % 8 == 0 && d->ld_aux0 % 4 == 0,
               "um_conv2d_tc: LN needs cout = cout_p = bn = 128, gamma/beta and 16-byte aligned rows");
  const bool win = d->win_dst != nullptr;
  UM_REQUIRE(d->out_f32 || d->out_split || win, "um_conv2d_tc: no output");
  Geom wg{};
  if (win) {
    UM_REQUIRE(d->mode == UM_CONV_LINEAR && d->act == UM_ACT_NONE && d->bn == 128 && d->batch == 1 && d->stride == 1 &&
                   d->kh == 1 && d->kw == 1 && d->nsrc == 1 && d->cin_p[0] == 128,
               "um_conv2d_tc: window-plane output needs a plain 128 -> cout Linear layer (bn 128, batch 1)");
    UM_REQUIRE(make_geom(&d->win_geom, &wg), "um_conv2d_tc: bad window geometry");
    UM_REQUIRE(d->win_c0 >= 0 && d->win_c0 % 128 == 0 && d->win_c1 % 128 == 0 && d->win_c1 > d->win_c0 && d->win_c1 <= d->cout_p,
               "um_conv2d_tc: window-plane channel range must be 128-aligned and inside cout_p");
    UM_REQUIRE(d->win_streams > 0 && d->win_lp >= wg.lw && d->win_lp % 128 == 0 &&
                   (long long)d->win_streams * wg.h * wg.w <= (long long)d->h * d->w,
               "um_conv2d_tc: window-plane rows (streams * h * w) exceed the GEMM rows / bad lp");
    UM_REQUIRE((reinterpret_cast<uintptr_t>(d->win_dst) & 15) == 0, "um_conv2d_tc: window planes must be 16-byte aligned");
    UM_REQUIRE(d->out_f32 || d->out_split || (d->win_c0 == 0 && d->win_c1 >= d->cout),
               "um_conv2d_tc: channels outside the window-plane range have no destination");
  }
  if (d->src_plane_stride || d->split_plane_stride)
    UM_REQUIRE(d->batch == 1 && d->src_plane_stride >= 0 && d->split_plane_stride >= 0 && d->src_plane_stride % 8 == 0 &&
                   d->split_plane_stride % 8 == 0,
               "um_conv2d_tc: explicit (hi, lo) plane strides need batch 1 and multiples of 8 halves");
  if (d->mode == UM_CONV_GRU_ZR)
    UM_REQUIRE(d->cout == 256 && (d->bn == 128 || d->bn == 256) && d->aux0 && d->out_f32 && d->out_split,
               "um_conv2d_tc: GRU_ZR needs cout 256, bn 128 or 256, h, z-out and rh-out");
  if (d->mode == UM_CONV_GRU_Q)
    UM_REQUIRE(d->cout == 128 && d->aux0 && d->aux1, "um_conv2d_tc: GRU_Q needs cout 128, h and z");

  if (d->pre)
    UM_REQUIRE(d->mode != UM_CONV_LN && d->bn >= 32 && d->ld_pre % 4 == 0 && d->ld_pre >= d->cout && d->cout % 32 == 0 &&
                   (reinterpret_cast<uintptr_t>(d->pre) & 15) == 0,
               "um_conv2d_tc: pre-accumulated input needs a non-LN mode, bn >= 32, cout %% 32 == 0 and 16-byte aligned rows");
  UM_REQUIRE(d->stride == 1 || d->stride == 2 || d->stride == 4 || d->stride == 8, "um_conv2d_tc: stride must be 1, 2, 4 or 8");
  const int ho = (d->h + 2 * d->pad_h - d->kh) / d->stride + 1, wo = (d->w + 2 * d->pad_w - d->kw) / d->stride + 1;
  UM_REQUIRE(ho > 0 && wo > 0, "um_conv2d_tc: empty output");
  ConvParams p{};
  p.B = d->batch; p.H = ho; p.W = wo; p.stride = d->stride;
  p.tiles_x = (wo + TW - 1) / TW; p.tiles_y = (ho + TH - 1) / TH;
  p.nsrc = d->nsrc; p.cin_p[0] = d->cin_p[0]; p.cin_p[1] = d->nsrc > 1 ? d->cin_p[1] : 0;
  p.KH = d->kh; p.KW = d->kw; p.PH = d->pad_h; p.PW = d->pad_w;
  p.cout = d->cout; p.cout_p = d->cout_p; p.bias = d->bias; p.mode = d->mode; p.act = d->act;
  p.out_f32 = d->out_f32; p.ld_f32 = d->ld_f32; p.off_f32 = d->off_f32;
  p.out_split = reinterpret_cast<__half*>(d->out_split); p.cp_split = d->cp_split; p.off_split = d->off_split;
  p.plane_split = (long long)d->batch * ho * wo * d->cp_split;
  p.aux0 = d->aux0; p.ld_aux0 = d->ld_aux0; p.aux1 = d->aux1; p.ld_aux1 = d->ld_aux1;
  p.gamma = d->gamma; p.beta = d->beta;
  p.pre = d->pre; p.ld_pre = d->ld_pre;
  if (d->split_plane_stride) p.plane_split = d->split_plane_stride;
  if (win) {
    p.win_dst = reinterpret_cast<__half*>(d->win_dst);
    p.win_g = wg; p.win_lp = d->win_lp; p.win_c0 = d->win_c0; p.win_c1 = d->win_c1;
    p.win_L = (long long)wg.h * wg.w;
    p.win_tokens = (long long)d->win_streams * p.win_L;
    p.win_plane = (long long)d->win_streams * wg.nwin * d->win_lp * 128;
  }

  long long ktot = 0;
  for (int s = 0; s < d->nsrc; ++s) ktot += (long long)d->kh * d->kw * d->cin_p[s];
  // long K loops sum per-stage partial accumulators with fp32 adds (see conv_tc_kernel); short ones (Linear layers) need none
  const long long nk = ktot / 64;
  const bool multi = nk >= 8;
  // the accumulator tile lives in registers of two warpgroups: 256- and 192-wide channel tiles run as two 128- / 96-wide ones
  const int bn = d->bn == 256 ? 128 : d->bn == 192 ? 96 : d->bn;
  p.tiles_n = d->cout_p / bn;
  p.ntiles = p.tiles_x * p.tiles_y * p.B * p.tiles_n;
  CUtensorMap m0, m1, mw;
  int rc;
  const uint64_t sps = (uint64_t)d->src_plane_stride;
  if ((rc = make_map_4d_f16(&m0, d->src[0], d->cin_p[0], d->w, d->h, 2ull * d->batch, d->stride, sps))) return rc;
  if (d->nsrc > 1) { if ((rc = make_map_4d_f16(&m1, d->src[1], d->cin_p[1], d->w, d->h, 2ull * d->batch, d->stride, sps))) return rc; }
  else m1 = m0;
  if ((rc = make_map_2d_f16(&mw, d->weights, 2ull * d->cout_p, (uint64_t)ktot, (uint32_t)bn))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  CUtensorMap mof = m0, mos = m0;
  if (d->bn >= 32) {
    const int c_f32 = (d->mode == UM_CONV_GRU_ZR) ? 128 : d->cout, c_split = (d->mode == UM_CONV_GRU_ZR) ? 128 : d->cout;
    if (d->out_f32) {
      UM_REQUIRE(d->ld_f32 % 4 == 0 && d->off_f32 % 4 == 0 && (reinterpret_cast<uintptr_t>(d->out_f32) & 15) == 0,
                 "um_conv2d_tc: fp32 output must be 16-byte aligned (ld, channel offset multiples of 4)");
      if ((rc = make_map_out(&mof, d->out_f32 + d->off_f32, 4, c_f32, d->ld_f32, wo, ho, d->batch))) return rc;
    }
    if (d->out_split) {
      UM_REQUIRE(d->cp_split % 8 == 0 && d->off_split % 8 == 0 && (reinterpret_cast<uintptr_t>(d->out_split) & 15) == 0,
                 "um_conv2d_tc: split output must be 16-byte aligned (cp, channel offset multiples of 8)");
      if ((rc = make_map_out(&mos, reinterpret_cast<__half*>(d->out_split) + d->off_split, 2, c_split, d->cp_split, wo, ho,
                             2ull * d->batch, (uint64_t)d->split_plane_stride))) return rc;
    }
  }
  // the post-operations the matching path uses get their own epilogue instantiation; anything else runs the generic one
#define UM_CONV_CASE(BN_, G_, MODE_, ACT_)                                                   \
  if (bn == BN_ && multi == (G_ > 1) && d->mode == MODE_ && ((MODE_) != UM_CONV_LINEAR || d->act == (ACT_))) \
    return launch_conv<BN_, G_, MODE_, (MODE_) == UM_CONV_LINEAR ? (ACT_) : 0>(m0, m1, mw, mof, mos, p, st);
  if (win) {
    UM_REQUIRE(nk <= 2, "um_conv2d_tc: window-plane output is built for K <= 128");
    return launch_conv<128, 1, UM_CONV_LINEAR, UM_ACT_NONE, true>(m0, m1, mw, mof, mos, p, st);
  }
  UM_CONV_CASE(128, 1, UM_CONV_LINEAR, UM_ACT_NONE)
  UM_CONV_CASE(128, 1, UM_CONV_LINEAR, UM_ACT_RELU)
  UM_CONV_CASE(128, 1, UM_CONV_LINEAR, UM_ACT_GELU)
  UM_CONV_CASE(128, 1, UM_CONV_LN, 0)
  UM_CONV_CASE(128, 2, UM_CONV_LN, 0)
  UM_CONV_CASE(128, 2, UM_CONV_LINEAR, UM_ACT_NONE)
  UM_CONV_CASE(128, 2, UM_CONV_LINEAR, UM_ACT_RELU)
  UM_CONV_CASE(128, 2, UM_CONV_GRU_ZR, 0)
  UM_CONV_CASE(128, 2, UM_CONV_GRU_Q, 0)
  UM_CONV_CASE(96, 2, UM_CONV_LINEAR, UM_ACT_RELU)
  UM_CONV_CASE(64, 4, UM_CONV_LINEAR, UM_ACT_NONE)
  UM_CONV_CASE(64, 4, UM_CONV_LINEAR, UM_ACT_RELU)
#undef UM_CONV_CASE
  if (bn == 128) return multi ? launch_conv<128, 2, -1, -1>(m0, m1, mw, mof, mos, p, st) : launch_conv<128, 1, -1, -1>(m0, m1, mw, mof, mos, p, st);
  if (bn == 96) return multi ? launch_conv<96, 2, -1, -1>(m0, m1, mw, mof, mos, p, st) : launch_conv<96, 1, -1, -1>(m0, m1, mw, mof, mos, p, st);
  if (bn == 64) return multi ? launch_conv<64, 4, -1, -1>(m0, m1, mw, mof, mos, p, st) : launch_conv<64, 1, -1, -1>(m0, m1, mw, mof, mos, p, st);
  return multi ? launch_conv<16, 4, -1, -1>(m0, m1, mw, mof, mos, p, st) : launch_conv<16, 1, -1, -1>(m0, m1, mw, mof, mos, p, st);
}

int um_split_planes(const float* src, int64_t rows, int32_t channels, int64_t ld, void* dst, int32_t cp, int32_t off,
                    int64_t dst_plane_stride, void* stream) {
  UM_REQUIRE(src && dst && rows > 0 && channels > 0 && off >= 0 && off + channels <= cp && ld >= channels,
             "um_split_planes: bad arguments");
  UM_REQUIRE(dst_plane_stride == 0 || (dst_plane_stride >= rows * cp && dst_plane_stride % 4 == 0),
             "um_split_planes: dst_plane_stride must cover rows * cp halves (multiple of 4)");
  const long long plane = dst_plane_stride ? (long long)dst_plane_stride : (long long)rows * cp;
  const bool vec = (channels % 4 == 0) && (ld % 4 == 0) && (off % 4 == 0) && (cp % 4 == 0) &&
                   ((reinterpret_cast<uintptr_t>(src) & 15) == 0);
  if (vec) {
    const long long total = (long long)rows * (channels / 4);
    um::split_planes_kernel<4><<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        src, ld, channels, reinterpret_cast<__half*>(dst), cp, off, plane, rows);
  } else {
    const long long total = (long long)rows * channels;
    um::split_planes_kernel<1><<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        src, ld, channels, reinterpret_cast<__half*>(dst), cp, off, plane, rows);
  }
  return um::check_launch("um_split_planes");
}

}  // extern "C"
