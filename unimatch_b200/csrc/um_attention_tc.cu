// Fused window attention on the Hopper tensor cores (wgmma + TMA), fp32-faithful.
//
//   out = softmax(Q K^T / sqrt(C) + mask) V   per Swin window; the Lw x Lw scores live only in registers.
//
// Precision: operands are fp32 values split into (hi, lo) fp16 pairs (same bytes as fp32); every product is
// formed as hi*hi + hi*lo + lo*hi on fp16 MMAs with fp32 accumulation ("3xFP16", error ~2^-22 per product, i.e. the
// accuracy of an fp32 dot product) -- one-pass TF32/BF16 moves the final flow by whole pixels on this network
// (SURVEY.md §7.2 #1), so it is not an option for parity.
//
// Data flow
//   1. um_split_windows: q/k/v fp32 token rows -> window-major, cyclically shifted, zero-padded fp16 hi/lo planes
//      [part][stream][window][Lp][128] (Lp = Lw rounded up to 128), so every tile is a dense 2-D TMA box.
//   2. attn_tc_kernel: one CTA per (128-query tile, window, stream); warp-specialised:
//        warp 0          TMA producer   Q once; K and V tiles of 64 keys through two 2-stage mbarrier rings
//        warpgroups 1-2  consumers      64 query rows each: S_j = Q K_j^T (24 wgmma 64x64x16) into registers, scale /
//                                       mask, online softmax with lazy rescale, P as fp16 (hi, lo) register operands
//                                       and O += P_j V_j (12 wgmma 64x128x16, V as MN-major B operand) into registers;
//                                       epilogue O / l -> smem transpose -> coalesced rows at the un-shifted tokens
//   3. the ragged last query tile (Lw mod 128 rows) runs the same code on zero-padded rows whose stores are masked.
//
// Reference semantics: attention.py:45-104 (split / roll / mask / softmax / merge / roll back), utils.py:84-108.
#include <math_constants.h>

#include "um_common.cuh"
#include "um_tc.cuh"

namespace um {

using namespace tc;

namespace {

constexpr int BM = 128, BN = 64;
// 2 consumer warpgroups (warps 0-7) + one TMA producer warp (warp 8)
constexpr int NTHREADS = 288;
constexpr int PRODUCER = 8;
constexpr uint32_t Q_BYTES = 4 * 16384;          // (hi, lo) x (ch 0-63, 64-127) x [128 rows x 128 B]
constexpr uint32_t KV_STAGE_BYTES = 4 * 8192;    // (hi, lo) x (2 halves) x [64 rows x 128 B]
constexpr uint32_t OFF_Q = 0;
constexpr uint32_t OFF_K = OFF_Q + Q_BYTES;                  // 2 stages
constexpr uint32_t OFF_V = OFF_K + 2 * KV_STAGE_BYTES;       // 2 stages
constexpr uint32_t OFF_X = OFF_V + 2 * KV_STAGE_BYTES;       // softmax-expectation key values [2][64][2] fp32
constexpr uint32_t OFF_BAR = OFF_X + 1024;
constexpr uint32_t OFF_KREG = OFF_BAR + 256;
constexpr int MAX_LP = 2048;
constexpr uint32_t SMEM_BYTES = OFF_KREG + MAX_LP;           // 200960
constexpr float SQRT_C = 11.313708498984761f;
constexpr float EXP_SCALE = 1.4426950408889634f / 11.313708498984761f;   // log2(e) / sqrt(128)
constexpr float LAZY_THRESH = 8.0f / EXP_SCALE;              // raw-logit units: rescale when the max grows by > 2^8

struct TcParams {
  float* out; long long ldo;
  int n_streams, kv_shift, lp;      // n_streams = streams in the operand planes (key stream = (n + kv_shift) mod n_streams)
  Geom g;
  // softmax-expectation variant (HAS_V = false): out[n, t, 0..vdim) = post(sum_k p_k value_k)
  const float* values; int vdim, value_mode, post_op;
  // optional second output: the same rows as fp16 (hi, lo) planes [2][rows][128] (token order), i.e. the operand planes of the
  // merge Linear layer -- saves the separate fp32 -> planes pass
  __half* out_split; long long split_plane;
};

__device__ __forceinline__ uint32_t pack_h2(__half a, __half b) {
  return (uint32_t)__half_as_ushort(a) | ((uint32_t)__half_as_ushort(b) << 16);
}

// HAS_V = true : fused attention, O = softmax(S) V through a second MMA chain.
// HAS_V = false: softmax expectation (global correlation soft-argmax, matching.py:7-36; global flow propagation,
//                attention.py:194-215): the values are 1-2 numbers per key, so sum_k p_k value_k is accumulated in
//                registers straight from the S tile -- no V tile, no second MMA.
template <bool HAS_V>
__global__ void __launch_bounds__(NTHREADS, 1)
attn_tc_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
               const __grid_constant__ CUtensorMap map_v, TcParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
  uint64_t* q_full = bars + 0;
  uint64_t* k_full = bars + 1;      // [2]   K and V tiles travel through SEPARATE rings: a K slot is free as soon as
  uint64_t* k_empty = bars + 3;     // [2]   S_j = Q K_j^T has been computed, long before P_j V_j releases the V slot
  uint64_t* v_full = bars + 5;      // [2]
  uint64_t* v_empty = bars + 7;     // [2]
  int8_t* kreg = reinterpret_cast<int8_t*>(smem + OFF_KREG);

  const Geom g = p.g;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.x * BM, win = blockIdx.y, n = blockIdx.z;
  const int nk = (n + p.kv_shift) % p.n_streams;
  const int nwin = g.nwin, lp = p.lp;
  const int T = (g.lw + BN - 1) / BN;                     // key tiles
  const int planes = p.n_streams * nwin * lp;             // rows per (hi | lo) plane

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(k_full + i, 1); mbar_init(k_empty + i, 8);   // empty: one arrival per consumer warp
      mbar_init(v_full + i, 1); mbar_init(v_empty + i, 8);
    }
    fence_barrier_init();
  }
  if (warp == PRODUCER && lane == 0) { tma_prefetch_desc(&map_q); tma_prefetch_desc(&map_k); tma_prefetch_desc(&map_v); }
  // shift-region table of the keys of this window (utils.py:84-108); uniform windows skip masking altogether
  bool masked = false;
  if (g.mask_mode == UM_MASK_SWIN) {
    const int wy = win / g.kw, wx = win - wy * g.kw;
    masked = (g.sh > 0 && wy == g.kh - 1) || (g.sw > 0 && wx == g.kw - 1);
    if (masked)
      for (int t = threadIdx.x; t < g.lw; t += NTHREADS) {
        int yr, xr;
        window_token(g, win, t, &yr, &xr);
        kreg[t] = (int8_t)shift_region(g, yr, xr);
      }
  }
  __syncthreads();

  if (warp == PRODUCER) {
    // =============================== TMA producer (converged warp, one elected lane issues) ===============================
    const int qrow = (n * nwin + win) * lp + m0;
    if (elect_one()) {
      mbar_arrive_expect_tx(q_full, Q_BYTES);
#pragma unroll
      for (int part = 0; part < 2; ++part)
#pragma unroll
        for (int half = 0; half < 2; ++half)
          tma_load_2d(smem + OFF_Q + (part * 2 + half) * 16384, &map_q, q_full, half * 64, part * planes + qrow);
    }
    __syncwarp();
    const int krow = (nk * nwin + win) * lp;
    auto load_tile = [&](int j, const CUtensorMap* map, uint32_t off, uint64_t* full, uint64_t* empty) {
      const int s = j & 1;
      mbar_wait_inline(empty + s, ((j >> 1) & 1) ^ 1);
      if (elect_one()) {
        mbar_arrive_expect_tx(full + s, KV_STAGE_BYTES);
#pragma unroll
        for (int part = 0; part < 2; ++part)
#pragma unroll
          for (int half = 0; half < 2; ++half)
            tma_load_2d(smem + off + s * KV_STAGE_BYTES + (part * 2 + half) * 8192, map, full + s, half * 64,
                        part * planes + krow + j * BN);
      }
      __syncwarp();
    };
    // K_{j+1} is requested before V_j: the K slot comes free (S_{j-1} done) a whole softmax earlier than the V slot
    load_tile(0, &map_k, OFF_K, k_full, k_empty);
    for (int j = 0; j < T; ++j) {
      if (j + 1 < T) load_tile(j + 1, &map_k, OFF_K, k_full, k_empty);
      if (HAS_V) load_tile(j, &map_v, OFF_V, v_full, v_empty);
    }
    return;
  }

  // =============================== consumers: softmax / PV / epilogue ===============================
  const int cw = warp;                                      // consumer warp 0..7
  const int wg = cw >> 2;                                   // query rows [64 wg, 64 wg + 64) of the tile
  const int fr = wg * 64 + (cw & 3) * 16 + (lane >> 2);     // this thread's rows fr and fr + 8 (MMA fragment layout)
  const int fc = 2 * (lane & 3);                            // ... and columns 8 j + fc + {0, 1}
  int rq[2] = {0, 0}, tok[2];
  bool row_valid[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int tq = m0 + fr + 8 * h;                         // rows >= lw of the last tile are zero padding
    row_valid[h] = tq < g.lw;
    int yr = 0, xr = 0;
    tok[h] = row_valid[h] ? window_token(g, win, tq, &yr, &xr) : -1;
    if (masked) rq[h] = shift_region(g, yr, xr);
  }
  float m_run[2] = {-CUDART_INF_F, -CUDART_INF_F}, l_run[2] = {0.f, 0.f};
  const uint32_t q_base = smem_u32(smem + OFF_Q) + wg * 8192;
  auto consumers_sync = [&]() { asm volatile("bar.sync 1, 256;" ::: "memory"); };

  // S_j = Q K_j^T for this warpgroup's 64 rows; the K slot is released as soon as the MMAs are complete
  auto compute_s = [&](int j, float (&sv)[32]) {
    const int s = j & 1;
    mbar_wait_inline(k_full + s, (j >> 1) & 1);
    const uint32_t k_base = smem_u32(smem + OFF_K + s * KV_STAGE_BYTES);
    const int qa[3] = {1, 0, 0}, kb[3] = {0, 1, 0};        // (q part, k part): lo*hi, hi*lo, hi*hi
    fence_acc(sv);
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
      for (int half = 0; half < 2; ++half)
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
          wgmma_ss<BN>(sv, desc_kmajor(q_base + (qa[c] * 2 + half) * 16384 + ks * 32),
                       desc_kmajor(k_base + (kb[c] * 2 + half) * 8192 + ks * 32), (c | half | ks) != 0);
    wgmma_commit();
    wgmma_wait<0>();
    fence_acc(sv);
    __syncwarp();
    if (lane == 0) mbar_arrive(k_empty + s);
  };
  mbar_wait_inline(q_full, 0);

  if (!HAS_V) {
    // ---------------- softmax expectation: per-key values staged in shared memory, sums kept in registers ----------------
    float* vals = reinterpret_cast<float*>(smem + OFF_X);  // [2 buffers][64 keys][2]
    const int et = threadIdx.x;
    const long long L = (long long)g.h * g.w;
    float a0[2] = {0.f, 0.f}, a1[2] = {0.f, 0.f};
    for (int j = 0; j < T; ++j) {
      const int s = j & 1;
      const int n0 = j * BN;
      if (et < BN) {                                       // value of key n0 + et (keys of the key stream nk)
        float v0 = 0.f, v1 = 0.f;
        const int t = n0 + et;
        if (t < g.lw) {
          const int ktok = window_token(g, win, t);
          if (p.value_mode == UM_VALUE_TENSOR) {
            const float* vp = p.values + ((long long)nk * L + ktok) * p.vdim;
            v0 = __ldg(vp); v1 = (p.vdim > 1) ? __ldg(vp + 1) : 0.f;
          } else {
            const int ky = ktok / g.w;
            v0 = (float)(ktok - ky * g.w); v1 = (float)ky;
          }
        }
        vals[(s * BN + et) * 2] = v0; vals[(s * BN + et) * 2 + 1] = v1;
      }
      float sv[32];
      compute_s(j, sv);
      consumers_sync();                                     // values of this tile are visible
      const float2* vv = reinterpret_cast<const float2*>(vals + s * BN * 2);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float mx = -CUDART_INF_F;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float& x = sv[4 * jj + 2 * h + e];
            if (n0 + 8 * jj + fc + e >= g.lw) x = -CUDART_INF_F;   // ragged last key tile
            mx = fmaxf(mx, x);
          }
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        const float m_new = fmaxf(m_run[h], mx);
        const float alpha = exp2f((m_run[h] - m_new) * EXP_SCALE);
        m_run[h] = m_new;
        const float mscaled = m_new * EXP_SCALE;
        float sum = 0.f, b0 = 0.f, b1 = 0.f;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float pe = ex2_approx(fmaf(sv[4 * jj + 2 * h + e], EXP_SCALE, -mscaled));
            const float2 kv = vv[8 * jj + fc + e];
            sum += pe;
            b0 = fmaf(pe, kv.x, b0);
            b1 = fmaf(pe, kv.y, b1);
          }
        l_run[h] = l_run[h] * alpha + sum;
        a0[h] = a0[h] * alpha + b0;
        a1[h] = a1[h] * alpha + b1;
      }
    }
    // combine the four threads of every row (same running max in all of them)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int o = 1; o <= 2; o <<= 1) {
        l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], o);
        a0[h] += __shfl_xor_sync(0xffffffffu, a0[h], o);
        a1[h] += __shfl_xor_sync(0xffffffffu, a1[h], o);
      }
      if (row_valid[h] && (lane & 3) == 0) {
        float r0 = a0[h] / l_run[h], r1 = a1[h] / l_run[h];
        const int oy = tok[h] / g.w, ox = tok[h] - oy * g.w;
        if (p.post_op == UM_POST_MINUS_OWN) { r0 -= (float)ox; r1 -= (float)oy; }
        else if (p.post_op == UM_POST_OWN_MINUS) { r0 = (float)ox - r0; }
        float* dst = p.out + ((long long)n * L + tok[h]) * p.vdim;
        dst[0] = r0;
        if (p.vdim > 1) dst[1] = r1;
      }
    }
    return;
  }

  float o[64];                                              // O: 64 rows x 128 channels of this warpgroup
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  for (int j = 0; j < T; ++j) {
    const int s = j & 1;
    const int n0 = j * BN;
    float sv[32];
    compute_s(j, sv);
    uint32_t ph[16], pl[16];                                // P as fp16 (hi, lo) pairs, already in the A-operand layout
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      // masks only where they can apply: windows touching a shift-region boundary, the ragged last key tile
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = n0 + 8 * jj + fc + e;
          float& x = sv[4 * jj + 2 * h + e];
          if (masked && kreg[col < g.lw ? col : 0] != rq[h]) x -= 100.0f * SQRT_C;
          if (col >= g.lw) x = -CUDART_INF_F;
        }
      float mx = -CUDART_INF_F;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) mx = fmaxf(mx, fmaxf(sv[4 * jj + 2 * h], sv[4 * jj + 2 * h + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      float alpha = 1.0f;
      if (mx > m_run[h] + LAZY_THRESH) {                    // first tile: m_run = -inf -> true
        alpha = exp2f((m_run[h] - mx) * EXP_SCALE);         // exp2(-inf) = 0 on the first tile
        m_run[h] = mx;
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) { o[4 * jj + 2 * h] *= alpha; o[4 * jj + 2 * h + 1] *= alpha; }
      }
      const float mscaled = m_run[h] * EXP_SCALE;
      float sum = 0.f;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const float p0 = ex2_approx(fmaf(sv[4 * jj + 2 * h], EXP_SCALE, -mscaled));
        const float p1 = ex2_approx(fmaf(sv[4 * jj + 2 * h + 1], EXP_SCALE, -mscaled));
        sum += p0 + p1;
        split_f16x2(p0, p1, &ph[2 * jj + h], &pl[2 * jj + h]);
      }
      l_run[h] = l_run[h] * alpha + sum;                    // partial row sum (combined in the epilogue)
    }
    // O += P V: A = P from registers (16 keys per MMA), B = V tile, MN-major
    mbar_wait_inline(v_full + s, (j >> 1) & 1);
    const uint32_t v_base = smem_u32(smem + OFF_V + s * KV_STAGE_BYTES);
    fence_acc(o);
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const uint32_t* pp = c == 0 ? pl : ph;              // lo*hi, hi*lo, hi*hi
        const uint32_t a[4] = {pp[4 * ks], pp[4 * ks + 1], pp[4 * ks + 2], pp[4 * ks + 3]};
        wgmma_rs_n128_tb(o, a, desc_mnmajor(v_base + (c == 1 ? 16384 : 0) + ks * 2048, 8192), true);
      }
    wgmma_commit();
    wgmma_wait<0>();
    fence_acc(o);
    __syncwarp();
    if (lane == 0) mbar_arrive(v_empty + s);
  }

  // ---- epilogue: O / l -> smem (reusing the Q region once both warpgroups are done with it) -> coalesced 512-byte rows ----
  float inv[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float l = l_run[h];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    inv[h] = 1.0f / l;
  }
  consumers_sync();
  float* osm = reinterpret_cast<float*>(smem + OFF_Q);     // [128][128] fp32, 16-byte chunks XOR-swizzled by row
#pragma unroll
  for (int jj = 0; jj < 16; ++jj)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = fr + 8 * h, col = 8 * jj + fc;
      *reinterpret_cast<float2*>(osm + row * 128 + (((col >> 2) ^ (row & 31)) << 2) + (col & 3)) =
          make_float2(o[4 * jj + 2 * h] * inv[h], o[4 * jj + 2 * h + 1] * inv[h]);
    }
  consumers_sync();
  float* obase = p.out + (long long)n * g.h * g.w * p.ldo;
  for (int row = cw * 16; row < cw * 16 + 16; ++row) {
    const int tq = m0 + row;
    if (tq >= g.lw) break;                                  // warp-uniform
    const int tk = window_token(g, win, tq);
    const float4 v = *reinterpret_cast<const float4*>(osm + row * 128 + ((lane ^ (row & 31)) << 2));
    if (p.out) *reinterpret_cast<float4*>(obase + (long long)tk * p.ldo + lane * 4) = v;
    if (p.out_split) {
      uint32_t h0, h1, l0, l1;
      split_f16x2(v.x, v.y, &h0, &l0);
      split_f16x2(v.z, v.w, &h1, &l1);
      __half* d = p.out_split + ((long long)n * g.h * g.w + tk) * 128 + lane * 4;
      *reinterpret_cast<uint2*>(d) = make_uint2(h0, h1);
      *reinterpret_cast<uint2*>(d + p.split_plane) = make_uint2(l0, l1);
    }
  }
}

// ---- q/k/v fp32 rows -> window-major fp16 (hi, lo) planes -----------------------------------------------------
struct SplitParams {
  const float* src[3]; long long ld[3];
  __half* dst[3];            // each: [2][n_streams][nwin][lp][128]
  int n_streams, lp;
  Geom g;
};

__global__ void __launch_bounds__(256) split_windows_kernel(SplitParams p) {
  const Geom g = p.g;
  const int lane = threadIdx.x & 31;
  const int t = blockIdx.x * 8 + (threadIdx.x >> 5);      // row inside the padded window
  const int win = blockIdx.y, n = blockIdx.z;
  if (t >= p.lp) return;
  const long long planes = (long long)p.n_streams * g.nwin * p.lp;
  const long long row = ((long long)n * g.nwin + win) * p.lp + t;
  const int tok = (t < g.lw) ? window_token(g, win, t) : -1;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    if (!p.src[a]) continue;
    float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
    if (tok >= 0) x = __ldg(reinterpret_cast<const float4*>(p.src[a] + ((long long)n * g.h * g.w + tok) * p.ld[a]) + lane);
    __half h[4], l[4];
    split_f16(x.x, &h[0], &l[0]); split_f16(x.y, &h[1], &l[1]);
    split_f16(x.z, &h[2], &l[2]); split_f16(x.w, &h[3], &l[3]);
    uint2 hv = make_uint2(pack_h2(h[0], h[1]), pack_h2(h[2], h[3]));
    uint2 lv = make_uint2(pack_h2(l[0], l[1]), pack_h2(l[2], l[3]));
    reinterpret_cast<uint2*>(p.dst[a] + row * 128)[lane] = hv;
    reinterpret_cast<uint2*>(p.dst[a] + (planes + row) * 128)[lane] = lv;
  }
}

}  // namespace

// ---- host side ---------------------------------------------------------------------------------------------------
PFN_encodeTiled get_encode_tiled() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* sym = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(sym);
  }
  return fn;
}

int make_map_2d_f16(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) { set_error("cuTensorMapEncodeTiled unavailable (no CUDA driver?)"); return UM_ECUDA; }
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols * 2};
  cuuint32_t box[2] = {64, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d)", (int)r); return UM_ECUDA; }
  return UM_OK;
}

static inline int padded_lw(int lw) { return (lw + 127) / 128 * 128; }

bool expectation_tc_supported(const Geom& g, int value_mode) {
  // one dense window covering the map (global matching / propagation), no mask
  return g.kh == 1 && g.kw == 1 && g.lw >= BM && g.mask_mode == UM_MASK_NONE && g.sh == 0 && g.sw == 0 &&
         (value_mode == UM_VALUE_TENSOR || value_mode == UM_VALUE_COORDS);
}

size_t expectation_tc_workspace_bytes(const Geom& g, int n_total) {
  return (size_t)2 * 2 * n_total * g.nwin * padded_lw(g.lw) * 128 * sizeof(__half);
}

bool attention_tc_supported(const Geom& g) {
  // dense 2-D windows with at least one full 128-query tile; the 1-D / tiny-window cases stay on CUDA cores
  return g.lw >= BM && padded_lw(g.lw) <= MAX_LP && (g.mask_mode == UM_MASK_NONE || g.mask_mode == UM_MASK_SWIN);
}

size_t attention_tc_workspace_bytes(const Geom& g, int n_streams) {
  return (size_t)3 * 2 * n_streams * g.nwin * padded_lw(g.lw) * 128 * sizeof(__half);
}

int split_windows_launch(const float* q, const float* k, const float* v, long long ldq, long long ldk, long long ldv,
                         __half* wq, __half* wk, __half* wv, int n_streams, const Geom& g, cudaStream_t st, const char* what) {
  SplitParams sp{};
  sp.src[0] = q; sp.src[1] = k; sp.src[2] = v;
  sp.ld[0] = ldq; sp.ld[1] = ldk; sp.ld[2] = ldv;
  sp.dst[0] = wq; sp.dst[1] = wk; sp.dst[2] = wv;
  sp.n_streams = n_streams; sp.lp = padded_lw(g.lw); sp.g = g;
  split_windows_kernel<<<dim3((sp.lp + 7) / 8, g.nwin, n_streams), 256, 0, st>>>(sp);
  return check_launch(what);
}

// the fused attention kernel on window-major operand planes [2][n_streams][nwin][lp][128] (one buffer per operand)

int attention_planes_launch(const __half* wq, const __half* wk, const __half* wv, float* out, long long ldo, __half* out_split,
                               long long split_plane, int n_streams, int kv_shift, const Geom& g, cudaStream_t st) {
  const int lp = padded_lw(g.lw);
  int rc;
  CUtensorMap mq, mk, mv;
  const uint64_t rows = (uint64_t)2 * n_streams * g.nwin * lp;
  if ((rc = make_map_2d_f16(&mq, wq, rows, 128, BM))) return rc;
  if ((rc = make_map_2d_f16(&mk, wk, rows, 128, BN))) return rc;
  if ((rc = make_map_2d_f16(&mv, wv, rows, 128, BN))) return rc;
  static PerDeviceBytes configured;
  if ((rc = ensure_smem(configured, attn_tc_kernel<true>, SMEM_BYTES, "attn_tc"))) return rc;
  TcParams p{};
  p.out = out; p.ldo = ldo; p.n_streams = n_streams; p.kv_shift = kv_shift; p.lp = lp; p.g = g;
  p.out_split = out_split; p.split_plane = split_plane;
  const int qtiles = (g.lw + BM - 1) / BM;                  // the ragged last tile is masked in the epilogue
  attn_tc_kernel<true><<<dim3(qtiles, g.nwin, n_streams), NTHREADS, SMEM_BYTES, st>>>(mq, mk, mv, p);
  return check_launch("um_window_attention(wgmma)");
}

// fp32 token rows in: split pass + kernel
int window_attention_tc(const float* q, const float* k, const float* v, float* out, int n_streams, int kv_shift,
                        long long ldq, long long ldk, long long ldv, long long ldo, const Geom& g, void* workspace,
                        cudaStream_t st) {
  const int lp = padded_lw(g.lw);
  const size_t plane_elems = (size_t)2 * n_streams * g.nwin * lp * 128;
  __half* wq = reinterpret_cast<__half*>(workspace);
  __half* wk = wq + plane_elems;
  __half* wv = wk + plane_elems;
  int rc = split_windows_launch(q, k, v, ldq, ldk, ldv, wq, wk, wv, n_streams, g, st, "um_window_attention(split)");
  if (rc) return rc;
  return attention_planes_launch(wq, wk, wv, out, ldo, nullptr, 0, n_streams, kv_shift, g, st);
}

int softmax_expectation_tc(const float* q, const float* k, const float* values, float* out, int n_streams, int n_total,
                           int kv_shift, long long ldq, long long ldk, int vdim, int value_mode, int post_op,
                           const Geom& g, void* workspace, cudaStream_t st) {
  const int lp = padded_lw(g.lw);
  const size_t plane_elems = (size_t)2 * n_total * g.nwin * lp * 128;
  __half* wq = reinterpret_cast<__half*>(workspace);
  __half* wk = wq + plane_elems;
  int rc = split_windows_launch(q, k, nullptr, ldq, ldk, 0, wq, wk, nullptr, n_total, g, st, "um_softmax_expectation(split)");
  if (rc) return rc;
  CUtensorMap mq, mk;
  const uint64_t rows = (uint64_t)2 * n_total * g.nwin * lp;
  if ((rc = make_map_2d_f16(&mq, wq, rows, 128, BM))) return rc;
  if ((rc = make_map_2d_f16(&mk, wk, rows, 128, BN))) return rc;
  static PerDeviceBytes configured;
  if ((rc = ensure_smem(configured, attn_tc_kernel<false>, SMEM_BYTES, "expect_tc"))) return rc;
  TcParams p{};
  p.out = out; p.ldo = vdim; p.n_streams = n_total; p.kv_shift = kv_shift; p.lp = lp; p.g = g;
  p.values = values; p.vdim = vdim; p.value_mode = value_mode; p.post_op = post_op;
  const int qtiles = (g.lw + BM - 1) / BM;
  attn_tc_kernel<false><<<dim3(qtiles, g.nwin, n_streams), NTHREADS, SMEM_BYTES, st>>>(mq, mk, mk, p);
  return check_launch("um_softmax_expectation(wgmma)");
}

}  // namespace um
