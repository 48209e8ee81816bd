// Fused windowed attention / softmax-expectation, exact-fp32 CUDA-core path.
//
// One CTA = one 64-query tile of one window of one stream; keys are streamed in 64-key tiles through
// shared memory with an online softmax, so the Lw x Lw score matrix never reaches HBM.  Window split,
// cyclic shift and the Swin region mask are pure index arithmetic (um::window_token / um::shift_region):
// no roll / split / merge copies, no [K*K, Lw, Lw] mask tensor.
//
// This is the general-shape path (any window length, 1-D row windows, causal stereo mask).  The
// tensor-core (wgmma) path in um_attention_tc.cu takes over the large 2-D windows.
//
// Reference semantics: attention.py:8-16, :19-42, :45-104, :107-163; matching.py:7-36, :126-151;
// attention.py:194-215.
#include <math_constants.h>

#include "um_common.cuh"

namespace {

constexpr int BM = 64;    // queries per CTA
constexpr int BN = 64;    // keys per tile
constexpr int NT = 256;   // threads: 16 x 16, each owns a 4 x 4 block of the score tile
constexpr int LDQ = BM + 4;
constexpr int LDK = BN + 4;
constexpr int LDP = BN + 4;
constexpr float SQRT_C = 11.313708498984761f;   // 128 ** 0.5

struct Params {
  const float* q; const float* k; const float* v; float* out;
  long long ldq, ldk, ldv, ldo;
  int n_total, kv_shift;
  um::Geom g;
  const float* values; int vdim, value_mode, post_op;
};

template <bool FEAT>
constexpr size_t smem_bytes() {
  size_t f = 128 * LDQ + 128 * LDK + (FEAT ? (BM * LDP + BN * 128) : (BN * 2));
  return f * sizeof(float) + (2 * BM + 2 * BN) * sizeof(int);
}

// gather a [rows x 128] tile of token rows into shared memory TRANSPOSED: dst[d * ld + m]
__device__ __forceinline__ void load_tile_transposed(float* dst, int ld, const float* base, long long ldg,
                                                     const int* tok, int tid) {
  const int m = tid & 63;
  const int t = tok[m];
  const float4* row = reinterpret_cast<const float4*>(base + (long long)(t < 0 ? 0 : t) * ldg);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c4 = (tid >> 6) + 4 * i;
    float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
    if (t >= 0) x = __ldg(row + c4);
    float* d = dst + (c4 * 4) * ld + m;
    d[0] = x.x; d[ld] = x.y; d[2 * ld] = x.z; d[3 * ld] = x.w;
  }
}

template <bool FEAT>
__global__ void __launch_bounds__(NT) attn_simt_kernel(Params p) {
  extern __shared__ __align__(16) float smem[];
  float* Qs = smem;
  float* Ks = Qs + 128 * LDQ;
  float* Ps = Ks + 128 * LDK;                         // FEAT only
  float* Vs = FEAT ? (Ps + BM * LDP) : Ps;             // FEAT: [BN][128]; else [BN][2] key values
  int* q_tok = reinterpret_cast<int*>(Vs + (FEAT ? BN * 128 : BN * 2));
  int* k_tok = q_tok + BM;
  int* q_aux = k_tok + BN;                             // region id (SWIN) or rolled x (CAUSAL)
  int* k_aux = q_aux + BM;

  const um::Geom g = p.g;
  const int win = blockIdx.y, n = blockIdx.z;
  const int nk = (n + p.kv_shift) % p.n_total;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int m0 = blockIdx.x * BM;
  const long long L = (long long)g.h * g.w;

  if (tid < BM) {
    int t = m0 + tid, tok = -1, aux = 0;
    if (t < g.lw) {
      int yr, xr;
      tok = um::window_token(g, win, t, &yr, &xr);
      aux = (g.mask_mode == UM_MASK_SWIN) ? um::shift_region(g, yr, xr) : xr;
    }
    q_tok[tid] = tok; q_aux[tid] = aux;
  }
  __syncthreads();
  load_tile_transposed(Qs, LDQ, p.q + (long long)n * L * p.ldq, p.ldq, q_tok, tid);

  float m_run[4], l_run[4];
  float o[4][8];       // FEAT: 4 rows x 8 channels.  else: o[i][0..1] = running sum p*value
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    m_run[i] = -CUDART_INF_F; l_run[i] = 0.f;
#pragma unroll
    for (int c = 0; c < 8; ++c) o[i][c] = 0.f;
  }

  const float* kbase = p.k + (long long)nk * L * p.ldk;
  const float* vbase = FEAT ? (p.v + (long long)nk * L * p.ldv) : nullptr;

  for (int n0 = 0; n0 < g.lw; n0 += BN) {
    __syncthreads();   // previous tile fully consumed
    if (tid < BN) {
      int t = n0 + tid, tok = -1, aux = 0;
      if (t < g.lw) {
        int yr, xr;
        tok = um::window_token(g, win, t, &yr, &xr);
        aux = (g.mask_mode == UM_MASK_SWIN) ? um::shift_region(g, yr, xr) : xr;
      }
      k_tok[tid] = tok; k_aux[tid] = aux;
      if (!FEAT) {
        float v0 = 0.f, v1 = 0.f;
        if (tok >= 0) {
          if (p.value_mode == UM_VALUE_TENSOR) {
            const float* vp = p.values + ((long long)nk * L + tok) * p.vdim;
            v0 = vp[0]; v1 = (p.vdim > 1) ? vp[1] : 0.f;
          } else {
            int y = tok / g.w; v0 = (float)(tok - y * g.w); v1 = (float)y;
          }
        }
        Vs[tid * 2] = v0; Vs[tid * 2 + 1] = v1;
      }
    }
    __syncthreads();
    load_tile_transposed(Ks, LDK, kbase, p.ldk, k_tok, tid);
    if (FEAT) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        int idx = tid + NT * i, r = idx >> 5, c4 = idx & 31;
        int t = k_tok[r];
        float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
        if (t >= 0) x = __ldg(reinterpret_cast<const float4*>(vbase + (long long)t * p.ldv) + c4);
        *reinterpret_cast<float4*>(Vs + r * 128 + c4 * 4) = x;
      }
    }
    __syncthreads();

    // ---- S = Q K^T (4x4 per thread) ----
    float s[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
#pragma unroll 8
    for (int d = 0; d < 128; ++d) {
      float4 a = *reinterpret_cast<const float4*>(Qs + d * LDQ + ty * 4);
      float4 b = *reinterpret_cast<const float4*>(Ks + d * LDK + tx * 4);
      const float av[4] = {a.x, a.y, a.z, a.w};
      const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) s[i][j] = fmaf(av[i], bv[j], s[i][j]);
    }

    // ---- scale, mask, online softmax ----
    float alpha[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int qa = q_aux[ty * 4 + i];
      float mx = -CUDART_INF_F;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int col = tx * 4 + j;
        float v = s[i][j] / SQRT_C;
        if (g.mask_mode == UM_MASK_SWIN) { if (k_aux[col] != qa) v += -100.0f; }
        else if (g.mask_mode == UM_MASK_CAUSAL) { if (k_aux[col] > qa) v = -1e9f; }
        if (n0 + col >= g.lw) v = -CUDART_INF_F;
        s[i][j] = v;
        mx = fmaxf(mx, v);
      }
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
      const float m_new = fmaxf(m_run[i], mx);
      alpha[i] = expf(m_run[i] - m_new);
      float sum = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) { s[i][j] = expf(s[i][j] - m_new); sum += s[i][j]; }
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
      l_run[i] = l_run[i] * alpha[i] + sum;
      m_run[i] = m_new;
    }

    if (FEAT) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        *reinterpret_cast<float4*>(Ps + (ty * 4 + i) * LDP + tx * 4) = make_float4(s[i][0], s[i][1], s[i][2], s[i][3]);
#pragma unroll
        for (int c = 0; c < 8; ++c) o[i][c] *= alpha[i];
      }
      __syncthreads();
#pragma unroll 4
      for (int kk = 0; kk < BN; ++kk) {
        float4 v0 = *reinterpret_cast<const float4*>(Vs + kk * 128 + tx * 8);
        float4 v1 = *reinterpret_cast<const float4*>(Vs + kk * 128 + tx * 8 + 4);
        const float vv[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float pv = Ps[(ty * 4 + i) * LDP + kk];
#pragma unroll
          for (int c = 0; c < 8; ++c) o[i][c] = fmaf(pv, vv[c], o[i][c]);
        }
      }
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float a0 = o[i][0] * alpha[i], a1 = o[i][1] * alpha[i];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          a0 = fmaf(s[i][j], Vs[(tx * 4 + j) * 2], a0);
          a1 = fmaf(s[i][j], Vs[(tx * 4 + j) * 2 + 1], a1);
        }
        o[i][0] = a0; o[i][1] = a1;
      }
    }
  }

  // ---- epilogue ----
  if (FEAT) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int tok = q_tok[ty * 4 + i];
      if (tok < 0) continue;
      const float inv = 1.0f / l_run[i];
      float* dst = p.out + ((long long)n * L + tok) * p.ldo + tx * 8;
      *reinterpret_cast<float4*>(dst) = make_float4(o[i][0] * inv, o[i][1] * inv, o[i][2] * inv, o[i][3] * inv);
      *reinterpret_cast<float4*>(dst + 4) = make_float4(o[i][4] * inv, o[i][5] * inv, o[i][6] * inv, o[i][7] * inv);
    }
  } else {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float a0 = o[i][0], a1 = o[i][1];
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) {
        a0 += __shfl_xor_sync(0xffffffffu, a0, off);
        a1 += __shfl_xor_sync(0xffffffffu, a1, off);
      }
      const int tok = q_tok[ty * 4 + i];
      if (tx != 0 || tok < 0) continue;
      float r0 = a0 / l_run[i], r1 = a1 / l_run[i];
      const int y = tok / g.w, x = tok - y * g.w;
      if (p.post_op == UM_POST_MINUS_OWN) { r0 -= (float)x; r1 -= (float)y; }
      else if (p.post_op == UM_POST_OWN_MINUS) { r0 = (float)x - r0; }
      float* dst = p.out + ((long long)n * L + tok) * p.vdim;
      dst[0] = r0;
      if (p.vdim > 1) dst[1] = r1;
    }
  }
}

template <bool FEAT>
int launch(const Params& p, int n_streams, cudaStream_t st) {
  static um::PerDeviceBytes configured;
  if (int rc = um::ensure_smem(configured, attn_simt_kernel<FEAT>, smem_bytes<FEAT>(), "attn_simt")) return rc;
  dim3 grid((p.g.lw + BM - 1) / BM, p.g.nwin, n_streams);
  attn_simt_kernel<FEAT><<<grid, NT, smem_bytes<FEAT>(), st>>>(p);
  return um::check_launch(FEAT ? "um_window_attention(simt)" : "um_softmax_expectation(simt)");
}

}  // namespace

namespace um {

int window_attention_simt(const float* q, const float* k, const float* v, float* out, int n_streams, int kv_shift,
                          long long ldq, long long ldk, long long ldv, long long ldo, const Geom& g, cudaStream_t st) {
  Params p{};
  p.q = q; p.k = k; p.v = v; p.out = out;
  p.ldq = ldq; p.ldk = ldk; p.ldv = ldv; p.ldo = ldo;
  p.n_total = n_streams; p.kv_shift = kv_shift; p.g = g;
  return launch<true>(p, n_streams, st);
}

int softmax_expectation_simt(const float* q, const float* k, const float* values, float* out, int n_streams,
                             int n_total, int kv_shift, long long ldq, long long ldk, int vdim, int value_mode,
                             int post_op, const Geom& g, cudaStream_t st) {
  Params p{};
  p.q = q; p.k = k; p.v = nullptr; p.out = out;
  p.ldq = ldq; p.ldk = ldk; p.ldv = 0; p.ldo = vdim;
  p.n_total = n_total; p.kv_shift = kv_shift; p.g = g;
  p.values = values; p.vdim = vdim; p.value_mode = value_mode; p.post_op = post_op;
  return launch<false>(p, n_streams, st);
}

}  // namespace um
