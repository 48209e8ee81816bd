// Evaluation statistics: predictions + ground truth of a batch -> a [B, S] float64 table of per-sample sufficient statistics
// (counts and sums), from which the host forms the metrics of the reference's validate_* loops (evaluate_flow.py,
// evaluate_stereo.py, evaluate_depth.py).
//
// Arithmetic: every per-pixel value is computed with explicitly rounded fp32 intrinsics (no FMA contraction), in the order
// the reference's torch / numpy expressions evaluate it, so each epe / error / ratio is the reference's fp32 value and every
// count equals the reference's count (logf may differ from numpy's float32 log by 1 ulp: only the log-error sum sees it; the
// reference's torch CPU sqrt is not correctly rounded, which can move a flow count only within one ulp of a threshold).
// Sums are fp64 in a fixed order: each thread walks a fixed pixel set, each CTA reduces its threads in a fixed tree into a
// partial row, and a second kernel adds the UM_EVAL_PARTS partial rows of a sample in index order.  The grid does not depend
// on the device, there are no floating-point atomics: a launch is bit-reproducible, eager or inside a CUDA graph.
#include "um_common.cuh"

namespace {

constexpr int kThreads = 256;

template <int TASK> struct Cols;
template <> struct Cols<UM_EVAL_FLOW> { static constexpr int n = UM_EVAL_FLOW_COLS; };
template <> struct Cols<UM_EVAL_STEREO> { static constexpr int n = UM_EVAL_STEREO_COLS; };
template <> struct Cols<UM_EVAL_DEPTH> { static constexpr int n = UM_EVAL_DEPTH_COLS; };

struct EvalArgs {
  const float* pred;
  long long sb, sc, sy, sx;        // prediction strides (elements)
  const float* gt;                 // contiguous [B, C, h, w]
  const float* valid;              // contiguous [B, h, w] or NULL
  const float* noc;                // contiguous [B, h, w] or NULL
  int mask_mode;
  float max_val, eval_min, eval_max;
  int h, w;
};

// utils/utils.py:compute_out_of_boundary_mask of the GT flow at pixel (x, y): the correspondence stays inside the image and
// neither component exceeds the image size.
__device__ __forceinline__ bool in_image(float gu, float gv, int x, int y, int h, int w) {
  const float mw = (float)(w - 1), mh = (float)(h - 1);
  const float cx = __fadd_rn((float)x, gu), cy = __fadd_rn((float)y, gv);
  return cx >= 0.f && cx <= mw && cy >= 0.f && cy <= mh && fabsf(gu) <= mw && fabsf(gv) <= mh;
}

template <int TASK>
__device__ __forceinline__ void accumulate(const EvalArgs& a, int b, int y, int x, double* acc) {
  const long long hw = (long long)a.h * a.w, pix = (long long)y * a.w + x;
  const float* pr = a.pred + b * a.sb + y * a.sy + x * a.sx;
  if (TASK == UM_EVAL_FLOW) {
    const float* g = a.gt + (long long)b * 2 * hw + pix;
    const float gu = __ldg(g), gv = __ldg(g + hw);
    const float du = __fsub_rn(__ldg(pr), gu), dv = __fsub_rn(__ldg(pr + a.sc), gv);
    // torch.sum((flow - flow_gt) ** 2, dim=0).sqrt() and the same of the GT (evaluate_flow.py:425, :436, :553-554)
    const float epe = __fsqrt_rn(__fadd_rn(__fmul_rn(du, du), __fmul_rn(dv, dv)));
    const float mag = __fsqrt_rn(__fadd_rn(__fmul_rn(gu, gu), __fmul_rn(gv, gv)));
    bool m = true;
    if (a.mask_mode != UM_EVAL_MASK_ALL) {
      const float v = __ldg(a.valid + b * hw + pix);
      m = v >= 0.5f && (a.mask_mode == UM_EVAL_MASK_VALID || mag < a.max_val);   // valid * (mag < max) >= 0.5 (:299-303)
    }
    if (!m) return;
    const double e = (double)epe;
    acc[UM_EVF_N] += 1.0;
    acc[UM_EVF_EPE] += e;
    acc[UM_EVF_1PX] += epe > 1.f ? 1.0 : 0.0;
    acc[UM_EVF_3PX] += epe > 3.f ? 1.0 : 0.0;
    acc[UM_EVF_5PX] += epe > 5.f ? 1.0 : 0.0;
    acc[UM_EVF_OUTLIER] += (epe > 3.f && __fdiv_rn(epe, mag) > 0.05f) ? 1.0 : 0.0;   // :593
    // speed bins (:437-447); a NaN speed falls in none.  Constant indices only: keeps `acc` in registers.
    const double s0 = mag < 10.f ? 1.0 : 0.0, s1 = (mag >= 10.f && mag <= 40.f) ? 1.0 : 0.0, s2 = mag > 40.f ? 1.0 : 0.0;
    acc[UM_EVF_S0_10_N] += s0;
    acc[UM_EVF_S0_10_EPE] += s0 != 0.0 ? e : 0.0;          // selects, not s * e: 0 * inf would be NaN
    acc[UM_EVF_S10_40_N] += s1;
    acc[UM_EVF_S10_40_EPE] += s1 != 0.0 ? e : 0.0;
    acc[UM_EVF_S40_N] += s2;
    acc[UM_EVF_S40_EPE] += s2 != 0.0 ? e : 0.0;
    if (a.noc) {
      const double mt = (__ldg(a.noc + b * hw + pix) > 0.5f && in_image(gu, gv, x, y, a.h, a.w)) ? 1.0 : 0.0;   // :429
      acc[UM_EVF_MATCHED_N] += mt;
      acc[UM_EVF_MATCHED_EPE] += mt != 0.0 ? e : 0.0;
      acc[UM_EVF_UNMATCHED_N] += 1.0 - mt;
      acc[UM_EVF_UNMATCHED_EPE] += mt != 0.0 ? 0.0 : e;
    }
  } else if (TASK == UM_EVAL_STEREO) {
    const float gt = __ldg(a.gt + b * hw + pix);
    if (!(gt > 0.f && (a.max_val <= 0.f || gt < a.max_val))) return;     // evaluate_stereo.py:350, :453
    const float e = fabsf(__fsub_rn(gt, __ldg(pr)));                      // loss/stereo_metric.py: |d_gt - d_est|
    acc[UM_EVS_N] += 1.0;
    acc[UM_EVS_ABS] += (double)e;
    const float rel = __fdiv_rn(e, gt);
    acc[UM_EVS_D1] += (e > 3.f && rel > 0.05f) ? 1.0 : 0.0;
    acc[UM_EVS_1PX] += e > 1.f ? 1.0 : 0.0;
    acc[UM_EVS_2PX] += e > 2.f ? 1.0 : 0.0;
    acc[UM_EVS_3PX] += e > 3.f ? 1.0 : 0.0;
  } else {
    const float gt = __ldg(a.gt + b * hw + pix);
    if (!(gt > a.eval_min && gt < a.eval_max)) return;                     // evaluate_depth.py:88-91
    if (a.valid && !(__ldg(a.valid + b * hw + pix) > 0.5f)) return;
    const float pd = __ldg(pr);
    // loss/depth_loss.py:compute_errors on float32 arrays
    const float d = __fsub_rn(gt, pd);
    const float d2 = __fmul_rn(d, d);
    const float lg = __fsub_rn(logf(gt), logf(pd));
    const float r0 = __fdiv_rn(gt, pd), r1 = __fdiv_rn(pd, gt);
    const float th = (r0 != r0 || r1 != r1) ? __int_as_float(0x7fc00000) : fmaxf(r0, r1);   // np.maximum propagates NaN
    acc[UM_EVD_N] += 1.0;
    acc[UM_EVD_ABS_REL] += (double)__fdiv_rn(fabsf(d), gt);
    acc[UM_EVD_SQ_REL] += (double)__fdiv_rn(d2, gt);
    acc[UM_EVD_SQ] += (double)d2;
    acc[UM_EVD_LOG_SQ] += (double)__fmul_rn(lg, lg);
    acc[UM_EVD_A1] += th < 1.25f ? 1.0 : 0.0;
    acc[UM_EVD_A2] += th < 1.5625f ? 1.0 : 0.0;
    acc[UM_EVD_A3] += th < 1.953125f ? 1.0 : 0.0;
  }
}

// grid (UM_EVAL_PARTS, B): CTA p of sample b walks pixels p*256 + t, p*256 + t + PARTS*256, ... and writes one partial row.
template <int TASK>
__global__ void __launch_bounds__(kThreads) eval_partial_kernel(EvalArgs a, double* __restrict__ partial) {
  constexpr int S = Cols<TASK>::n;
  double acc[S];
#pragma unroll
  for (int c = 0; c < S; ++c) acc[c] = 0.0;
  const int b = blockIdx.y;
  const int hw = a.h * a.w;                          // < 2^31 (checked by the launcher): 32-bit index arithmetic
  for (int p = blockIdx.x * kThreads + threadIdx.x; p < hw; p += UM_EVAL_PARTS * kThreads) {
    const int y = p / a.w, x = p - y * a.w;
    accumulate<TASK>(a, b, y, x, acc);
  }
  __shared__ double red[kThreads / 32][S];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int c = 0; c < S; ++c) {
    double v = acc[c];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) red[warp][c] = v;
  }
  __syncthreads();
  if (threadIdx.x < S) {
    double v = red[0][threadIdx.x];
#pragma unroll
    for (int i = 1; i < kThreads / 32; ++i) v += red[i][threadIdx.x];
    partial[((long long)b * UM_EVAL_PARTS + blockIdx.x) * S + threadIdx.x] = v;
  }
}

// out[b, c] = sum over p = 0 .. PARTS-1 of partial[b, p, c], in that order.
__global__ void __launch_bounds__(kThreads) eval_final_kernel(const double* __restrict__ partial, double* __restrict__ out,
                                                              int S, int total) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= total) return;
  const int b = i / S, c = i - b * S;
  const double* p = partial + (long long)b * UM_EVAL_PARTS * S + c;
  double v = 0.0;
  for (int k = 0; k < UM_EVAL_PARTS; ++k) v += p[(long long)k * S];
  out[i] = v;
}

template <int TASK>
int launch(const EvalArgs& a, int batch, double* scratch, double* out, cudaStream_t st) {
  constexpr int S = Cols<TASK>::n;
  eval_partial_kernel<TASK><<<dim3(UM_EVAL_PARTS, (unsigned)batch), kThreads, 0, st>>>(a, scratch);
  if (int rc = um::check_launch("um_eval_stats")) return rc;
  const int total = batch * S;
  eval_final_kernel<<<(total + kThreads - 1) / kThreads, kThreads, 0, st>>>(scratch, out, S, total);
  return um::check_launch("um_eval_stats");
}

}  // namespace

extern "C" {

int um_eval_stats(const float* pred, int64_t pred_sb, int64_t pred_sc, int64_t pred_sy, int64_t pred_sx, const float* gt,
                  const float* valid, const float* noc_valid, int32_t task, int32_t mask_mode, float max_val, float eval_min,
                  float eval_max, int32_t batch, int32_t h, int32_t w, double* scratch, double* out, void* stream) {
  UM_REQUIRE(pred && gt && scratch && out, "um_eval_stats: pred, gt, scratch and out must be non-null");
  UM_REQUIRE(task == UM_EVAL_FLOW || task == UM_EVAL_STEREO || task == UM_EVAL_DEPTH, "um_eval_stats: unknown task %d", task);
  UM_REQUIRE(batch > 0 && h > 0 && w > 0 && batch <= 65535 && (int64_t)h * w < ((int64_t)1 << 31) - UM_EVAL_PARTS * 256,
             "um_eval_stats: bad sizes (batch %d, %d x %d)", batch, h, w);
  UM_REQUIRE(pred_sx >= 1 && pred_sy >= (int64_t)w * pred_sx &&
                 (task != UM_EVAL_FLOW || pred_sc >= (int64_t)h * pred_sy) &&
                 pred_sb >= (task == UM_EVAL_FLOW ? 2 * pred_sc : (int64_t)h * pred_sy),
             "um_eval_stats: bad prediction strides (b %lld, c %lld, y %lld, x %lld): the view must not overlap itself",
             (long long)pred_sb, (long long)pred_sc, (long long)pred_sy, (long long)pred_sx);
  if (task == UM_EVAL_FLOW) {
    UM_REQUIRE(mask_mode == UM_EVAL_MASK_ALL || mask_mode == UM_EVAL_MASK_VALID || mask_mode == UM_EVAL_MASK_VALID_MAX,
               "um_eval_stats: unknown flow mask mode %d", mask_mode);
    UM_REQUIRE(mask_mode == UM_EVAL_MASK_ALL || valid, "um_eval_stats: this flow mask mode needs the valid mask");
  } else {
    UM_REQUIRE(!noc_valid, "um_eval_stats: noc_valid is a flow-only mask");
  }
  const EvalArgs a{pred, pred_sb, pred_sc, pred_sy, pred_sx, gt, valid, noc_valid, mask_mode, max_val, eval_min, eval_max, h, w};
  cudaStream_t st = (cudaStream_t)stream;
  if (task == UM_EVAL_FLOW) return launch<UM_EVAL_FLOW>(a, batch, scratch, out, st);
  if (task == UM_EVAL_STEREO) return launch<UM_EVAL_STEREO>(a, batch, scratch, out, st);
  return launch<UM_EVAL_DEPTH>(a, batch, scratch, out, st);
}

}  // extern "C"
