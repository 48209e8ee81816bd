// C-ABI glue: error reporting, launch accounting, the attention entry points (argument checking + dispatch
// between the tensor-core and the general CUDA-core kernels) the point-track entries and the disparity warp (um_tracks.cu).  See include/unimatch_sm100.h.
#include <stdarg.h>

#include <atomic>
#include <initializer_list>

#include <cuda_fp16.h>

#include "um_common.cuh"

namespace um {

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int window_attention_simt(const float* q, const float* k, const float* v, float* out, int n_streams, int kv_shift,
                          long long ldq, long long ldk, long long ldv, long long ldo, const Geom& g, cudaStream_t st);
bool attention_tc_supported(const Geom& g);
size_t attention_tc_workspace_bytes(const Geom& g, int n_streams);
int window_attention_tc(const float* q, const float* k, const float* v, float* out, int n_streams, int kv_shift,
                        long long ldq, long long ldk, long long ldv, long long ldo, const Geom& g, void* workspace,
                        cudaStream_t st);
int attention_planes_launch(const __half* wq, const __half* wk, const __half* wv, float* out, long long ldo, __half* out_split,
                            long long split_plane, int n_streams, int kv_shift, const Geom& g, cudaStream_t st);
bool expectation_tc_supported(const Geom& g, int value_mode);
size_t expectation_tc_workspace_bytes(const Geom& g, int n_total);
int softmax_expectation_tc(const float* q, const float* k, const float* values, float* out, int n_streams, int n_total,
                           int kv_shift, long long ldq, long long ldk, int vdim, int value_mode, int post_op,
                           const Geom& g, void* workspace, cudaStream_t st);
int softmax_expectation_simt(const float* q, const float* k, const float* values, float* out, int n_streams,
                             int n_total, int kv_shift, long long ldq, long long ldk, int vdim, int value_mode,
                             int post_op, const Geom& g, cudaStream_t st);
int chain_tracks_launch(const float* flow, const float* occ, int n, int h, int w, float* pos, uint8_t* vis, float* pos_out,
                        uint8_t* vis_out, cudaStream_t st);
int track_points_forward_launch(const float* flow, const float* occ, int n, int h, int w, int t0, const float* queries,
                                int nq, int nt, float* pos, uint8_t* vis, float* tracks, uint8_t* visible, cudaStream_t st);
int track_points_backward_launch(const float* flow, const float* occ, int n, int h, int w, const float* queries, int nq,
                                 int nt, float* tracks, uint8_t* visible, cudaStream_t st);
int multi_flow_tracks_launch(const float* flow, const float* occ, const float* err, const int* src, const int* dst, int n,
                             int k, int h, int w, int r, float* pos, float* sig, uint8_t* vis, float* tracks,
                             uint8_t* visible, float* sigma, cudaStream_t st);
int warp_disparity_launch(const float* disp_next, const float* flow, float* disp1, uint8_t* in_frame, int batch, int h, int w,
                          cudaStream_t st);

static bool overlap(const void* a, long long abytes, const void* b, long long bbytes) {
  const uintptr_t x = reinterpret_cast<uintptr_t>(a), y = reinterpret_cast<uintptr_t>(b);
  return x < y + (uintptr_t)bbytes && y < x + (uintptr_t)abytes;
}

// every written buffer (the first n_out of bufs) overlaps no other buffer; NULL entries are absent
struct Span {
  const void* p;
  long long bytes;
};
static bool written_disjoint(std::initializer_list<Span> bufs, size_t n_out) {
  const Span* b = bufs.begin();
  for (size_t i = 0; i < n_out; ++i)
    for (size_t j = 0; j < bufs.size(); ++j)
      if (j != i && b[i].p && b[j].p && overlap(b[i].p, b[i].bytes, b[j].p, b[j].bytes)) return false;
  return true;
}

static bool aligned(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

}  // namespace um

extern "C" {

int um_abi_version(void) { return UM_ABI_VERSION; }

const char* um_build_info(void) {
  return "libunimatch_sm100 abi=" UM_STR(UM_ABI_VERSION) " arch=sm_90a cuda=" UM_STR(CUDART_VERSION) " built " __DATE__ " "
         __TIME__;
}

const char* um_last_error(void) { return um::g_err; }

int64_t um_launch_count(void) { return (int64_t)um::g_launches.load(std::memory_order_relaxed); }

int64_t um_window_attention_workspace(const um_attn_geom* geom, int32_t n_streams) {
  um::Geom g;
  if (!um::make_geom(geom, &g) || n_streams <= 0 || !um::attention_tc_supported(g)) return 0;
  return (int64_t)um::attention_tc_workspace_bytes(g, n_streams);
}

int32_t um_attention_planes_lp(const um_attn_geom* geom) {
  um::Geom g;
  if (!um::make_geom(geom, &g) || !um::attention_tc_supported(g)) return 0;
  return (g.lw + 127) / 128 * 128;
}

int um_window_attention_planes(const void* q_planes, const void* k_planes, const void* v_planes, float* out, int64_t ldo,
                               void* out_split, int64_t split_plane_stride, int32_t n_streams, int32_t kv_shift,
                               const um_attn_geom* geom, void* stream) {
  um::Geom g;
  UM_REQUIRE(q_planes && k_planes && v_planes && (out || out_split) && n_streams > 0,
             "um_window_attention_planes: null operand planes / no output / empty batch");
  UM_REQUIRE(um::make_geom(geom, &g), "um_window_attention_planes: bad geometry (h,w must be divisible by kh,kw)");
  UM_REQUIRE(um::attention_tc_supported(g),
             "um_window_attention_planes: geometry not built for the tensor-core kernel (um_attention_planes_lp() == 0)");
  UM_REQUIRE(kv_shift >= 0 && kv_shift < n_streams, "um_window_attention_planes: kv_shift out of range");
  UM_REQUIRE(!out || (ldo % 4 == 0 && ldo >= UM_C), "um_window_attention_planes: ldo must be >= 128 and a multiple of 4");
  UM_REQUIRE(!out_split || (split_plane_stride >= (int64_t)n_streams * g.h * g.w * UM_C && split_plane_stride % 8 == 0),
             "um_window_attention_planes: split_plane_stride must cover n_streams*h*w rows of 128 halves");
  UM_REQUIRE(((reinterpret_cast<uintptr_t>(q_planes) | reinterpret_cast<uintptr_t>(k_planes) |
               reinterpret_cast<uintptr_t>(v_planes) | reinterpret_cast<uintptr_t>(out_split)) & 15) == 0,
             "um_window_attention_planes: planes must be 16-byte aligned");
  return um::attention_planes_launch(reinterpret_cast<const __half*>(q_planes), reinterpret_cast<const __half*>(k_planes),
                                     reinterpret_cast<const __half*>(v_planes), out, ldo, reinterpret_cast<__half*>(out_split),
                                     split_plane_stride, n_streams, kv_shift, g, (cudaStream_t)stream);
}

int um_window_attention(const float* q, const float* k, const float* v, float* out, int32_t n_streams,
                        int32_t kv_shift, int64_t ldq, int64_t ldk, int64_t ldv, int64_t ldo,
                        const um_attn_geom* geom, void* workspace, int64_t workspace_bytes, int32_t flags,
                        void* stream) {
  um::Geom g;
  UM_REQUIRE(q && k && v && out && n_streams > 0, "um_window_attention: null pointer or empty batch");
  UM_REQUIRE(um::make_geom(geom, &g), "um_window_attention: bad geometry (h,w must be divisible by kh,kw)");
  UM_REQUIRE(kv_shift >= 0 && kv_shift < n_streams, "um_window_attention: kv_shift out of range");
  UM_REQUIRE(ldq % 4 == 0 && ldk % 4 == 0 && ldv % 4 == 0 && ldo % 4 == 0 && ldq >= UM_C && ldk >= UM_C &&
                 ldv >= UM_C && ldo >= UM_C,
             "um_window_attention: row strides must be >= 128 and multiples of 4 floats");
  UM_REQUIRE(g.mask_mode >= UM_MASK_NONE && g.mask_mode <= UM_MASK_CAUSAL, "um_window_attention: bad mask_mode");
  cudaStream_t st = (cudaStream_t)stream;
  if (!(flags & UM_ATTN_FORCE_CUDA_CORES) && um::attention_tc_supported(g)) {
    UM_REQUIRE(workspace && workspace_bytes >= (int64_t)um::attention_tc_workspace_bytes(g, n_streams),
               "um_window_attention: workspace too small (%lld bytes needed, see um_window_attention_workspace)",
               (long long)um::attention_tc_workspace_bytes(g, n_streams));
    return um::window_attention_tc(q, k, v, out, n_streams, kv_shift, ldq, ldk, ldv, ldo, g, workspace, st);
  }
  return um::window_attention_simt(q, k, v, out, n_streams, kv_shift, ldq, ldk, ldv, ldo, g, st);
}

int64_t um_softmax_expectation_workspace(const um_attn_geom* geom, int32_t n_total, int32_t value_mode) {
  um::Geom g;
  if (!um::make_geom(geom, &g) || n_total <= 0 || !um::expectation_tc_supported(g, value_mode)) return 0;
  return (int64_t)um::expectation_tc_workspace_bytes(g, n_total);
}

int um_softmax_expectation(const float* q, const float* k, const float* values, float* out, int32_t n_streams,
                           int32_t n_total, int32_t kv_shift, int64_t ldq, int64_t ldk, int32_t vdim,
                           int32_t value_mode, int32_t post_op, const um_attn_geom* geom, void* workspace,
                           int64_t workspace_bytes, int32_t flags, void* stream) {
  um::Geom g;
  UM_REQUIRE(q && k && out && n_streams > 0 && n_total >= n_streams, "um_softmax_expectation: bad batch arguments");
  UM_REQUIRE(um::make_geom(geom, &g), "um_softmax_expectation: bad geometry");
  UM_REQUIRE(kv_shift >= 0 && kv_shift < n_total, "um_softmax_expectation: kv_shift out of range");
  UM_REQUIRE(ldq % 4 == 0 && ldk % 4 == 0 && ldq >= UM_C && ldk >= UM_C, "um_softmax_expectation: bad row strides");
  UM_REQUIRE(vdim == 1 || vdim == 2, "um_softmax_expectation: vdim must be 1 or 2");
  UM_REQUIRE(value_mode >= UM_VALUE_TENSOR && value_mode <= UM_VALUE_XCOORD, "um_softmax_expectation: bad value_mode");
  UM_REQUIRE(value_mode != UM_VALUE_TENSOR || values, "um_softmax_expectation: values is NULL");
  UM_REQUIRE(value_mode != UM_VALUE_COORDS || vdim == 2, "um_softmax_expectation: COORDS needs vdim 2");
  UM_REQUIRE(value_mode != UM_VALUE_XCOORD || vdim == 1, "um_softmax_expectation: XCOORD needs vdim 1");
  UM_REQUIRE(post_op >= UM_POST_NONE && post_op <= UM_POST_OWN_MINUS, "um_softmax_expectation: bad post_op");
  if (!(flags & UM_ATTN_FORCE_CUDA_CORES) && um::expectation_tc_supported(g, value_mode)) {
    UM_REQUIRE(workspace && workspace_bytes >= (int64_t)um::expectation_tc_workspace_bytes(g, n_total),
               "um_softmax_expectation: workspace too small (%lld bytes needed, see um_softmax_expectation_workspace)",
               (long long)um::expectation_tc_workspace_bytes(g, n_total));
    return um::softmax_expectation_tc(q, k, values, out, n_streams, n_total, kv_shift, ldq, ldk, vdim, value_mode, post_op,
                                      g, workspace, (cudaStream_t)stream);
  }
  return um::softmax_expectation_simt(q, k, values, out, n_streams, n_total, kv_shift, ldq, ldk, vdim, value_mode,
                                      post_op, g, (cudaStream_t)stream);
}

int um_chain_tracks(const float* flow, const float* occ, int32_t n, int32_t h, int32_t w, float* pos, uint8_t* vis,
                    float* pos_out, uint8_t* vis_out, void* stream) {
  UM_REQUIRE(flow && pos && vis && pos_out && vis_out, "um_chain_tracks: flow, state and outputs must not be NULL");
  UM_REQUIRE(n > 0 && h > 1 && w > 1, "um_chain_tracks: bad shape (n >= 1 flows of at least 2 x 2)");
  UM_REQUIRE((long long)h * w <= 0x7fffffffLL, "um_chain_tracks: a frame has at most 2^31 - 1 pixels");
  UM_REQUIRE(((reinterpret_cast<uintptr_t>(pos) | reinterpret_cast<uintptr_t>(pos_out)) & 7) == 0,
             "um_chain_tracks: pos and pos_out must be 8-byte aligned");
  const long long hw = (long long)h * w, p1 = 8 * hw, v1 = hw, pn = 8 * n * hw, vn = n * hw;
  UM_REQUIRE(!um::overlap(pos, p1, vis, v1) && !um::overlap(pos, p1, pos_out, pn) && !um::overlap(pos, p1, vis_out, vn) &&
                 !um::overlap(vis, v1, pos_out, pn) && !um::overlap(vis, v1, vis_out, vn) &&
                 !um::overlap(pos_out, pn, vis_out, vn),
             "um_chain_tracks: the state and output buffers must not overlap");
  return um::chain_tracks_launch(flow, occ, n, h, w, pos, vis, pos_out, vis_out, (cudaStream_t)stream);
}

int um_track_points_forward(const float* flow, const float* occ, int32_t n, int32_t h, int32_t w, int32_t t0,
                            const float* queries, int32_t nq, int32_t nt, float* pos, uint8_t* vis, float* tracks,
                            uint8_t* visible, void* stream) {
  UM_REQUIRE(flow && queries && pos && vis && tracks && visible,
             "um_track_points_forward: flow, queries, state and tables must not be NULL");
  UM_REQUIRE(n > 0 && h > 1 && w > 1 && nq > 0, "um_track_points_forward: bad shape (n >= 1 flows of at least 2 x 2, "
             "nq >= 1 queries)");
  UM_REQUIRE((long long)h * w <= 0x7fffffffLL, "um_track_points_forward: a frame has at most 2^31 - 1 pixels");
  UM_REQUIRE(t0 >= 0 && (long long)t0 + n < nt, "um_track_points_forward: frames t0 .. t0+n must lie inside the table "
             "(t0 = %d, n = %d, nt = %d)", t0, n, nt);
  UM_REQUIRE(um::aligned(flow, 4) && um::aligned(occ, 4) && um::aligned(queries, 4) && um::aligned(pos, 8) &&
                 um::aligned(tracks, 8),
             "um_track_points_forward: flow, occ and queries must be 4-byte aligned, pos and tracks 8-byte aligned");
  const long long hw = (long long)h * w, tab = (long long)nq * nt;
  UM_REQUIRE(um::written_disjoint({{pos, 8LL * nq}, {vis, nq}, {tracks, 8 * tab}, {visible, tab}, {queries, 12LL * nq},
                                   {flow, 8LL * n * hw}, {occ, 4LL * n * hw}}, 4),
             "um_track_points_forward: the state and tables must not overlap each other or the inputs");
  return um::track_points_forward_launch(flow, occ, n, h, w, t0, queries, nq, nt, pos, vis, tracks, visible,
                                         (cudaStream_t)stream);
}

int um_track_points_backward(const float* flow, const float* occ, int32_t n, int32_t h, int32_t w, const float* queries,
                             int32_t nq, int32_t nt, float* tracks, uint8_t* visible, void* stream) {
  UM_REQUIRE(queries && tracks && visible && (flow || n == 0),
             "um_track_points_backward: queries, tables and (n > 0) flow must not be NULL");
  UM_REQUIRE(n >= 0 && h > 1 && w > 1 && nq > 0, "um_track_points_backward: bad shape (n >= 0 flows of at least 2 x 2, "
             "nq >= 1 queries)");
  UM_REQUIRE((long long)h * w <= 0x7fffffffLL, "um_track_points_backward: a frame has at most 2^31 - 1 pixels");
  UM_REQUIRE(nt >= 2 && n < nt, "um_track_points_backward: the n stored pairs must lie inside a table of nt >= 2 frames "
             "(n = %d, nt = %d)", n, nt);
  UM_REQUIRE(um::aligned(flow, 4) && um::aligned(occ, 4) && um::aligned(queries, 4) && um::aligned(tracks, 8),
             "um_track_points_backward: flow, occ and queries must be 4-byte aligned, tracks 8-byte aligned");
  const long long hw = (long long)h * w, tab = (long long)nq * nt;
  UM_REQUIRE(um::written_disjoint({{tracks, 8 * tab}, {visible, tab}, {queries, 12LL * nq}, {flow, 8LL * n * hw},
                                   {occ, 4LL * n * hw}}, 2),
             "um_track_points_backward: the tables must not overlap each other or the inputs");
  return um::track_points_backward_launch(n > 0 ? flow : nullptr, n > 0 ? occ : nullptr, n, h, w, queries, nq, nt, tracks,
                                          visible, (cudaStream_t)stream);
}

int um_multi_flow_tracks(const float* flow, const float* occ, const float* err, const int32_t* src, const int32_t* dst,
                         int32_t n, int32_t k, int32_t h, int32_t w, int32_t r, float* pos, float* sig, uint8_t* vis,
                         float* tracks, uint8_t* visible, float* sigma, void* stream) {
  UM_REQUIRE(flow && occ && err && src && dst && pos && sig && vis && tracks && visible && sigma,
             "um_multi_flow_tracks: flows, masks, residuals, tables, state and outputs must not be NULL");
  UM_REQUIRE(n > 0 && k > 0 && r > 0 && h > 1 && w > 1,
             "um_multi_flow_tracks: bad shape (n >= 1 frames of k >= 1 candidates, r >= 1 slots, frames of at least 2 x 2)");
  UM_REQUIRE((long long)h * w <= 0x7fffffffLL && (long long)n * k <= 0x7fffffffLL,
             "um_multi_flow_tracks: a frame has at most 2^31 - 1 pixels, a launch at most 2^31 - 1 candidates");
  UM_REQUIRE(um::aligned(flow, 4) && um::aligned(occ, 4) && um::aligned(err, 4) && um::aligned(src, 4) &&
                 um::aligned(dst, 4) && um::aligned(pos, 8) && um::aligned(sig, 4) && um::aligned(tracks, 8) &&
                 um::aligned(sigma, 4),
             "um_multi_flow_tracks: pos and tracks must be 8-byte aligned, the other float and int32 buffers 4-byte aligned");
  const long long hw = (long long)h * w, c = (long long)n * k * hw;
  UM_REQUIRE(um::written_disjoint({{pos, 8 * r * hw}, {sig, 4 * r * hw}, {vis, r * hw}, {tracks, 8 * n * hw},
                                   {visible, n * hw}, {sigma, 4 * n * hw}, {flow, 8 * c}, {occ, 4 * c}, {err, 4 * c},
                                   {src, 4LL * n * k}, {dst, 4LL * n}}, 6),
             "um_multi_flow_tracks: the state and outputs must not overlap each other or the inputs");
  return um::multi_flow_tracks_launch(flow, occ, err, src, dst, n, k, h, w, r, pos, sig, vis, tracks, visible, sigma,
                                      (cudaStream_t)stream);
}

int um_warp_disparity(const float* disp_next, const float* flow, float* disp1, uint8_t* in_frame, int32_t batch, int32_t h,
                      int32_t w, void* stream) {
  UM_REQUIRE(disp_next && flow && disp1 && in_frame, "um_warp_disparity: disp_next, flow, disp1 and in_frame must not be NULL");
  UM_REQUIRE(batch > 0 && batch <= 65535 && h > 0 && w > 0, "um_warp_disparity: bad shape (batch %d, %d x %d)", batch, h, w);
  UM_REQUIRE((long long)h * w <= 0x7fffffffLL && (long long)batch * h * w <= 0x7fffffffLL * 256,
             "um_warp_disparity: a frame has at most 2^31 - 1 pixels, a batch at most 2^39 - 256");
  UM_REQUIRE(um::aligned(disp_next, 4) && um::aligned(flow, 4) && um::aligned(disp1, 4),
             "um_warp_disparity: disp_next, flow and disp1 must be 4-byte aligned");
  const long long n = (long long)batch * h * w;
  UM_REQUIRE(um::written_disjoint({{disp1, 4 * n}, {in_frame, n}, {disp_next, 4 * n}, {flow, 8 * n}}, 2),
             "um_warp_disparity: disp1 and in_frame must not overlap each other or the inputs");
  return um::warp_disparity_launch(disp_next, flow, disp1, in_frame, batch, h, w, (cudaStream_t)stream);
}

}  // extern "C"
