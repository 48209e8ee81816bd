// C-ABI glue: error reporting, launch accounting, the attention entry points (argument checking + dispatch
// between the tensor-core and the general CUDA-core kernels) the point-track entries and the disparity warp (um_tracks.cu),
// TSDF fusion (um_fusion.cu), ICP tracking against the volume (um_icp.cu), the point-cloud ops (um_cloud.cu) and the mesh
// rasteriser, point visibility and depth metrics (um_raster.cu) and the multi-view consistency of depth maps and their
// export as points (um_consistency.cu).  See include/unimatch_sm100.h.
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
int tsdf_integrate_launch(float* tsdf, float* weight, float* color, int X, int Y, int Z, const float* origin,
                          float voxel_size, float trunc, const float* depth, const uint8_t* frames, const float* w2c, int n,
                          int h, int w, float fx, float fy, float cx, float cy, const int* n_valid, cudaStream_t st);
int tsdf_surface_count_launch(const float* tsdf, const float* weight, int X, int Y, int Z, long long* offsets,
                              cudaStream_t st);
int tsdf_surface_points_launch(const float* tsdf, const float* weight, const float* color, int X, int Y, int Z,
                               const float* origin, float voxel_size, const long long* offsets, float* points,
                               uint8_t* colors, cudaStream_t st);
int tsdf_mesh_count_launch(const float* tsdf, const float* weight, int X, int Y, int Z, long long* offsets, cudaStream_t st);
int tsdf_mesh_launch(const float* tsdf, const float* weight, const float* color, int X, int Y, int Z, const float* origin,
                     float voxel_size, const long long* point_offsets, const long long* face_offsets, long long n_faces,
                     int* first_vertex, float* points, uint8_t* colors, float* normals, int* faces, cudaStream_t st);
int tsdf_raycast_launch(const float* tsdf, const float* weight, const float* color, int X, int Y, int Z, const float* origin,
                        float voxel_size, float trunc, const float* c2w, int n, int h, int w, float fx, float fy, float cx,
                        float cy, float near, float far, float* depth, uint8_t* rgb, float* normal, cudaStream_t st);
int icp_downsample_launch(const float* src, float* dst, int n, int h, int w, float trunc, cudaStream_t st);
int icp_normals_launch(const float* depth, float* normal, int n, int h, int w, float fx, float fy, float cx, float cy,
                       cudaStream_t st);
int icp_init_launch(const double* poses, const double* correction, int n, const int* n_valid, double* state, float* c2w,
                    float* w2c, cudaStream_t st);
int icp_reduce_launch(const float* depth, const float* live_normal, const float* model_depth, const float* model_normal,
                      const double* state, const float* c2w, const float* w2c, int n, int h, int w, float fx, float fy,
                      float cx, float cy, float max_distance, float cos_max_angle, const int* n_valid, double* partials,
                      cudaStream_t st);
int icp_solve_launch(const double* partials, int nb, int n, const int* n_valid, double min_inliers, double min_pivot,
                     int record, double* state, cudaStream_t st);
int icp_accept_launch(const double* partials, int nb, int n, const int* n_valid, double min_inlier_fraction,
                      const double* poses, double* correction, double* state, float* pose_out, uint8_t* tracked,
                      int64_t* inliers, float* rmse, float* w2c, cudaStream_t st);
int cloud_keys_launch(const float* points, long long n, const double* origin, double cell, const int* dims,
                      long long* keys, cudaStream_t st);
int cloud_ranges_launch(const long long* keys, const long long* order, const float* points, long long n, long long n_cells,
                        int* start, int* end, float* sorted, cudaStream_t st);
int cloud_down_sample_count_launch(const long long* keys, long long n, long long* offsets, cudaStream_t st);
int cloud_down_sample_launch(const long long* keys, const long long* order, const float* points, long long n,
                             const long long* offsets, float* out, cudaStream_t st);
int cloud_nearest_launch(const float* queries, long long nq, const float* sorted, const int* start, const int* end,
                         const double* origin, double cell, const int* dims, float threshold, float* distance,
                         long long* index, double* partial_sum, long long* partial_count, cudaStream_t st);
int cloud_stats_launch(const double* partial_sum, const long long* partial_count, long long nb, double* out,
                       cudaStream_t st);
int mesh_bin_count_launch(const float* points, const int* faces, long long T, const float* w2c, int n, int h, int w,
                          float fx, float fy, float cx, float cy, float near, float far, long long* offsets,
                          cudaStream_t st);
int mesh_bin_launch(const float* points, const int* faces, long long T, const float* w2c, int n, int h, int w, float fx,
                    float fy, float cx, float cy, float near, float far, const long long* offsets, long long* keys,
                    long long* values, cudaStream_t st);
int mesh_ranges_launch(const long long* sorted_keys, long long total, long long n_bins, int* start, int* end,
                       cudaStream_t st);
int mesh_raster_launch(const float* points, const int* faces, const uint8_t* colors, const float* w2c, int n, int h,
                       int w, float fx, float fy, float cx, float cy, float near, float far, const long long* order,
                       const long long* values, const int* start, const int* end, float* depth, int* face,
                       uint8_t* rgb, cudaStream_t st);
int visible_points_launch(const float* points, long long P, const float* depth, int n, int h, int w, const float* w2c,
                          float fx, float fy, float cx, float cy, float tolerance, uint8_t* visible, cudaStream_t st);
int depth_metrics_launch(const float* pred, const float* gt, int n, int h, int w, float max_depth, double* partials,
                         double* out, cudaStream_t st);
int depth_consistency_launch(const float* depth, int N, int H, int W, float fx, float fy, float cx, float cy,
                             const float* c2w, const float* w2c, const int* refs, int R, const int* src, int S,
                             float max_pixel, float max_relative, int min_views, uint8_t* views, float* out,
                             cudaStream_t st);
int depth_points_count_launch(const float* depth, long long total, long long* offsets, cudaStream_t st);
int depth_points_launch(const float* depth, const uint8_t* frames, int N, int H, int W, float fx, float fy, float cx,
                        float cy, const float* c2w, const long long* offsets, float* points, uint8_t* colors,
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

// A TSDF volume of X x Y x Z voxels: every dimension positive, at most 2^31 - 1 voxels in all.
static bool tsdf_dims(int32_t X, int32_t Y, int32_t Z) {
  return X > 0 && Y > 0 && Z > 0 && (long long)X * Y * Z <= 0x7fffffffLL;
}

static bool positive_finite(float v) { return v > 0.f && v <= 3.402823466e38f; }
static bool finite_value(float v) { return v >= -3.402823466e38f && v <= 3.402823466e38f; }

int um_tsdf_integrate(float* tsdf, float* weight, float* color, int32_t X, int32_t Y, int32_t Z, const float* origin,
                      float voxel_size, float trunc, const float* depth, const uint8_t* frames, const float* w2c, int32_t n,
                      int32_t h, int32_t w, float fx, float fy, float cx, float cy, const int32_t* n_valid, void* stream) {
  UM_REQUIRE(tsdf && weight && color && origin && depth && frames && w2c && n_valid,
             "um_tsdf_integrate: no pointer may be NULL");
  UM_REQUIRE(tsdf_dims(X, Y, Z), "um_tsdf_integrate: bad volume %d x %d x %d (at most 2^31 - 1 voxels)", X, Y, Z);
  UM_REQUIRE(positive_finite(voxel_size) && positive_finite(trunc),
             "um_tsdf_integrate: voxel_size and trunc must be positive and finite");
  UM_REQUIRE(n > 0 && h > 0 && w > 0 && (long long)h * w <= 0x7fffffffLL, "um_tsdf_integrate: bad frames (%d x %d x %d)",
             n, h, w);
  UM_REQUIRE(um::aligned(tsdf, 4) && um::aligned(weight, 4) && um::aligned(color, 4) && um::aligned(depth, 4) &&
                 um::aligned(w2c, 4) && um::aligned(n_valid, 4),
             "um_tsdf_integrate: the fp32 and int32 buffers must be 4-byte aligned");
  const long long nv = (long long)X * Y * Z, px = (long long)n * h * w;
  UM_REQUIRE(um::written_disjoint({{tsdf, 4 * nv}, {weight, 4 * nv}, {color, 12 * nv}, {depth, 4 * px}, {frames, 3 * px},
                                   {w2c, 48LL * n}, {n_valid, 4}},
                                  3),
             "um_tsdf_integrate: the volume planes must not overlap each other or the inputs");
  return um::tsdf_integrate_launch(tsdf, weight, color, X, Y, Z, origin, voxel_size, trunc, depth, frames, w2c, n, h, w, fx,
                                   fy, cx, cy, n_valid, (cudaStream_t)stream);
}

int um_tsdf_surface_count(const float* tsdf, const float* weight, int32_t X, int32_t Y, int32_t Z, int64_t* offsets,
                          void* stream) {
  UM_REQUIRE(tsdf && weight && offsets, "um_tsdf_surface_count: no pointer may be NULL");
  UM_REQUIRE(tsdf_dims(X, Y, Z), "um_tsdf_surface_count: bad volume %d x %d x %d (at most 2^31 - 1 voxels)", X, Y, Z);
  UM_REQUIRE(um::aligned(tsdf, 4) && um::aligned(weight, 4) && um::aligned(offsets, 8),
             "um_tsdf_surface_count: tsdf and weight must be 4-byte aligned, offsets 8-byte aligned");
  const long long nv = (long long)X * Y * Z, nb = (nv + UM_TSDF_THREADS - 1) / UM_TSDF_THREADS;
  UM_REQUIRE(um::written_disjoint({{offsets, 8 * (nb + 1)}, {tsdf, 4 * nv}, {weight, 4 * nv}}, 1),
             "um_tsdf_surface_count: offsets must not overlap the volume");
  return um::tsdf_surface_count_launch(tsdf, weight, X, Y, Z, reinterpret_cast<long long*>(offsets), (cudaStream_t)stream);
}

int um_tsdf_surface_points(const float* tsdf, const float* weight, const float* color, int32_t X, int32_t Y, int32_t Z,
                           const float* origin, float voxel_size, const int64_t* offsets, int64_t n_points, float* points,
                           uint8_t* colors, void* stream) {
  UM_REQUIRE(tsdf && weight && color && origin && offsets, "um_tsdf_surface_points: no input may be NULL");
  UM_REQUIRE(n_points == 0 || (points && colors), "um_tsdf_surface_points: points and colors must not be NULL");
  UM_REQUIRE(tsdf_dims(X, Y, Z), "um_tsdf_surface_points: bad volume %d x %d x %d (at most 2^31 - 1 voxels)", X, Y, Z);
  UM_REQUIRE(positive_finite(voxel_size), "um_tsdf_surface_points: voxel_size must be positive and finite");
  const long long nv = (long long)X * Y * Z, nb = (nv + UM_TSDF_THREADS - 1) / UM_TSDF_THREADS;
  UM_REQUIRE(n_points >= 0 && n_points <= 3 * nv, "um_tsdf_surface_points: bad point count %lld", (long long)n_points);
  UM_REQUIRE(um::aligned(tsdf, 4) && um::aligned(weight, 4) && um::aligned(color, 4) && um::aligned(offsets, 8) &&
                 um::aligned(points, 4),
             "um_tsdf_surface_points: tsdf, weight, color and points must be 4-byte aligned, offsets 8-byte aligned");
  UM_REQUIRE(um::written_disjoint({{points, 12 * n_points}, {colors, 3 * n_points}, {tsdf, 4 * nv}, {weight, 4 * nv},
                                   {color, 12 * nv}, {offsets, 8 * (nb + 1)}},
                                  2),
             "um_tsdf_surface_points: points and colors must not overlap each other, the volume or the offsets");
  if (n_points == 0) return UM_OK;
  return um::tsdf_surface_points_launch(tsdf, weight, color, X, Y, Z, origin, voxel_size,
                                        reinterpret_cast<const long long*>(offsets), points, colors, (cudaStream_t)stream);
}

int um_tsdf_mesh_count(const float* tsdf, const float* weight, int32_t X, int32_t Y, int32_t Z, int64_t* face_offsets,
                       void* stream) {
  UM_REQUIRE(tsdf && weight && face_offsets, "um_tsdf_mesh_count: no pointer may be NULL");
  UM_REQUIRE(tsdf_dims(X, Y, Z), "um_tsdf_mesh_count: bad volume %d x %d x %d (at most 2^31 - 1 voxels)", X, Y, Z);
  UM_REQUIRE(um::aligned(tsdf, 4) && um::aligned(weight, 4) && um::aligned(face_offsets, 8),
             "um_tsdf_mesh_count: tsdf and weight must be 4-byte aligned, face_offsets 8-byte aligned");
  const long long nv = (long long)X * Y * Z, nb = (nv + UM_TSDF_THREADS - 1) / UM_TSDF_THREADS;
  UM_REQUIRE(um::written_disjoint({{face_offsets, 8 * (nb + 1)}, {tsdf, 4 * nv}, {weight, 4 * nv}}, 1),
             "um_tsdf_mesh_count: face_offsets must not overlap the volume");
  return um::tsdf_mesh_count_launch(tsdf, weight, X, Y, Z, reinterpret_cast<long long*>(face_offsets),
                                    (cudaStream_t)stream);
}

int um_tsdf_mesh(const float* tsdf, const float* weight, const float* color, int32_t X, int32_t Y, int32_t Z,
                 const float* origin, float voxel_size, const int64_t* point_offsets, int64_t n_points,
                 const int64_t* face_offsets, int64_t n_faces, int32_t* first_vertex, float* points, uint8_t* colors,
                 float* normals, int32_t* faces, void* stream) {
  UM_REQUIRE(tsdf && weight && color && origin && point_offsets && face_offsets, "um_tsdf_mesh: no input may be NULL");
  UM_REQUIRE(n_points == 0 || (first_vertex && points && colors && normals),
             "um_tsdf_mesh: first_vertex, points, colors and normals must not be NULL");
  UM_REQUIRE(n_faces == 0 || faces, "um_tsdf_mesh: faces must not be NULL");
  UM_REQUIRE(tsdf_dims(X, Y, Z), "um_tsdf_mesh: bad volume %d x %d x %d (at most 2^31 - 1 voxels)", X, Y, Z);
  UM_REQUIRE(positive_finite(voxel_size), "um_tsdf_mesh: voxel_size must be positive and finite");
  const long long nv = (long long)X * Y * Z, nb = (nv + UM_TSDF_THREADS - 1) / UM_TSDF_THREADS;
  UM_REQUIRE(n_points >= 0 && n_points <= 3 * nv && n_points <= 0x7fffffffLL, "um_tsdf_mesh: bad point count %lld",
             (long long)n_points);
  UM_REQUIRE(n_faces >= 0 && n_faces <= 5 * nv && n_faces <= 0x7fffffffLL && (n_faces == 0 || n_points >= 3),
             "um_tsdf_mesh: bad face count %lld (with %lld points)", (long long)n_faces, (long long)n_points);
  UM_REQUIRE(um::aligned(tsdf, 4) && um::aligned(weight, 4) && um::aligned(color, 4) && um::aligned(point_offsets, 8) &&
                 um::aligned(face_offsets, 8) && um::aligned(first_vertex, 4) && um::aligned(points, 4) &&
                 um::aligned(normals, 4) && um::aligned(faces, 4),
             "um_tsdf_mesh: the fp32 and int32 buffers must be 4-byte aligned, the offsets 8-byte aligned");
  const long long P = n_points, T = n_faces;
  UM_REQUIRE(um::written_disjoint({{points, 12 * P}, {colors, 3 * P}, {normals, 12 * P}, {first_vertex, P ? 4 * nv : 0},
                                   {faces, 12 * T}, {tsdf, 4 * nv}, {weight, 4 * nv}, {color, 12 * nv},
                                   {point_offsets, 8 * (nb + 1)}, {face_offsets, 8 * (nb + 1)}},
                                  5),
             "um_tsdf_mesh: the outputs and first_vertex must not overlap each other, the volume or the offsets");
  if (n_points == 0) return UM_OK;
  return um::tsdf_mesh_launch(tsdf, weight, color, X, Y, Z, origin, voxel_size,
                              reinterpret_cast<const long long*>(point_offsets),
                              reinterpret_cast<const long long*>(face_offsets), n_faces, first_vertex, points, colors,
                              normals, faces, (cudaStream_t)stream);
}

int um_tsdf_raycast(const float* tsdf, const float* weight, const float* color, int32_t X, int32_t Y, int32_t Z,
                    const float* origin, float voxel_size, float trunc, const float* c2w, int32_t n, int32_t h, int32_t w,
                    float fx, float fy, float cx, float cy, float near, float far, float* depth, uint8_t* rgb,
                    float* normal, void* stream) {
  UM_REQUIRE(tsdf && weight && color && origin && c2w && depth && rgb && normal, "um_tsdf_raycast: no pointer may be NULL");
  UM_REQUIRE(tsdf_dims(X, Y, Z), "um_tsdf_raycast: bad volume %d x %d x %d (at most 2^31 - 1 voxels)", X, Y, Z);
  UM_REQUIRE(positive_finite(voxel_size) && positive_finite(trunc),
             "um_tsdf_raycast: voxel_size and trunc must be positive and finite");
  UM_REQUIRE(n > 0 && n <= 65535 && h > 0 && w > 0 && (long long)h * w <= 0x7fffffffLL,
             "um_tsdf_raycast: bad views (%d x %d x %d; at most 65535 views of 2^31 - 1 pixels)", n, h, w);
  UM_REQUIRE(fx != 0.f && fy != 0.f && finite_value(fx) && finite_value(fy) && finite_value(cx) && finite_value(cy),
             "um_tsdf_raycast: fx and fy must be finite and nonzero, cx and cy finite");
  UM_REQUIRE(near >= 0.f && finite_value(near) && far > near,
             "um_tsdf_raycast: near must be finite and >= 0, far > near (+inf for no limit)");
  UM_REQUIRE(um::aligned(tsdf, 4) && um::aligned(weight, 4) && um::aligned(color, 4) && um::aligned(c2w, 4) &&
                 um::aligned(depth, 4) && um::aligned(normal, 4),
             "um_tsdf_raycast: the fp32 buffers must be 4-byte aligned");
  const long long nv = (long long)X * Y * Z, px = (long long)n * h * w;
  UM_REQUIRE(um::written_disjoint({{depth, 4 * px}, {rgb, 3 * px}, {normal, 12 * px}, {tsdf, 4 * nv}, {weight, 4 * nv},
                                   {color, 12 * nv}, {c2w, 48LL * n}},
                                  3),
             "um_tsdf_raycast: depth, rgb and normal must not overlap each other, the volume or c2w");
  return um::tsdf_raycast_launch(tsdf, weight, color, X, Y, Z, origin, voxel_size, trunc, c2w, n, h, w, fx, fy, cx, cy,
                                 near, far, depth, rgb, normal, (cudaStream_t)stream);
}


// ---- ICP tracking against the volume (um_icp.cu) ----
static bool icp_frames(int32_t n, int32_t h, int32_t w) {
  return n > 0 && n <= 65535 && h > 0 && w > 0 && (long long)h * w <= 0x7fffffffLL;
}

static bool icp_intrinsics(float fx, float fy, float cx, float cy) {
  return fx != 0.f && fy != 0.f && finite_value(fx) && finite_value(fy) && finite_value(cx) && finite_value(cy);
}

int um_icp_downsample(const float* src, float* dst, int32_t n, int32_t h, int32_t w, float trunc, void* stream) {
  UM_REQUIRE(src && dst, "um_icp_downsample: no pointer may be NULL");
  UM_REQUIRE(icp_frames(n, h, w) && h >= 2 && w >= 2,
             "um_icp_downsample: bad depths (%d x %d x %d; at most 65535 maps of 2 x 2 to 2^31 - 1 pixels)", n, h, w);
  UM_REQUIRE(positive_finite(trunc), "um_icp_downsample: trunc must be positive and finite");
  UM_REQUIRE(um::aligned(src, 4) && um::aligned(dst, 4), "um_icp_downsample: src and dst must be 4-byte aligned");
  const long long px = (long long)n * h * w, px2 = (long long)n * (h / 2) * (w / 2);
  UM_REQUIRE(um::written_disjoint({{dst, 4 * px2}, {src, 4 * px}}, 1), "um_icp_downsample: dst must not overlap src");
  return um::icp_downsample_launch(src, dst, n, h, w, trunc, (cudaStream_t)stream);
}

int um_icp_normals(const float* depth, float* normal, int32_t n, int32_t h, int32_t w, float fx, float fy, float cx,
                   float cy, void* stream) {
  UM_REQUIRE(depth && normal, "um_icp_normals: no pointer may be NULL");
  UM_REQUIRE(icp_frames(n, h, w), "um_icp_normals: bad depths (%d x %d x %d; at most 65535 maps of 2^31 - 1 pixels)", n,
             h, w);
  UM_REQUIRE(icp_intrinsics(fx, fy, cx, cy), "um_icp_normals: fx and fy must be finite and nonzero, cx and cy finite");
  UM_REQUIRE(um::aligned(depth, 4) && um::aligned(normal, 4), "um_icp_normals: depth and normal must be 4-byte aligned");
  const long long px = (long long)n * h * w;
  UM_REQUIRE(um::written_disjoint({{normal, 12 * px}, {depth, 4 * px}}, 1), "um_icp_normals: normal must not overlap depth");
  return um::icp_normals_launch(depth, normal, n, h, w, fx, fy, cx, cy, (cudaStream_t)stream);
}

int um_icp_init(const double* poses, const double* correction, int32_t n, const int32_t* n_valid, double* state,
                float* c2w, float* w2c, void* stream) {
  UM_REQUIRE(poses && n_valid && state && c2w && w2c, "um_icp_init: no pointer but correction may be NULL");
  UM_REQUIRE(n > 0 && n <= 65535, "um_icp_init: bad frame count %d (1 .. 65535)", n);
  UM_REQUIRE(um::aligned(poses, 8) && um::aligned(correction, 8) && um::aligned(state, 8) && um::aligned(n_valid, 4) &&
                 um::aligned(c2w, 4) && um::aligned(w2c, 4),
             "um_icp_init: the fp64 buffers must be 8-byte aligned, the fp32 and int32 buffers 4-byte aligned");
  UM_REQUIRE(um::written_disjoint({{state, 8LL * UM_ICP_STATE * n}, {c2w, 48LL * n}, {w2c, 48LL * n}, {poses, 128LL * n},
                                   {correction, 128}, {n_valid, 4}},
                                  3),
             "um_icp_init: state, c2w and w2c must not overlap each other or the inputs");
  return um::icp_init_launch(poses, correction, n, n_valid, state, c2w, w2c, (cudaStream_t)stream);
}

int um_icp_reduce(const float* depth, const float* live_normal, const float* model_depth, const float* model_normal,
                  const double* state, const float* c2w, const float* w2c, int32_t n, int32_t h, int32_t w, float fx,
                  float fy, float cx, float cy, float max_distance, float cos_max_angle, const int32_t* n_valid,
                  double* partials, void* stream) {
  UM_REQUIRE(depth && live_normal && model_depth && model_normal && state && c2w && w2c && n_valid && partials,
             "um_icp_reduce: no pointer may be NULL");
  UM_REQUIRE(icp_frames(n, h, w), "um_icp_reduce: bad frames (%d x %d x %d; at most 65535 frames of 2^31 - 1 pixels)", n,
             h, w);
  UM_REQUIRE(icp_intrinsics(fx, fy, cx, cy), "um_icp_reduce: fx and fy must be finite and nonzero, cx and cy finite");
  UM_REQUIRE(positive_finite(max_distance) && finite_value(cos_max_angle) && cos_max_angle >= -1.f && cos_max_angle <= 1.f,
             "um_icp_reduce: max_distance must be positive and finite, cos_max_angle in [-1, 1]");
  UM_REQUIRE(um::aligned(depth, 4) && um::aligned(live_normal, 4) && um::aligned(model_depth, 4) &&
                 um::aligned(model_normal, 4) && um::aligned(state, 8) && um::aligned(c2w, 4) && um::aligned(w2c, 4) &&
                 um::aligned(n_valid, 4) && um::aligned(partials, 8),
             "um_icp_reduce: the fp64 buffers must be 8-byte aligned, the fp32 and int32 buffers 4-byte aligned");
  const long long px = (long long)n * h * w, nb = (long long)((w + 15) / 16) * ((h + 7) / 8);
  UM_REQUIRE(um::written_disjoint({{partials, 8LL * UM_ICP_TERMS * nb * n}, {depth, 4 * px}, {live_normal, 12 * px},
                                   {model_depth, 4 * px}, {model_normal, 12 * px}, {state, 8LL * UM_ICP_STATE * n},
                                   {c2w, 48LL * n}, {w2c, 48LL * n}, {n_valid, 4}},
                                  1),
             "um_icp_reduce: partials must not overlap the inputs");
  return um::icp_reduce_launch(depth, live_normal, model_depth, model_normal, state, c2w, w2c, n, h, w, fx, fy, cx, cy,
                               max_distance, cos_max_angle, n_valid, partials, (cudaStream_t)stream);
}

static bool icp_partials(int32_t nb, int32_t n) { return n > 0 && n <= 65535 && nb > 0; }

int um_icp_solve(const double* partials, int32_t nb, int32_t n, const int32_t* n_valid, double min_inliers,
                 double min_pivot, int32_t record, double* state, void* stream) {
  UM_REQUIRE(partials && n_valid && state, "um_icp_solve: no pointer may be NULL");
  UM_REQUIRE(icp_partials(nb, n), "um_icp_solve: bad partials (%d frames of %d blocks)", n, nb);
  UM_REQUIRE(min_inliers >= 0.0 && min_inliers <= 1e300 && min_pivot > 0.0 && min_pivot <= 1.0,
             "um_icp_solve: min_inliers must be finite and >= 0, min_pivot in (0, 1]");
  UM_REQUIRE(um::aligned(partials, 8) && um::aligned(state, 8) && um::aligned(n_valid, 4),
             "um_icp_solve: partials and state must be 8-byte aligned, n_valid 4-byte aligned");
  UM_REQUIRE(um::written_disjoint({{state, 8LL * UM_ICP_STATE * n}, {partials, 8LL * UM_ICP_TERMS * nb * n}, {n_valid, 4}},
                                  1),
             "um_icp_solve: state must not overlap the inputs");
  return um::icp_solve_launch(partials, nb, n, n_valid, min_inliers, min_pivot, record != 0, state, (cudaStream_t)stream);
}

int um_icp_accept(const double* partials, int32_t nb, int32_t n, const int32_t* n_valid, double min_inlier_fraction,
                  const double* poses, double* correction, double* state, float* pose_out, uint8_t* tracked,
                  int64_t* inliers, float* rmse, float* w2c, void* stream) {
  UM_REQUIRE(partials && n_valid && state && pose_out && tracked && inliers && rmse && w2c,
             "um_icp_accept: no pointer but poses and correction may be NULL");
  UM_REQUIRE(icp_partials(nb, n), "um_icp_accept: bad partials (%d frames of %d blocks)", n, nb);
  UM_REQUIRE(!correction || (poses && n == 1), "um_icp_accept: a correction takes the poses of exactly one frame");
  UM_REQUIRE(min_inlier_fraction >= 0.0 && min_inlier_fraction <= 1.0,
             "um_icp_accept: min_inlier_fraction must be in [0, 1]");
  UM_REQUIRE(um::aligned(partials, 8) && um::aligned(state, 8) && um::aligned(poses, 8) && um::aligned(correction, 8) &&
                 um::aligned(inliers, 8) && um::aligned(n_valid, 4) && um::aligned(pose_out, 4) && um::aligned(rmse, 4) &&
                 um::aligned(w2c, 4),
             "um_icp_accept: the fp64 and int64 buffers must be 8-byte aligned, the fp32 and int32 buffers 4-byte aligned");
  UM_REQUIRE(um::written_disjoint({{state, 8LL * UM_ICP_STATE * n}, {pose_out, 64LL * n}, {tracked, n}, {inliers, 8LL * n},
                                   {rmse, 4LL * n}, {w2c, 48LL * n}, {correction, 128},
                                   {partials, 8LL * UM_ICP_TERMS * nb * n}, {poses, 128LL * n}, {n_valid, 4}},
                                  7),
             "um_icp_accept: the outputs must not overlap each other or the inputs");
  return um::icp_accept_launch(partials, nb, n, n_valid, min_inlier_fraction, poses, correction, state, pose_out, tracked,
                               inliers, rmse, w2c, (cudaStream_t)stream);
}

// ---- point clouds (um_cloud.cu) ----
static const long long kCloudMax = 0x7fffffffLL;            // int32 input indices and table positions

static long long cloud_blocks(long long n) { return (n + 255) / 256; }

// A grid: a finite origin, a positive finite cell size and 1 .. 2^21 cells per axis.
static bool cloud_grid(double ox, double oy, double oz, double cell, int32_t gx, int32_t gy, int32_t gz) {
  const double lim = 1.7976931348623157e308;
  return ox >= -lim && ox <= lim && oy >= -lim && oy <= lim && oz >= -lim && oz <= lim && cell > 0.0 && cell <= lim &&
         gx >= 1 && gy >= 1 && gz >= 1 && gx <= (1 << 21) && gy <= (1 << 21) && gz <= (1 << 21);
}

int um_cloud_keys(const float* points, int64_t n, double ox, double oy, double oz, double cell, int32_t gx, int32_t gy,
                  int32_t gz, int64_t* keys, void* stream) {
  UM_REQUIRE(n >= 0 && n <= kCloudMax, "um_cloud_keys: bad point count %lld (0 .. 2^31 - 1)", (long long)n);
  UM_REQUIRE(n == 0 || (points && keys), "um_cloud_keys: points and keys must not be NULL");
  UM_REQUIRE(cloud_grid(ox, oy, oz, cell, gx, gy, gz),
             "um_cloud_keys: bad grid (finite origin, positive finite cell, 1 .. 2^21 cells per axis)");
  UM_REQUIRE(um::aligned(points, 4) && um::aligned(keys, 8), "um_cloud_keys: points 4-byte, keys 8-byte aligned");
  UM_REQUIRE(um::written_disjoint({{keys, 8 * n}, {points, 12 * n}}, 1), "um_cloud_keys: keys must not overlap points");
  if (n == 0) return UM_OK;
  const double o[3] = {ox, oy, oz};
  const int g[3] = {gx, gy, gz};
  return um::cloud_keys_launch(points, n, o, cell, g, reinterpret_cast<long long*>(keys), (cudaStream_t)stream);
}

int um_cloud_ranges(const int64_t* sorted_keys, const int64_t* order, const float* points, int64_t n, int32_t gx,
                    int32_t gy, int32_t gz, int32_t* start, int32_t* end, float* sorted_points, void* stream) {
  UM_REQUIRE(sorted_keys && order && points && start && end && sorted_points, "um_cloud_ranges: no pointer may be NULL");
  UM_REQUIRE(n >= 1 && n <= kCloudMax, "um_cloud_ranges: bad point count %lld (1 .. 2^31 - 1)", (long long)n);
  UM_REQUIRE(gx >= 1 && gy >= 1 && gz >= 1 && (long long)gx * gy * gz <= kCloudMax,
             "um_cloud_ranges: bad table %d x %d x %d (at most 2^31 - 1 cells)", gx, gy, gz);
  UM_REQUIRE(um::aligned(sorted_keys, 8) && um::aligned(order, 8) && um::aligned(points, 4) && um::aligned(start, 4) &&
                 um::aligned(end, 4) && um::aligned(sorted_points, 16),
             "um_cloud_ranges: keys and order 8-byte, points and tables 4-byte, sorted_points 16-byte aligned");
  const long long c = (long long)gx * gy * gz;
  UM_REQUIRE(um::written_disjoint({{start, 4 * c}, {end, 4 * c}, {sorted_points, 16 * n}, {sorted_keys, 8 * n},
                                   {order, 8 * n}, {points, 12 * n}},
                                  3),
             "um_cloud_ranges: the tables and sorted_points must not overlap each other or the inputs");
  return um::cloud_ranges_launch(reinterpret_cast<const long long*>(sorted_keys), reinterpret_cast<const long long*>(order),
                                 points, n, c, start, end, sorted_points, (cudaStream_t)stream);
}

int um_cloud_down_sample_count(const int64_t* sorted_keys, int64_t n, int64_t* offsets, void* stream) {
  UM_REQUIRE(sorted_keys && offsets, "um_cloud_down_sample_count: no pointer may be NULL");
  UM_REQUIRE(n >= 1 && n <= kCloudMax, "um_cloud_down_sample_count: bad point count %lld (1 .. 2^31 - 1)", (long long)n);
  UM_REQUIRE(um::aligned(sorted_keys, 8) && um::aligned(offsets, 8),
             "um_cloud_down_sample_count: keys and offsets must be 8-byte aligned");
  UM_REQUIRE(um::written_disjoint({{offsets, 8 * (cloud_blocks(n) + 1)}, {sorted_keys, 8 * n}}, 1),
             "um_cloud_down_sample_count: offsets must not overlap the keys");
  return um::cloud_down_sample_count_launch(reinterpret_cast<const long long*>(sorted_keys), n,
                                            reinterpret_cast<long long*>(offsets), (cudaStream_t)stream);
}

int um_cloud_down_sample(const int64_t* sorted_keys, const int64_t* order, const float* points, int64_t n,
                         const int64_t* offsets, int64_t m, float* out, void* stream) {
  UM_REQUIRE(sorted_keys && order && points && offsets && out, "um_cloud_down_sample: no pointer may be NULL");
  UM_REQUIRE(n >= 1 && n <= kCloudMax && m >= 1 && m <= n, "um_cloud_down_sample: bad counts (%lld points, %lld cells)",
             (long long)n, (long long)m);
  UM_REQUIRE(um::aligned(sorted_keys, 8) && um::aligned(order, 8) && um::aligned(offsets, 8) && um::aligned(points, 4) &&
                 um::aligned(out, 4),
             "um_cloud_down_sample: keys, order and offsets 8-byte, points and out 4-byte aligned");
  UM_REQUIRE(um::written_disjoint({{out, 12 * m}, {sorted_keys, 8 * n}, {order, 8 * n}, {points, 12 * n},
                                   {offsets, 8 * (cloud_blocks(n) + 1)}},
                                  1),
             "um_cloud_down_sample: out must not overlap the inputs");
  return um::cloud_down_sample_launch(reinterpret_cast<const long long*>(sorted_keys),
                                      reinterpret_cast<const long long*>(order), points, n,
                                      reinterpret_cast<const long long*>(offsets), out, (cudaStream_t)stream);
}

int um_cloud_nearest(const float* queries, int64_t nq, const float* sorted_points, const int32_t* start,
                     const int32_t* end, int64_t n, double ox, double oy, double oz, double cell, int32_t gx, int32_t gy,
                     int32_t gz, float threshold, float* distance, int64_t* index, double* partial_sum,
                     int64_t* partial_count, void* stream) {
  UM_REQUIRE(nq >= 0 && nq <= kCloudMax && n >= 1 && n <= kCloudMax,
             "um_cloud_nearest: bad counts (%lld queries, %lld points; 0 .. 2^31 - 1 queries, 1 .. 2^31 - 1 points)",
             (long long)nq, (long long)n);
  UM_REQUIRE(sorted_points && start && end && (nq == 0 || queries), "um_cloud_nearest: no input may be NULL");
  UM_REQUIRE((distance && index && !partial_sum && !partial_count) || (!distance && !index && partial_sum && partial_count),
             "um_cloud_nearest: give distance and index, or partial_sum and partial_count");
  UM_REQUIRE(cloud_grid(ox, oy, oz, cell, gx, gy, gz) && (long long)gx * gy * gz <= kCloudMax,
             "um_cloud_nearest: bad grid (finite origin, positive finite cell, 1 .. 2^21 cells per axis, at most 2^31 - 1)");
  UM_REQUIRE(!partial_sum || (threshold > 0.f && threshold <= 3.402823466e38f),
             "um_cloud_nearest: threshold must be positive and finite");
  UM_REQUIRE(um::aligned(queries, 4) && um::aligned(sorted_points, 16) && um::aligned(start, 4) && um::aligned(end, 4) &&
                 um::aligned(distance, 4) && um::aligned(index, 8) && um::aligned(partial_sum, 8) &&
                 um::aligned(partial_count, 8),
             "um_cloud_nearest: sorted_points 16-byte, index and partials 8-byte, the rest 4-byte aligned");
  const long long c = (long long)gx * gy * gz, nb = cloud_blocks(nq);
  UM_REQUIRE(um::written_disjoint({{distance, 4 * nq}, {index, 8 * nq}, {partial_sum, 8 * nb}, {partial_count, 8 * nb},
                                   {queries, 12 * nq}, {sorted_points, 16 * n}, {start, 4 * c}, {end, 4 * c}},
                                  4),
             "um_cloud_nearest: the outputs must not overlap each other or the inputs");
  if (nq == 0) return UM_OK;
  const double o[3] = {ox, oy, oz};
  const int g[3] = {gx, gy, gz};
  return um::cloud_nearest_launch(queries, nq, sorted_points, start, end, o, cell, g, threshold, distance,
                                  reinterpret_cast<long long*>(index), partial_sum,
                                  reinterpret_cast<long long*>(partial_count), (cudaStream_t)stream);
}

int um_cloud_stats(const double* partial_sum, const int64_t* partial_count, int64_t nb, double* out, void* stream) {
  UM_REQUIRE(out && (nb == 0 || (partial_sum && partial_count)), "um_cloud_stats: no pointer may be NULL");
  UM_REQUIRE(nb >= 0 && nb <= cloud_blocks(kCloudMax), "um_cloud_stats: bad block count %lld", (long long)nb);
  UM_REQUIRE(um::aligned(partial_sum, 8) && um::aligned(partial_count, 8) && um::aligned(out, 8),
             "um_cloud_stats: the buffers must be 8-byte aligned");
  UM_REQUIRE(um::written_disjoint({{out, 16}, {partial_sum, 8 * nb}, {partial_count, 8 * nb}}, 1),
             "um_cloud_stats: out must not overlap the partials");
  return um::cloud_stats_launch(partial_sum, reinterpret_cast<const long long*>(partial_count), nb, out,
                                (cudaStream_t)stream);
}

// ---- triangle meshes (um_raster.cu) ----
static const long long kMeshMax = 0x7fffffffLL;             // int32 face indices, vertex indices and bin positions

static long long mesh_tiles(int32_t h, int32_t w) { return (((long long)h + 15) / 16) * (((long long)w + 15) / 16); }

// n views of h x w pixels and the camera: n 1 .. 65535, h w <= 2^31 - 1, fx fy finite nonzero, cx cy finite,
// near finite > 0, far > near.
static bool mesh_camera(int32_t n, int32_t h, int32_t w, float fx, float fy, float cx, float cy, float near, float far) {
  return n > 0 && n <= 65535 && h > 0 && w > 0 && (long long)h * w <= kMeshMax && fx != 0.f && fy != 0.f &&
         finite_value(fx) && finite_value(fy) && finite_value(cx) && finite_value(cy) && near > 0.f &&
         finite_value(near) && far > near;
}

static bool mesh_counts(int64_t n_points, int64_t n_faces) {
  return n_points >= 1 && n_points <= kMeshMax && n_faces >= 1 && n_faces <= kMeshMax;
}

int um_mesh_bin_count(const float* points, int64_t n_points, const int32_t* faces, int64_t n_faces, const float* w2c,
                      int32_t n, int32_t h, int32_t w, float fx, float fy, float cx, float cy, float near, float far,
                      int64_t* offsets, void* stream) {
  UM_REQUIRE(points && faces && w2c && offsets, "um_mesh_bin_count: no pointer may be NULL");
  UM_REQUIRE(mesh_counts(n_points, n_faces), "um_mesh_bin_count: bad mesh (%lld points, %lld faces; 1 .. 2^31 - 1 each)",
             (long long)n_points, (long long)n_faces);
  UM_REQUIRE(mesh_camera(n, h, w, fx, fy, cx, cy, near, far),
             "um_mesh_bin_count: bad cameras (1 .. 65535 views of at most 2^31 - 1 pixels, fx fy finite nonzero, cx cy "
             "finite, near finite > 0, far > near)");
  UM_REQUIRE(um::aligned(points, 4) && um::aligned(faces, 4) && um::aligned(w2c, 4) && um::aligned(offsets, 8),
             "um_mesh_bin_count: points, faces and w2c 4-byte, offsets 8-byte aligned");
  const long long nb = (long long)n * ((n_faces + 255) / 256);
  UM_REQUIRE(um::written_disjoint({{offsets, 8 * (nb + 1)}, {points, 12 * n_points}, {faces, 12 * n_faces},
                                   {w2c, 48LL * n}},
                                  1),
             "um_mesh_bin_count: offsets must not overlap the inputs");
  return um::mesh_bin_count_launch(points, faces, n_faces, w2c, n, h, w, fx, fy, cx, cy, near, far,
                                   reinterpret_cast<long long*>(offsets), (cudaStream_t)stream);
}

int um_mesh_bin(const float* points, int64_t n_points, const int32_t* faces, int64_t n_faces, const float* w2c, int32_t n,
                int32_t h, int32_t w, float fx, float fy, float cx, float cy, float near, float far,
                const int64_t* offsets, int64_t n_entries, int64_t* keys, int64_t* values, void* stream) {
  UM_REQUIRE(points && faces && w2c && offsets && keys && values, "um_mesh_bin: no pointer may be NULL");
  UM_REQUIRE(mesh_counts(n_points, n_faces), "um_mesh_bin: bad mesh (%lld points, %lld faces; 1 .. 2^31 - 1 each)",
             (long long)n_points, (long long)n_faces);
  UM_REQUIRE(mesh_camera(n, h, w, fx, fy, cx, cy, near, far), "um_mesh_bin: bad cameras (see um_mesh_bin_count)");
  UM_REQUIRE(n_entries >= 1 && n_entries <= kMeshMax, "um_mesh_bin: bad entry count %lld (1 .. 2^31 - 1)",
             (long long)n_entries);
  UM_REQUIRE(um::aligned(points, 4) && um::aligned(faces, 4) && um::aligned(w2c, 4) && um::aligned(offsets, 8) &&
                 um::aligned(keys, 8) && um::aligned(values, 8),
             "um_mesh_bin: points, faces and w2c 4-byte, offsets, keys and values 8-byte aligned");
  const long long nb = (long long)n * ((n_faces + 255) / 256);
  UM_REQUIRE(um::written_disjoint({{keys, 8 * n_entries}, {values, 8 * n_entries}, {offsets, 8 * (nb + 1)},
                                   {points, 12 * n_points}, {faces, 12 * n_faces}, {w2c, 48LL * n}},
                                  2),
             "um_mesh_bin: keys and values must not overlap each other or the inputs");
  return um::mesh_bin_launch(points, faces, n_faces, w2c, n, h, w, fx, fy, cx, cy, near, far,
                             reinterpret_cast<const long long*>(offsets), reinterpret_cast<long long*>(keys),
                             reinterpret_cast<long long*>(values), (cudaStream_t)stream);
}

int um_mesh_ranges(const int64_t* sorted_keys, int64_t n_entries, int32_t n, int32_t h, int32_t w, int32_t* start,
                   int32_t* end, void* stream) {
  UM_REQUIRE(start && end && (n_entries == 0 || sorted_keys), "um_mesh_ranges: no pointer may be NULL");
  UM_REQUIRE(n_entries >= 0 && n_entries <= kMeshMax, "um_mesh_ranges: bad entry count %lld (0 .. 2^31 - 1)",
             (long long)n_entries);
  UM_REQUIRE(n > 0 && n <= 65535 && h > 0 && w > 0 && (long long)h * w <= kMeshMax,
             "um_mesh_ranges: bad views (%d x %d x %d; at most 65535 views of 2^31 - 1 pixels)", n, h, w);
  UM_REQUIRE(um::aligned(sorted_keys, 8) && um::aligned(start, 4) && um::aligned(end, 4),
             "um_mesh_ranges: keys 8-byte, tables 4-byte aligned");
  const long long bins = n * mesh_tiles(h, w);
  UM_REQUIRE(um::written_disjoint({{start, 4 * bins}, {end, 4 * bins}, {sorted_keys, 8 * n_entries}}, 2),
             "um_mesh_ranges: the tables must not overlap each other or the keys");
  return um::mesh_ranges_launch(reinterpret_cast<const long long*>(sorted_keys), n_entries, bins, start, end,
                                (cudaStream_t)stream);
}

int um_mesh_raster(const float* points, int64_t n_points, const int32_t* faces, int64_t n_faces, const uint8_t* colors,
                   const float* w2c, int32_t n, int32_t h, int32_t w, float fx, float fy, float cx, float cy, float near,
                   float far, const int64_t* order, const int64_t* values, int64_t n_entries, const int32_t* start,
                   const int32_t* end, float* depth, int32_t* face, uint8_t* rgb, void* stream) {
  UM_REQUIRE(points && faces && w2c && start && end && depth && face && (n_entries == 0 || (order && values)),
             "um_mesh_raster: no pointer but colors and rgb may be NULL");
  UM_REQUIRE(!colors == !rgb, "um_mesh_raster: give colors and rgb together");
  UM_REQUIRE(mesh_counts(n_points, n_faces), "um_mesh_raster: bad mesh (%lld points, %lld faces; 1 .. 2^31 - 1 each)",
             (long long)n_points, (long long)n_faces);
  UM_REQUIRE(mesh_camera(n, h, w, fx, fy, cx, cy, near, far), "um_mesh_raster: bad cameras (see um_mesh_bin_count)");
  UM_REQUIRE(n_entries >= 0 && n_entries <= kMeshMax, "um_mesh_raster: bad entry count %lld (0 .. 2^31 - 1)",
             (long long)n_entries);
  UM_REQUIRE(um::aligned(points, 4) && um::aligned(faces, 4) && um::aligned(w2c, 4) && um::aligned(order, 8) &&
                 um::aligned(values, 8) && um::aligned(start, 4) && um::aligned(end, 4) && um::aligned(depth, 4) &&
                 um::aligned(face, 4),
             "um_mesh_raster: order and values 8-byte, the other int32 and fp32 buffers 4-byte aligned");
  const long long px = (long long)n * h * w, bins = n * mesh_tiles(h, w);
  UM_REQUIRE(um::written_disjoint({{depth, 4 * px}, {face, 4 * px}, {rgb, 3 * px}, {points, 12 * n_points},
                                   {faces, 12 * n_faces}, {colors, 3 * n_points}, {w2c, 48LL * n},
                                   {order, 8 * n_entries}, {values, 8 * n_entries}, {start, 4 * bins}, {end, 4 * bins}},
                                  3),
             "um_mesh_raster: depth, face and rgb must not overlap each other or the inputs");
  return um::mesh_raster_launch(points, faces, colors, w2c, n, h, w, fx, fy, cx, cy, near, far,
                                reinterpret_cast<const long long*>(order), reinterpret_cast<const long long*>(values),
                                start, end, depth, face, rgb, (cudaStream_t)stream);
}

int um_visible_points(const float* points, int64_t n_points, const float* depth, int32_t n, int32_t h, int32_t w,
                      const float* w2c, float fx, float fy, float cx, float cy, float tolerance, uint8_t* visible,
                      void* stream) {
  UM_REQUIRE(n_points >= 0 && n_points <= kMeshMax, "um_visible_points: bad point count %lld (0 .. 2^31 - 1)",
             (long long)n_points);
  UM_REQUIRE(n_points == 0 || (points && visible), "um_visible_points: points and visible must not be NULL");
  UM_REQUIRE(n >= 0 && n <= 65535 && h > 0 && w > 0 && (long long)h * w <= kMeshMax,
             "um_visible_points: bad views (%d x %d x %d; at most 65535 views of 2^31 - 1 pixels)", n, h, w);
  UM_REQUIRE(n == 0 || (depth && w2c), "um_visible_points: depth and w2c must not be NULL");
  UM_REQUIRE(fx != 0.f && fy != 0.f && finite_value(fx) && finite_value(fy) && finite_value(cx) && finite_value(cy),
             "um_visible_points: fx and fy must be finite and nonzero, cx and cy finite");
  UM_REQUIRE(finite_value(tolerance) && tolerance >= 0.f, "um_visible_points: tolerance must be finite and >= 0");
  UM_REQUIRE(um::aligned(points, 4) && um::aligned(depth, 4) && um::aligned(w2c, 4),
             "um_visible_points: the fp32 buffers must be 4-byte aligned");
  UM_REQUIRE(um::written_disjoint({{visible, n_points}, {points, 12 * n_points}, {depth, 4LL * n * h * w},
                                   {w2c, 48LL * n}},
                                  1),
             "um_visible_points: visible must not overlap the inputs");
  if (n_points == 0) return UM_OK;
  return um::visible_points_launch(points, n_points, depth, n, h, w, w2c, fx, fy, cx, cy, tolerance, visible,
                                   (cudaStream_t)stream);
}

int um_depth_metrics(const float* pred, const float* gt, int32_t n, int32_t h, int32_t w, float max_depth,
                     double* partials, double* out, void* stream) {
  UM_REQUIRE(pred && gt && partials && out, "um_depth_metrics: no pointer may be NULL");
  UM_REQUIRE(n > 0 && n <= 65535 && h > 0 && w > 0 && (long long)h * w <= kMeshMax,
             "um_depth_metrics: bad frames (%d x %d x %d; at most 65535 frames of 2^31 - 1 pixels)", n, h, w);
  UM_REQUIRE(max_depth > 0.f, "um_depth_metrics: max_depth must be > 0");
  UM_REQUIRE(um::aligned(pred, 4) && um::aligned(gt, 4) && um::aligned(partials, 8) && um::aligned(out, 8),
             "um_depth_metrics: pred and gt 4-byte, partials and out 8-byte aligned");
  const long long px = (long long)n * h * w, nb = ((long long)h * w + 255) / 256;
  UM_REQUIRE(um::written_disjoint({{partials, 8LL * UM_DEPTH_METRIC_TERMS * n * nb}, {out, 8LL * UM_DEPTH_METRIC_TERMS * n},
                                   {pred, 4 * px}, {gt, 4 * px}},
                                  2),
             "um_depth_metrics: partials and out must not overlap each other or the inputs");
  return um::depth_metrics_launch(pred, gt, n, h, w, max_depth, partials, out, (cudaStream_t)stream);
}

// ---- multi-view consistency of depth maps and their points (um_consistency.cu) ----
static const long long kMaxDepthPixels = 1LL << 39;          // the point passes' blocks of 256 fit a 2^31 - 1 grid

// n maps of h x w: n 1 .. 65535, h w <= 2^31 - 1, n h w <= 2^39
static bool depth_maps(int32_t n, int32_t h, int32_t w) {
  return n > 0 && n <= 65535 && h > 0 && w > 0 && (long long)h * w <= 0x7fffffffLL && (long long)n * h * w <= kMaxDepthPixels;
}

int um_depth_consistency(const float* depth, int32_t n, int32_t h, int32_t w, float fx, float fy, float cx, float cy,
                         const float* c2w, const float* w2c, const int32_t* refs, int32_t r, const int32_t* sources,
                         int32_t s, float max_pixel, float max_relative, int32_t min_views, uint8_t* views, float* out,
                         void* stream) {
  UM_REQUIRE(depth && c2w && w2c && refs && sources && views && out, "um_depth_consistency: no pointer may be NULL");
  UM_REQUIRE(depth_maps(n, h, w),
             "um_depth_consistency: bad depths (%d x %d x %d; 1 .. 65535 maps of 1 .. 2^31 - 1 pixels, 2^39 in all)", n, h,
             w);
  UM_REQUIRE(r > 0 && r <= 65535, "um_depth_consistency: bad reference count %d (1 .. 65535)", r);
  UM_REQUIRE(s > 0 && s <= 255, "um_depth_consistency: bad source count %d (1 .. 255: views is uint8)", s);
  UM_REQUIRE(min_views >= 1 && min_views <= s, "um_depth_consistency: min_views %d outside [1, %d]", min_views, s);
  UM_REQUIRE(positive_finite(max_pixel) && positive_finite(max_relative),
             "um_depth_consistency: max_pixel and max_relative must be positive and finite");
  UM_REQUIRE(icp_intrinsics(fx, fy, cx, cy), "um_depth_consistency: fx and fy must be finite and nonzero, cx and cy finite");
  UM_REQUIRE(um::aligned(depth, 4) && um::aligned(c2w, 4) && um::aligned(w2c, 4) && um::aligned(refs, 4) &&
                 um::aligned(sources, 4) && um::aligned(out, 4),
             "um_depth_consistency: the fp32 and int32 buffers must be 4-byte aligned");
  const long long hw = (long long)h * w, px = (long long)r * hw;
  UM_REQUIRE(um::written_disjoint({{views, px}, {out, 4 * px}, {depth, 4 * n * hw}, {c2w, 48LL * n}, {w2c, 48LL * n},
                                   {refs, 4LL * r}, {sources, 4LL * r * s}},
                                  2),
             "um_depth_consistency: views and out must not overlap each other or the inputs");
  return um::depth_consistency_launch(depth, n, h, w, fx, fy, cx, cy, c2w, w2c, refs, r, sources, s, max_pixel,
                                      max_relative, min_views, views, out, (cudaStream_t)stream);
}

int um_depth_points_count(const float* depth, int32_t n, int32_t h, int32_t w, int64_t* offsets, void* stream) {
  UM_REQUIRE(depth && offsets, "um_depth_points_count: no pointer may be NULL");
  UM_REQUIRE(depth_maps(n, h, w),
             "um_depth_points_count: bad depths (%d x %d x %d; 1 .. 65535 maps of 1 .. 2^31 - 1 pixels, 2^39 in all)", n,
             h, w);
  UM_REQUIRE(um::aligned(depth, 4) && um::aligned(offsets, 8),
             "um_depth_points_count: depth 4-byte, offsets 8-byte aligned");
  const long long px = (long long)n * h * w, nb = (px + 255) / 256;
  UM_REQUIRE(um::written_disjoint({{offsets, 8 * (nb + 1)}, {depth, 4 * px}}, 1),
             "um_depth_points_count: offsets must not overlap depth");
  return um::depth_points_count_launch(depth, px, reinterpret_cast<long long*>(offsets), (cudaStream_t)stream);
}

int um_depth_points(const float* depth, const uint8_t* frames, int32_t n, int32_t h, int32_t w, float fx, float fy,
                    float cx, float cy, const float* c2w, const int64_t* offsets, int64_t n_points, float* points,
                    uint8_t* colors, void* stream) {
  UM_REQUIRE(depth && frames && c2w && offsets, "um_depth_points: no pointer may be NULL");
  UM_REQUIRE(n_points == 0 || (points && colors), "um_depth_points: points and colors must not be NULL");
  UM_REQUIRE(depth_maps(n, h, w),
             "um_depth_points: bad depths (%d x %d x %d; 1 .. 65535 maps of 1 .. 2^31 - 1 pixels, 2^39 in all)", n, h, w);
  const long long px = (long long)n * h * w, nb = (px + 255) / 256;
  UM_REQUIRE(n_points >= 0 && n_points <= px && n_points <= 0x7fffffffLL,
             "um_depth_points: bad point count %lld (0 .. min(pixels, 2^31 - 1))", (long long)n_points);
  UM_REQUIRE(icp_intrinsics(fx, fy, cx, cy), "um_depth_points: fx and fy must be finite and nonzero, cx and cy finite");
  UM_REQUIRE(um::aligned(depth, 4) && um::aligned(c2w, 4) && um::aligned(offsets, 8) && um::aligned(points, 4),
             "um_depth_points: depth, c2w and points 4-byte, offsets 8-byte aligned");
  UM_REQUIRE(um::written_disjoint({{points, 12 * n_points}, {colors, 3 * n_points}, {depth, 4 * px}, {frames, 3 * px},
                                   {c2w, 48LL * n}, {offsets, 8 * (nb + 1)}},
                                  2),
             "um_depth_points: points and colors must not overlap each other or the inputs");
  if (n_points == 0) return UM_OK;
  return um::depth_points_launch(depth, frames, n, h, w, fx, fy, cx, cy, c2w, reinterpret_cast<const long long*>(offsets),
                                 points, colors, (cudaStream_t)stream);
}

}  // extern "C"
