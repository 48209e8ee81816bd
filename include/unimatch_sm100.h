/* unimatch_sm100.h -- C ABI of libunimatch_sm100.so (H100 / sm_90a kernels for the UniMatch matching path).
 *
 * The reference (autonomousvision/unimatch) is pure Python/PyTorch and has no FFI of its own; these entry
 * points are what a binding for its hot-path functions would call.  Each declaration cites the reference
 * function it replaces (paths relative to the reference checkout).
 *
 * Conventions
 *  - Every pointer is a DEVICE pointer to fp32 data unless stated otherwise; the caller owns all memory
 *    (outputs pre-allocated); nothing is allocated, freed or retained.
 *  - Feature maps are channel-last: a "token matrix" [N, L, C] with L = h*w (row-major y, x) and C = 128.
 *    Two-view tensors stack view 0 of all B pairs, then view 1: N = 2B, stream n = view*B + b.
 *  - Flow-like maps are channel-last too: [B, h, w, F] with F = 2 (flow: x, y) or 1 (disparity, inverse depth).
 *  - `stream` is a cudaStream_t passed as void*.  Work is enqueued, never synchronised.
 *  - Return value: 0 on success, a negative UM_E* code otherwise; um_last_error() gives the message
 *    (thread-local).  There is no CPU fallback: without a usable device every launcher fails.
 */
#ifndef UNIMATCH_SM100_H_
#define UNIMATCH_SM100_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define UM_OK 0
#define UM_EINVAL (-22)   /* bad argument (shape, alignment, unsupported mode) */
#define UM_ECUDA (-5)     /* CUDA runtime error at launch */

#define UM_FEATURE_DIM 128

/* ABI version and build info.  The version changes when an entry point changes or is removed; new entry points (the
 * tracks, the submission encoder, the scene-flow warp and statistics, TSDF fusion, meshing, ray casting, ICP, the
 * point-cloud ops and the mesh rasteriser) leave existing callers working and keep it. */
#define UM_ABI_VERSION 4
int um_abi_version(void);
const char* um_build_info(void);
const char* um_last_error(void);
/* Number of kernel launches issued through this library by the calling process (for bench `gpu_launches`). */
int64_t um_launch_count(void);

/* ---- window attention ------------------------------------------------------------------------------------
 * mask_mode */
#define UM_MASK_NONE 0
#define UM_MASK_SWIN 1     /* additive -100 between different shift regions (utils.py:84-108, :199-216)   */
#define UM_MASK_CAUSAL 2   /* keys with x_k > x_q get logit -1e9 (matching.py:138-142)                    */

/* Geometry of one windowed-attention problem over an h x w token grid.
 *   kh, kw : number of windows along y and x (window = (h/kh) x (w/kw) tokens)
 *   sh, sw : cyclic roll applied before splitting (attention.py:72-79, :132-138), 0 = unshifted
 * 2-D Swin: kh = kw = K, (sh, sw) = (wh/2, ww/2) on shifted layers.  1-D (per image row): kh = h.
 * Full attention: kh = kw = 1. */
typedef struct um_attn_geom {
  int32_t h, w;
  int32_t kh, kw;
  int32_t sh, sw;
  int32_t mask_mode;
} um_attn_geom;

/* out[n, t, :] = softmax_k( q[n,t,:] . k[m,k,:] / sqrt(128) + mask ) v[m,k,:],  m = (n + kv_shift) mod N,
 * keys k ranging over the window of token t.
 * Replaces single_head_full_attention (attention.py:8-16), single_head_full_attention_1d (:19-42),
 * single_head_split_window_attention (:45-104) and single_head_split_window_attention_1d (:107-163).
 * q, k, v, out: [N, L, *] with row strides ldq, ldk, ldv, ldo (floats, multiples of 4) and batch stride L*ld. */
int um_window_attention(const float* q, const float* k, const float* v, float* out,
                        int32_t n_streams, int32_t kv_shift,
                        int64_t ldq, int64_t ldk, int64_t ldv, int64_t ldo,
                        const um_attn_geom* geom, void* workspace, int64_t workspace_bytes, int32_t flags,
                        void* stream);
/* Dense 2-D windows of >= 128 tokens run on the Hopper tensor cores (wgmma, fp16 hi/lo split operands, fp32
 * accumulation, fp32-faithful); they need a device scratch buffer of um_window_attention_workspace() bytes for the
 * window-major operand planes (0 = this geometry runs on CUDA cores and needs none).  flags: */
#define UM_ATTN_FORCE_CUDA_CORES 1   /* diagnostic: use the exact-fp32 CUDA-core kernel for every shape */
int64_t um_window_attention_workspace(const um_attn_geom* geom, int32_t n_streams);

/* The same attention on operands that are ALREADY window-major fp16 (hi, lo) planes [2][n_streams][kh*kw][lp][128]
 * (lp = um_attention_planes_lp(geom): the window length rounded up to 128; rows [lw, lp) of every window must be zero):
 * the projection GEMM writes them directly (um_conv_desc.win_dst), so the fp32 q/k/v rows never exist.
 * Output: fp32 rows (out, row stride ldo) and/or fp16 (hi, lo) planes [2][>= n_streams*h*w rows][128] in token order
 * (out_split, planes split_plane_stride halves apart) = the operand planes of the merge Linear layer.
 * um_attention_planes_lp() == 0: geometry runs on the CUDA-core kernel (um_window_attention) instead.
 * Replaces single_head_split_window_attention / single_head_full_attention (attention.py:8-16, :45-104). */
int32_t um_attention_planes_lp(const um_attn_geom* geom);
int um_window_attention_planes(const void* q_planes, const void* k_planes, const void* v_planes, float* out, int64_t ldo,
                               void* out_split, int64_t split_plane_stride, int32_t n_streams, int32_t kv_shift,
                               const um_attn_geom* geom, void* stream);

/* value_mode for um_softmax_expectation */
#define UM_VALUE_TENSOR 0   /* values[m, k, 0..vdim)                                                        */
#define UM_VALUE_COORDS 1   /* analytic pixel coordinates of key k: (x_k, y_k), vdim = 2                    */
#define UM_VALUE_XCOORD 2   /* analytic x_k only, vdim = 1                                                   */
/* post_op */
#define UM_POST_NONE 0
#define UM_POST_MINUS_OWN 1   /* out = E[value] - (x_t, y_t)   (matching.py:31-34)                          */
#define UM_POST_OWN_MINUS 2   /* out = x_t - E[value]          (matching.py:146-149)                        */

/* out[n, t, 0..vdim) = post( sum_k softmax_k( q[n,t,:] . k[m,k,:] / sqrt(128) + mask ) value_k ).
 * The L x L score matrix never leaves the SM.
 * Replaces global_correlation_softmax (matching.py:7-36), global_correlation_softmax_stereo (:126-151)
 * and the global branch of SelfAttnPropagation.forward (attention.py:194-215).
 * n_streams queries streams are processed (n = 0..n_streams-1), keys taken from stream (n + kv_shift) mod
 * n_total.  values (UM_VALUE_TENSOR): [n_total, L, vdim] contiguous, indexed by the KEY stream. */
int um_softmax_expectation(const float* q, const float* k, const float* values, float* out,
                           int32_t n_streams, int32_t n_total, int32_t kv_shift,
                           int64_t ldq, int64_t ldk, int32_t vdim, int32_t value_mode, int32_t post_op,
                           const um_attn_geom* geom, void* workspace, int64_t workspace_bytes, int32_t flags,
                           void* stream);
/* Global (one window = the whole map) problems of >= 128 tokens run on the Hopper tensor cores: S = Q K^T tiles in
 * registers, softmax and sum_k p_k value_k in registers.  Scratch bytes (0 = CUDA-core path, none needed); flags as above. */
int64_t um_softmax_expectation_workspace(const um_attn_geom* geom, int32_t n_total, int32_t value_mode);

/* ---- local (windowed, HBM/L2-bound) matching --------------------------------------------------------------
 * flow[b, y, x, :] = sum_k softmax_k( f0[b,y,x,:] . f1[b, y+dy_k, x+dx_k, :] / sqrt(128) ) (dx_k, dy_k),
 * (2ry+1) x (2rx+1) integer window, out-of-image taps get logit -1e9.
 * stereo != 0: returns -flow_x only ([B,h,w,1]).
 * Replaces local_correlation_softmax (matching.py:39-83) and local_correlation_softmax_stereo (:154-200). */
int um_local_corr_softmax(const float* f0, const float* f1, float* flow,
                          int32_t batch, int32_t h, int32_t w, int32_t ry, int32_t rx, int32_t stereo,
                          void* stream);

/* corr[b, y, x, k] = f0[b,y,x,:] . bilinear(f1[b], x + dx_k + u, y + dy_k + v) / sqrt(128), k = iy*(2r+1)+ix,
 * zero padding, align_corners=True; (u, v) = flow[b,y,x,:] (flow_dim 2) or (-flow[b,y,x,0], 0) when
 * flow_dim == 1 (disparity, unimatch.py:277-287).  corr is channel-last [B, h, w, (2r+1)^2].
 * Replaces local_correlation_with_flow (matching.py:86-123). */
int um_local_corr_volume(const float* f0, const float* f1, const float* flow, float* corr,
                         int32_t batch, int32_t h, int32_t w, int32_t radius, int32_t flow_dim, void* stream);

/* out[b,y,x,:] = bilinear(f[b], x + u, y + v), zeros outside, align_corners=True; (u,v) as above.
 * Replaces flow_warp (geometry.py:65-72, bilinear_sample :41-62). */
int um_flow_warp(const float* f, const float* flow, float* out,
                 int32_t batch, int32_t h, int32_t w, int32_t flow_dim, void* stream);

/* Occlusion masks from a forward / backward flow pair, both PLANAR [B,2,H,W] (what UniMatch.forward returns):
 * fwd_occ[b,y,x] = | fwd + warp(bwd, fwd) | > alpha (|fwd| + |bwd|) + beta, bwd_occ likewise with the roles swapped;
 * 1.0 = occluded.  Replaces forward_backward_consistency_check (geometry.py:75-96; called at evaluate_flow.py:792). */
int um_fb_consistency(const float* fwd_flow, const float* bwd_flow, float alpha, float beta, float* fwd_occ,
                      float* bwd_occ, int32_t batch, int32_t h, int32_t w, void* stream);

/* um_fb_consistency plus the forward residual: fwd_occ and bwd_occ are bit-identical to um_fb_consistency's (the same
 * kernel), and fwd_err [B,H,W] = | fwd + warp(bwd, fwd) |, the very fp32 value that the forward mask compares with
 * alpha (|fwd| + |bwd|) + beta.  In fp32, with (u, v) = fwd[b,:,y,x] and s = size - 1 per axis: px = x + u,
 * ix = ((2 px / s - 1) + 1) / 2 * s (likewise iy), x0 = floor(ix), the weights nw = (x0 + 1 - ix)(y0 + 1 - iy),
 * ne = (ix - x0)(y0 + 1 - iy), sw = (x0 + 1 - ix)(iy - y0), se = (ix - x0)(iy - y0), and warp = fma(se, v11, fma(sw, v10,
 * fma(ne, v01, nw v00))) over the corners inside the frame (zero padding); dx = u + warp.u, dy = v + warp.v,
 * fwd_err = sqrt(fma(dx, dx, dy * dy)), every other operation correctly rounded on its own.  The uncertainty of the
 * multi-flow tracks (um_multi_flow_tracks). */
int um_fb_consistency_error(const float* fwd_flow, const float* bwd_flow, float alpha, float beta, float* fwd_occ,
                            float* bwd_occ, float* fwd_err, int32_t batch, int32_t h, int32_t w, void* stream);

/* out[b,y,x,:] = sum_{3x3 nb} softmax( q[b,y,x,:] . k[b,nb,:] / sqrt(128) ) flow[b,nb,:]; out-of-image
 * neighbours take part with logit 0 and value 0 (zero-padded unfold).
 * Replaces SelfAttnPropagation.forward_local_window_attn (attention.py:217-253). */
int um_propagate_local(const float* q, const float* k, const float* flow, float* out,
                       int32_t batch, int32_t h, int32_t w, int32_t radius, int32_t flow_dim,
                       int64_t ldq, int64_t ldk, void* stream);

/* Plane-sweep matching: out[b,y,x,0] = sum_d softmax_d( f0 . bilinear(f1, proj_d(x,y)) / sqrt(128) ) cand_d
 * (or cand_argmax when from_argmax), proj_d = K (R K^-1 [x,y,1]^T / cand_d + t), uv = xy / max(z, 1e-3).
 * Kmat [B,9] (already scaled to the feature resolution), Kinv [B,9], pose [B,16] row-major (host computes the
 * 3x3 inverse).  cand: [D] inverse-depth candidates.
 * Replaces correlation_softmax_depth (matching.py:203-236) + warp_with_pose_depth_candidates (:239-282). */
int um_depth_corr_softmax(const float* f0, const float* f1, const float* Kmat, const float* Kinv,
                          const float* pose, const float* cand, float* out,
                          int32_t batch, int32_t h, int32_t w, int32_t num_cand, int32_t from_argmax,
                          void* stream);

/* ---- glue on the path ---------------------------------------------------------------------------------------
 * x[n, y, x, :] += table[(y mod wh), (x mod ww), :], table [wh, ww, 128] = PositionEmbeddingSine on the window.
 * Replaces feature_add_position (utils.py:111-131). */
int um_add_position(const float* x, const float* table, float* out,
                    int32_t n_streams, int32_t h, int32_t w, int32_t wh, int32_t ww, void* stream);

/* Convex upsampling: up[b, c, y*F+ky, x*F+kx] = sum_t softmax_t(mask[b,y,x, t*F*F + ky*F + kx]) * mult*flow[b, nb_t, c],
 * 3x3 zero-padded neighbourhood.  mask channel-last [B,h,w,9*F*F]; flow [B,h,w,fd]; up is PLANAR [B, fd, h*F, w*F]
 * (the layout the reference returns).  Replaces upsample_flow_with_mask (utils.py:134-152). */
int um_convex_upsample(const float* flow, const float* mask, float* up,
                       int32_t batch, int32_t h, int32_t w, int32_t flow_dim, int32_t factor, float mult,
                       void* stream);

/* Bilinear x2 upsampling (align_corners=True) of a channel-last flow map, values multiplied by `mult`.
 * Replaces F.interpolate(flow, scale_factor=2, mode='bilinear', align_corners=True) * 2 (unimatch.py:154). */
int um_upsample2x(const float* flow, float* out, int32_t batch, int32_t h, int32_t w, int32_t flow_dim,
                  float mult, void* stream);

/* Planar bilinear resize with align_corners=True: out[b,c] = scale[c] * resize(in[b,c]) for [B, C <= 3, H, W] fp32 tensors;
 * `scale` = HOST array of C floats or NULL; flip_x != 0 mirrors the output horizontally.  The callers' side of the boundary:
 * F.interpolate(..., mode='bilinear', align_corners=True) before the model and on its output, with the flow-component /
 * disparity rescale and the hflip of the bidirectional-disparity trick folded in (evaluate_flow.py:733-755,
 * evaluate_stereo.py:776-813, evaluate_depth.py:372-400). */
int um_resize_bilinear(const float* in, float* out, int32_t batch, int32_t channels, int32_t h_in, int32_t w_in,
                       int32_t h_out, int32_t w_out, const float* scale, int32_t flip_x, void* stream);

/* Video frames to model input: frames = DEVICE uint8 [n, h, w, 3] channel-last (what decoders produce) -> out fp32 planar
 * [n, 3, h_out, w_out], bit-identical to um_resize_bilinear of the float-converted planar frames.  transpose != 0 reads each
 * frame as its transpose [3, w, h] first (the portrait rule of evaluate_flow.py:713-717), so (h_out, w_out) is the size of
 * the transposed image.  At (h_out, w_out) equal to the source size the pass is an exact conversion.  Replaces the host-side
 * `torch.from_numpy(image).permute(2, 0, 1).float()`, transpose and F.interpolate of evaluate_flow.py:710-733. */
int um_frames_to_planar(const uint8_t* frames, float* out, int32_t n, int32_t h, int32_t w, int32_t transpose,
                        int32_t h_out, int32_t w_out, void* stream);

/* Depth-sequence frames to model input: frames = DEVICE uint8 [n, h, w, 3] channel-last -> out fp32 planar
 * [n, 3, h_out, w_out], ImageNet-normalised.  mean, std = HOST arrays of 3 floats.  Each source sample is normalised as
 * the depth data pipeline does it, three correctly rounded fp32 operations in this order: x / 255, - mean[c], / std[c];
 * the normalised samples are then resampled with align_corners=True.  The result is bit-identical to um_resize_bilinear of
 * the normalised planar frames, and at (h_out, w_out) = (h, w) it is exactly those frames.  No transpose.
 * Replaces the host-side ToTensor / Normalize (dataloader/depth/augmentation.py:30, 56-61) and the F.interpolate of
 * evaluate_depth.py:372-376. */
int um_frames_to_planar_normalized(const uint8_t* frames, float* out, int32_t n, int32_t h, int32_t w, int32_t h_out,
                                   int32_t w_out, const float* mean, const float* std, void* stream);

/* ---- ragged batches: images of different sizes packed back to back ------------------------------------------
 * Per-image geometry of the *_ragged entries, a DEVICE array of n items (read by the kernels, so a CUDA graph replay picks
 * up whatever the table holds at that time).  offset: where image i starts in the packed buffer, in elements of that
 * buffer (bytes for uint8 frames [h, w, 3]; floats for disparities [h, w], whose BGR pictures start at 3 * offset bytes);
 * (h, w): its size as stored; scale: used by um_resize_bilinear_ragged only; flags: UM_RAGGED_*, each entry names the ones
 * it reads and ignores the others.  An item with h or w outside 1..capacity, or
 * that does not fit in the packed buffer (numel / bytes arguments), is skipped: nothing of it is read or written.  Each
 * entry validates its scalar arguments before any CUDA call, launches a grid sized by the capacity (h_max, w_max) or the
 * uniform side, and never synchronises: graph-capturable.  n <= 65535. */
typedef struct um_ragged_item {
  int64_t offset;
  int32_t h, w;
  float scale;
  int32_t flags;
} um_ragged_item;
#define UM_RAGGED_FLIP_X 1   /* um_resize_bilinear_ragged: mirror the item's output horizontally */
/* A portrait item of the flow drivers, which run the model on the transposed (landscape) image (evaluate_flow.py:713-717,
 * :757-758).  um_frames_to_planar_ragged: the frame [h, w, 3] is read as its transpose [w, h, 3].
 * um_resize_bilinear_ragged: the item stored as [h, w] is the transpose of the (w, h) resize of the source. */
#define UM_RAGGED_TRANSPOSE 2

/* um_frames_to_planar_normalized per frame: frame i = DEVICE uint8 [h_i, w_i, 3] at frames + items[i].offset (frames_bytes
 * = size of the packed buffer) -> out fp32 planar [n, 3, h_out, w_out].  Image i is bit-identical to
 * um_frames_to_planar_normalized of frame i alone (the same device code: three correctly rounded fp32 operations per
 * sample, then the align-corners resample; a frame at the output size comes out as its normalised samples). */
int um_frames_to_planar_normalized_ragged(const uint8_t* frames, int64_t frames_bytes, const um_ragged_item* items, float* out,
                                          int32_t n, int32_t h_max, int32_t w_max, int32_t h_out, int32_t w_out,
                                          const float* mean, const float* std, void* stream);

/* um_frames_to_planar per frame: frame i = DEVICE uint8 [h_i, w_i, 3] at frames + items[i].offset (frames_bytes = size of the
 * packed buffer) -> out fp32 planar [n, 3, h_out, w_out] in [0, 255].  Image i is bit-identical to um_frames_to_planar of
 * frame i alone with transpose = (items[i].flags & UM_RAGGED_TRANSPOSE) (the same device code).  Replaces the host-side
 * conversion, transpose and F.interpolate of inference_flow (evaluate_flow.py:710-733) for pairs of different sizes. */
int um_frames_to_planar_ragged(const uint8_t* frames, int64_t frames_bytes, const um_ragged_item* items, float* out, int32_t n,
                               int32_t h_max, int32_t w_max, int32_t h_out, int32_t w_out, void* stream);

/* um_resize_bilinear per item: in = uniform planar [n, 1, h_in, w_in] fp32 -> item i at out + items[i].offset (out_numel
 * floats in all), size (h_i, w_i), multiplied by items[i].scale unless it is 1.0f, mirrored with UM_RAGGED_FLIP_X.  Item i is
 * bit-identical to um_resize_bilinear of image i alone with scale = &items[i].scale; an item at (h_in, w_in) without the flip
 * is copied as it is (what the stereo driver does with a disparity it does not resize, evaluate_stereo.py:813-836).
 * With UM_RAGGED_TRANSPOSE the item [h_i, w_i] is the transpose of um_resize_bilinear of image i to (w_i, h_i) (mirrored
 * before the transpose when both flags are set), and it is copied, transposed, when (w_i, h_i) = (h_in, w_in).
 * A flow batch [B, 2, H, W] is 2B images: pair i's u plane with scale = (float)(ori_w / size_w) and its v plane with
 * (float)(ori_h / size_h), packed back to back, give the planar flow [2, h_i, w_i] of evaluate_flow.py:750-758.
 * Replaces the resize back, disparity rescale and flip back of inference_stereo, and the resize back, flow rescale and
 * transpose back of inference_flow, for pairs of different sizes. */
int um_resize_bilinear_ragged(const float* in, float* out, int64_t out_numel, const um_ragged_item* items, int32_t n,
                              int32_t h_in, int32_t w_in, int32_t h_max, int32_t w_max, void* stream);

/* um_disparity_to_image per item: disparity i = fp32 [h_i, w_i] at disp + items[i].offset (numel floats in all) -> its BGR
 * picture at out + 3 * items[i].offset bytes, rows of 3 w_i bytes.  Picture i is bit-identical to um_disparity_to_image of
 * disparity i alone (NaN / constant / inf rule included).  minmax_scratch: DEVICE buffer of 2n words, reset inside the call.
 * Replaces vis_disparity on each predicted disparity of inference_stereo (evaluate_stereo.py:820-841). */
int um_disparity_to_image_ragged(const float* disp, int64_t numel, const um_ragged_item* items, uint8_t* out,
                                 float* minmax_scratch, int32_t n, int32_t h_max, int32_t w_max, void* stream);

/* um_flow_to_image per item: flow i = fp32 planar [2, h_i, w_i] at flow + flow_items[i].offset (offset in floats, flow_numel
 * floats in all) -> its RGB picture at out + picture_items[i].offset (offset in BYTES, out_bytes in all), rows of 3 w_i
 * bytes.  Picture i is bit-identical to um_flow_to_image of flow i alone (unknown-flow / NaN / all-zero rule included).
 * An item is skipped unless both of its descriptors fit and have the same (h, w).  max_scratch: DEVICE buffer of n words,
 * reset inside the call.  Replaces flow_to_image on each predicted flow of inference_flow (evaluate_flow.py:771, :784). */
int um_flow_to_image_ragged(const float* flow, int64_t flow_numel, const um_ragged_item* flow_items, uint8_t* out,
                            int64_t out_bytes, const um_ragged_item* picture_items, float* max_scratch, int32_t n,
                            int32_t h_max, int32_t w_max, void* stream);

/* um_fb_consistency per pair: flow_items and occ_items hold 2n items each, pair i's forward flow [2, h_i, w_i] (mask
 * [h_i, w_i]) at index i and its backward one at index n + i; offsets in floats into flow (flow_numel floats in all) and
 * occ (occ_numel).  The masks of pair i are bit-identical to um_fb_consistency of pair i alone.  A pair is skipped unless
 * its four items fit and have one size of at least 2 x 2 (what um_fb_consistency accepts).  Replaces
 * forward_backward_consistency_check on each pair of inference_flow, at its original size (evaluate_flow.py:789-792). */
int um_fb_consistency_ragged(const float* flow, int64_t flow_numel, const um_ragged_item* flow_items, float alpha, float beta,
                             float* occ, int64_t occ_numel, const um_ragged_item* occ_items, int32_t n, int32_t h_max,
                             int32_t w_max, void* stream);

/* ---- dense point tracks ----------------------------------------------------------------------------------------
 * Chains the forward flows of consecutive pairs from every pixel of a first frame (composition of flow_warp, geometry.py:65-72,
 * with the fwd_occ of forward_backward_consistency_check, :75-96, as visibility).  Coordinates are pixels (x, y) at the
 * flows' size.  State: pos [h, w, 2] (track positions) and vis [h, w] (uint8, 1 = visible), read and updated in place; the
 * caller starts them at pos(y, x) = (x, y), vis = 1.  For each flow t = 0..n-1 in order, F = flow[t] (planar [2, h, w]) and
 * O = occ[t] ([h, w]; occ NULL: O = 0, nothing occluded):
 *   d = bilinear(F, p), o = bilinear(O, p);  p = p + d;
 *   vis = vis && o < 0.5 && 0 <= p.x <= w-1 && 0 <= p.y <= h-1;
 *   pos_out[t] = p, vis_out[t] = vis   (pos_out [n, h, w, 2], vis_out [n, h, w]).
 * An invisible track stays invisible; its position is still advanced.  bilinear is bilinear_sample (geometry.py:41-62) in
 * pixel coordinates: align_corners=True, zero padding.  fp32 order of operations, every step rounded on its own (no FMA):
 *   x0 = floor(x), fx = x - x0 (exact), gx = 1 - fx, likewise y;  a corner outside [0, w-1] x [0, h-1] reads 0;
 *   bilinear = gy (gx v00 + fx v01) + fy (gx v10 + fx v11);  a track with x <= -1, x >= w, y <= -1, y >= h or a NaN
 *   coordinate samples 0 (it has no corner inside).
 * One thread per track, one launch for the n flows; no host synchronisation (graph-capturable).  pos and pos_out are 8-byte
 * aligned; the four state / output buffers do not overlap.  Frames of at least 2 x 2 (bilinear_sample divides by size - 1). */
int um_chain_tracks(const float* flow, const float* occ, int32_t n, int32_t h, int32_t w, float* pos, uint8_t* vis,
                    float* pos_out, uint8_t* vis_out, void* stream);

/* ---- query point tracks ----------------------------------------------------------------------------------------
 * Tracks nq query points through a clip of nt frames, each forward and backward in time from the frame it is given at (the
 * question TAP-Vid asks).  queries [nq, 3] = (t_q, y, x): t_q an integer frame index (stored as float), (x, y) pixels at the
 * flows' size, pixel centres at integers.  Tables: tracks [nq, nt, 2] (x, y) and visible [nq, nt] (uint8, 1 = visible),
 * row q holding query q's track in every frame.  Every step is um_chain_tracks's step with the same bilinear, the same fp32
 * order of operations and no FMA:
 *   frame t_q:          p = (x, y), visible;
 *   forward, t > t_q:   pair (t-1, t), F its forward flow, O its fwd_occ:   p_t = p_{t-1} + bilinear(F, p_{t-1}),
 *                       vis_t = vis_{t-1} && bilinear(O, p_{t-1}) < 0.5 && 0 <= p_t.x <= w-1 && 0 <= p_t.y <= h-1;
 *   backward, t < t_q:  pair (t, t+1), B its backward flow (frame t+1 -> t), Ob its bwd_occ:   p_t = p_{t+1} +
 *                       bilinear(B, p_{t+1}), vis_t = vis_{t+1} && bilinear(Ob, p_{t+1}) < 0.5 && p_t inside the frame.
 * An invisible track still moves.  A masks pointer of NULL means nothing is occluded.  So for a query at an integer pixel
 * the forward part is um_chain_tracks over the flows from pair t_q on, and the backward part um_chain_tracks over the
 * backward flows of pairs t_q-1, ..., 0 in that order, bit for bit.
 *
 * um_track_points_forward: the n forward flows [n, 2, h, w] and masks [n, h, w] of pairs t0 .. t0+n-1, frames t0+1 .. t0+n
 * of the table, which must exist (t0 + n < nt).  A stream is chained by launches over its pairs in order, the first at
 * t0 = 0, each at the previous t0 + n: a query joins at pair t_q from the query itself, and otherwise continues from the
 * state pos [nq, 2] / vis [nq] the previous launch left (read and written in place, never initialised by the caller).
 * Writes the table entries t > t_q it reaches; a query whose t_q is not an integer in [0, nt) is skipped.
 * um_track_points_backward: the n backward flows [n, 2, h, w] and masks [n, h, w] of pairs 0 .. n-1 (flow NULL when n = 0,
 * n < nt), in one launch; writes entries 0 .. t_q of every row.  A query it cannot serve (t_q not an integer in
 * [0, min(nt, n + 1))) gets NaN positions and visible = 0 in all nt entries.
 * One thread per query; no host synchronisation.  flow, occ and queries 4-byte aligned, pos and tracks 8-byte aligned; the
 * buffers a launch writes overlap nothing it reads or writes.  Frames of at least 2 x 2, nq >= 1. */
int um_track_points_forward(const float* flow, const float* occ, int32_t n, int32_t h, int32_t w, int32_t t0,
                            const float* queries, int32_t nq, int32_t nt, float* pos, uint8_t* vis, float* tracks,
                            uint8_t* visible, void* stream);
int um_track_points_backward(const float* flow, const float* occ, int32_t n, int32_t h, int32_t w, const float* queries,
                             int32_t nq, int32_t nt, float* tracks, uint8_t* visible, void* stream);

/* ---- multi-flow dense point tracks -----------------------------------------------------------------------------
 * Every pixel of a first frame tracked through a clip, each new frame t reached from k candidate source frames (e.g.
 * t-1, t-2, t-4, ... and frame 0: multi-flow tracking after MFT, Neoral, Serych and Matas, WACV 2024), keeping the most
 * certain visible candidate, so a point occluded for a while comes back through a longer flow.  Coordinates are pixels
 * (x, y) at the flows' size.  The state of every pixel p in frame s lives in one of r slots: pos [r, h, w, 2] (x, y),
 * sig [r, h, w] (accumulated uncertainty sigma^2) and vis [r, h, w] (uint8, 1 = visible); the caller starts frame 0's slot
 * at pos(y, x) = (x, y), sig = 0, vis = 1.
 * Per frame t = 0..n-1 of the launch, in order, candidate j = 0..k-1 (c = t k + j) is pair c: F = flow[c] (planar
 * [2, h, w], source -> frame), O = occ[c] (its fwd_occ, [h, w]) and E = err[c] (its fwd_err of um_fb_consistency_error),
 * and src[t][j] the slot of its source frame's state; an entry outside [0, r) is absent and its pair is not read.
 * From the source state (x_s, sigma2_s, v_s), with bilinear and its fp32 order of operations as for um_chain_tracks:
 *   d = bilinear(F, x_s), o = bilinear(O, x_s), e = bilinear(E, x_s);  x = x_s + d;  sigma2 = sigma2_s + e * e;
 *   valid = v_s && o < 0.5 && 0 <= x.x <= w-1 && 0 <= x.y <= h-1
 * (each + and * rounded on its own, no FMA; x and v are exactly um_chain_tracks's step).  The frame takes the valid
 * candidate of smallest sigma2, the first in j order on ties (a NaN never wins over an earlier candidate), visible; if no
 * candidate is valid, the present candidate of smallest sigma2 under the same rule, invisible.  A frame without a present
 * candidate is NaN, NaN, invisible.  The choice goes to tracks [n, h, w, 2], visible [n, h, w] and sigma [n, h, w], and
 * into slot dst[t] (no state is written when dst[t] is outside [0, r)).
 * src [n, k] and dst [n] are DEVICE int32 tables, read by the kernel, so a CUDA graph replay picks up whatever they hold.
 * One thread per pixel walks the n frames in order, and pixel p of every slot is touched by that thread only: a later frame
 * of the same launch may read the slot an earlier frame wrote, and then reads that frame's state.  Condition on the
 * tables: dst[t] is no slot that a candidate of frame t' >= t reads for a frame other than t, i.e. a launch never
 * overwrites a state one of its candidates still needs.  No host synchronisation (graph-capturable).  pos and tracks
 * 8-byte aligned, the other buffers 4-byte aligned (vis and visible bytes); the six state and output buffers overlap
 * nothing.  Frames of at least 2 x 2. */
int um_multi_flow_tracks(const float* flow, const float* occ, const float* err, const int32_t* src, const int32_t* dst,
                         int32_t n, int32_t k, int32_t h, int32_t w, int32_t r, float* pos, float* sig, uint8_t* vis,
                         float* tracks, uint8_t* visible, float* sigma, void* stream);

/* ---- stereo scene flow -------------------------------------------------------------------------------------------
 * The second disparity of scene flow (KITTI 2015's disp_1): the disparity at t+1 of the scene point seen at pixel p of the
 * left frame at t, stored in frame t's grid.  disp_next [B, h, w] is the disparity of left frame t+1 and flow [B, 2, h, w]
 * (planar) the optical flow from left frame t to left frame t+1, both contiguous at one size.  For pixel p = (x, y), in
 * fp32 with each operation rounded on its own (no FMA), (u, v) = flow[b, :, y, x]:
 *   q = (x + u, y + v);   in_frame[b, y, x] = 0 <= q.x <= w-1 && 0 <= q.y <= h-1   (uint8; a NaN coordinate gives 0);
 *   c = (fminf(fmaxf(q.x, 0), w-1), fminf(fmaxf(q.y, 0), h-1))   (a NaN coordinate clamps to 0, as fmaxf does);
 *   disp1[b, y, x] = bilinear(disp_next[b], c) with um_chain_tracks's bilinear and order of operations:
 *     x0 = floor(c.x), fx = c.x - x0 (exact), gx = 1 - fx, likewise y;  gy (gx v00 + fx v01) + fy (gx v10 + fx v11),
 *     a corner outside the frame (only ever at x0 + 1 = w or y0 + 1 = h, with weight 0) reads 0.
 * That is grid_sample(disp_next, q, mode='bilinear', padding_mode='border', align_corners=True).  Decision: disp1 is
 * dense.  A point that leaves the frame takes the nearest in-frame value rather than 0, because KITTI's disparity PNGs read
 * 0 as "no estimate", and a dense map is scored without the server's background interpolation; in_frame says which pixels
 * were sampled inside.  No occlusion handling: a point hidden at t+1 takes the disparity of whatever is in front of it.
 * One thread per pixel, no host synchronisation (graph-capturable).  disp1 and in_frame overlap nothing.  Frames of at
 * least 1 x 1, B <= 65535. */
int um_warp_disparity(const float* disp_next, const float* flow, float* disp1, uint8_t* in_frame, int32_t batch, int32_t h,
                      int32_t w, void* stream);

/* KITTI 2015 scene-flow statistics (the devkit's D1, D2, Fl and SF outliers) of a batch at ground-truth resolution, on
 * um_eval_stats's scaffold: UM_EVAL_PARTS CTAs per sample, each writing one partial row, then one ordered pass; no
 * floating-point atomics, bit-reproducible.  Counts are kept per thread in 32-bit integers and converted at the reduction.
 *   disp0, disp1: predictions [B, h, w]; flow: prediction [B, 2, h, w] (planar); all contiguous fp32;
 *   gt_*: HOST arrays of 2 device pointers, gt_*[s] for s = UM_SF_OCC (all pixels) and UM_SF_NOC (non-occluded): disparities [B, h, w] (> 0 = valid, KITTI's PNG / 256),
 *   flow [B, 2, h, w] and flow_valid [B, h, w] (>= 0.5 = valid); the UM_SF_NOC maps may all be NULL (that set then counts 0);
 *   obj_map [B, h, w] or NULL: != 0 is foreground, NULL makes every pixel background;
 *   scratch: DEVICE buffer of batch * UM_EVAL_PARTS * UM_SF_COLS doubles; out: DEVICE [batch, UM_SF_COLS] doubles.
 * Per pixel and set, with um_eval_stats's fp32 expressions:
 *   disparity (D1 on disp0, D2 on disp1): valid gt > 0, e = |gt - pred|, outlier e > 3 && e / gt > 0.05 (UM_EVS_D1);
 *   flow (Fl): valid flow_valid >= 0.5, epe = sqrt(du du + dv dv), mag likewise of the gt, outlier epe > 3 && epe / mag > 0.05
 *   (UM_EVF_OUTLIER);  SF: valid where all three are valid, an outlier where any of the three is.
 * Column of (set, region, metric, kind) = UM_SF_COL(s, r, m, k). */
#define UM_SF_OCC 0
#define UM_SF_NOC 1
#define UM_SF_BG 0
#define UM_SF_FG 1
#define UM_SF_D1 0
#define UM_SF_D2 1
#define UM_SF_FL 2
#define UM_SF_SF 3
#define UM_SF_N 0            /* valid pixels   */
#define UM_SF_OUTLIERS 1     /* their outliers */
#define UM_SF_COL(s, r, m, k) ((((s) * 2 + (r)) * 4 + (m)) * 2 + (k))
#define UM_SF_COLS 32
int um_scene_flow_stats(const float* disp0, const float* disp1, const float* flow, const float* const* gt_disp0,
                        const float* const* gt_disp1, const float* const* gt_flow, const float* const* gt_flow_valid,
                        const float* obj_map, int32_t batch, int32_t h, int32_t w, double* scratch, double* out,
                        void* stream);

/* ---- TSDF fusion of posed depth maps ---------------------------------------------------------------------------------
 * A dense volume of X x Y x Z voxels (x fastest, at most 2^31 - 1 voxels, N = X Y Z), 20 bytes per voxel in three
 * contiguous fp32 planes: tsdf [Z, Y, X], weight [Z, Y, X] and color [3, Z, Y, X] (R, G, B; channel offsets are 64-bit).
 * origin is a HOST array of 3 floats; the centre of voxel (i, j, k) is, per axis, p = fma(idx + 0.5f, voxel_size, origin)
 * (idx + 0.5f rounded first).  A zeroed volume is empty (weight 0 = never observed).
 *
 * Integration: depth [n, h, w] fp32 (metric z-depth), frames [n, h, w, 3] uint8 RGB at the same size, w2c [n, 3, 4] fp32
 * row-major world-to-camera matrices M, and a DEVICE int32 n_valid: only frames 0 .. min(max(n_valid, 0), n) - 1 are
 * fused, so one captured CUDA graph serves a short last step.  One thread per voxel walks those frames in order; per
 * frame, in fp32 with every operation rounded on its own (__fmaf_rn, __fdiv_rn, ...):
 *   c.x = fma(M02, p.z, fma(M01, p.y, fma(M00, p.x, M03))), likewise c.y (row 1) and c.z (row 2);  skip unless c.z > 0;
 *   u = fma(fx, c.x / c.z, cx),  v = fma(fy, c.y / c.z, cy);  xi = floor(u + 0.5f), yi = floor(v + 0.5f);
 *   skip unless 0 <= xi < w and 0 <= yi < h (a NaN is skipped);  d = depth[t, yi, xi];  skip unless d is finite and d > 0;
 *   sdf = d - c.z;  skip if sdf < -trunc;  f = fminf(1, sdf / trunc);
 *   W' = W + 1;  F' = fma(F, W, f) / W';  each colour channel C' = fma(C, W, frames[t, yi, xi, ch]) / W';  W = W'.
 * The voxel's state is read at its first update and written once after its last, so voxels no frame reaches move no
 * state bytes.  Because each voxel sees its frames in order, fusing frames in one launch or split over several gives the
 * same volume bit for bit.  No atomics, no host synchronisation (graph-capturable).  voxel_size and trunc > 0 and finite;
 * the volume planes overlap each other and the inputs nowhere; all fp32 buffers 4-byte aligned. */
#define UM_TSDF_THREADS 256
int um_tsdf_integrate(float* tsdf, float* weight, float* color, int32_t X, int32_t Y, int32_t Z, const float* origin,
                      float voxel_size, float trunc, const float* depth, const uint8_t* frames, const float* w2c, int32_t n,
                      int32_t h, int32_t w, float fx, float fy, float cx, float cy, const int32_t* n_valid, void* stream);

/* Offsets tables.  A count op (um_tsdf_surface_count, um_tsdf_mesh_count, um_cloud_down_sample_count, um_mesh_bin_count,
 * um_depth_points_count) takes its items in blocks of UM_TSDF_THREADS in item order and writes offsets [nb + 1] (DEVICE
 * int64, nb the number of blocks): offsets[b] the first output of block b, offsets[nb] the total, which the caller reads
 * to allocate the outputs.  It launches a count pass, then one CTA's ordered exclusive int64 scan of the block counts in
 * place.  Its fill op writes each item's outputs from its block's offset plus the outputs of the block's earlier items.
 * No atomics: the output is the same from run to run. */

/* Surface extraction: the zero-crossing vertices of marching cubes, as coloured points.  Each voxel owns its +x, +y and +z
 * edges that lie inside the grid; the edge from voxel 0 to voxel 1 emits a point iff weight0 > 0, weight1 > 0 and
 * (F0 < 0) != (F1 < 0).  With s = F0 / (F0 - F1) the point is voxel 0's centre with fma(s, voxel_size, p0) on the edge's
 * axis, and its colour per channel is __float2int_rn(fma(s, C1 - C0, C0)) clamped to 0..255.  Points are ordered by voxel
 * linear index, then edge axis x, y, z.
 * um_tsdf_surface_count writes the offsets table (see Offsets tables) of the points over the N voxels,
 * nb = ceil(N / UM_TSDF_THREADS), the total P; the caller allocates points [P, 3] fp32 and colors [P, 3] uint8, and
 * um_tsdf_surface_points (n_points = P) writes them, and with P = 0 launches nothing. */
int um_tsdf_surface_count(const float* tsdf, const float* weight, int32_t X, int32_t Y, int32_t Z, int64_t* offsets,
                          void* stream);
int um_tsdf_surface_points(const float* tsdf, const float* weight, const float* color, int32_t X, int32_t Y, int32_t Z,
                           const float* origin, float voxel_size, const int64_t* offsets, int64_t n_points, float* points,
                           uint8_t* colors, void* stream);

/* Mesh extraction: marching cubes' triangles over the same vertices, with per-vertex normals.
 * Cubes: cube (i, j, k) has voxel (i, j, k) as its low corner, for i < X-1, j < Y-1, k < Z-1, and emits triangles only when
 * all 8 corners have weight > 0.  Corner c = bx + 2 by + 4 bz; bit c of the cube's configuration is set when F(corner) < 0
 * (the sign predicate of the point extraction: F == 0 counts as outside).
 * Edges: edge e = 4 axis + b0 + 2 b1, where b0, b1 are the corner bits of the other two axes in increasing axis order, is
 * the `axis` edge owned by voxel (i, j, k) + (those bits), so its vertex is the point um_tsdf_surface_points emits for
 * that (voxel, axis): the mesh's vertices and colours are the point extraction's, bit for bit and in the same order.  A
 * vertex on an edge whose cubes all have an unobserved corner is kept; no face references it.
 * Triangles per configuration: unimatch_b200/csrc/um_mc_table.cuh, generated by um_mc_table.py (which states the rule):
 * the crossing edges of each cube face are joined by segments that depend only on that face's four signs (an ambiguous
 * face cuts each negative corner off), so neighbouring cubes meet without cracks; the segments are chained into loops and
 * each loop fanned from its lowest edge id, loops in order of their lowest edge id.  At most 5 triangles per cube, each
 * counter-clockwise seen from the F >= 0 (free-space) side.  Over observed cubes the mesh is closed (each edge in as many
 * faces one way as the other); where both cubes at an ambiguous face fan a diagonal between the same two of its crossings,
 * the two sheets touch along that edge.
 * Faces: int32 [T, 3] vertex indices, ordered by cube linear index, then table order.
 * Normals: fp32 [P, 3], from the TSDF gradient, in fp32 with every operation rounded on its own.  Per voxel v and axis,
 * with v- and v+ the voxel's neighbours on that axis, each counted only inside the grid and observed (weight > 0):
 *   g = (F(v+) - F(v-)) * 0.5f with both,  F(v+) - F(v) with only v+,  F(v) - F(v-) with only v-,  0 with neither.
 * The vertex on the edge from voxel 0 to voxel 1 (s as for its point): n = fma(s, g1 - g0, g0) per component,
 * l = sqrt(fma(n.z, n.z, fma(n.y, n.y, n.x * n.x))) (correctly rounded), normal = n / l, or (0, 0, 0) when l == 0.
 * um_tsdf_mesh_count writes face_offsets, the offsets table (see Offsets tables) of the triangles over the N cubes,
 * nb as um_tsdf_surface_count's, the total T.  um_tsdf_mesh takes both offset tables and both totals
 * (n_points = P, n_faces = T, each at most 2^31 - 1) and writes points [P, 3] fp32, colors [P, 3] uint8 (as
 * um_tsdf_surface_points), normals [P, 3] fp32 and faces [T, 3] int32, through first_vertex, caller-provided DEVICE scratch
 * of N int32 (each voxel's first point).  Two launches: the vertex pass, then the face pass (none with T = 0); with P = 0
 * nothing is launched.  No atomics, no host synchronisation (graph-capturable); the output is the same from run to run. */
int um_tsdf_mesh_count(const float* tsdf, const float* weight, int32_t X, int32_t Y, int32_t Z, int64_t* face_offsets,
                       void* stream);
int um_tsdf_mesh(const float* tsdf, const float* weight, const float* color, int32_t X, int32_t Y, int32_t Z,
                 const float* origin, float voxel_size, const int64_t* point_offsets, int64_t n_points,
                 const int64_t* face_offsets, int64_t n_faces, int32_t* first_vertex, float* points, uint8_t* colors,
                 float* normals, int32_t* faces, void* stream);

/* Ray casting: the depth, colour and normal images of the fused surface seen by n pinhole cameras of h x w pixels with
 * intrinsics fx, fy, cx, cy, from c2w [n, 3, 4] fp32 row-major camera-to-world rows M (DEVICE).  One thread per pixel
 * (x, y) of view v, in fp32 with every operation rounded on its own (__fmaf_rn, __fdiv_rn, ...):
 * Ray:  xc = (x - cx) / fx,  yc = (y - cy) / fy;  per axis a (x, y, z; origin o_a, voxel size vs, dims D_a):
 *   d_a = fma(M_a0, xc, fma(M_a1, yc, M_a2))  (world direction, camera z-component 1, not normalised),
 *   gd_a = d_a / vs,  go_a = (M_a3 - o_a) / vs - 0.5f;  the grid coordinate g_a(t) = fma(t, gd_a, go_a) puts voxel
 *   centres on the integers, and t is the camera z-depth of the point at g(t).
 * Range (slab test on the box of voxel centres, g_a in [0, D_a - 1]): t_lo = near, t_hi = far; per axis, if gd_a == 0 the
 *   ray misses unless 0 <= go_a <= D_a - 1, else t0 = -go_a / gd_a, t1 = (D_a - 1 - go_a) / gd_a,
 *   t_lo = fmaxf(t_lo, fminf(t0, t1)), t_hi = fminf(t_hi, fmaxf(t0, t1)).  The ray misses unless every gd_a and go_a is
 *   finite, t_lo <= t_hi, t_hi is finite and every D_a >= 2 (a volume with a dimension below 2 has no cell).
 * Sample at t: per axis g = fma(t, gd, go), i = clamp((int)floor(g), 0, D - 2), f = g - i.  Known iff all 8 voxels of the
 *   cell have weight > 0 (the TSDF values are read only then).  F is trilinear with lerp(f, a, b) = fma(f, b - a, a) over
 *   the corners c = bx + 2 by + 4 bz: along x (pairs 0-1, 2-3, 4-5, 6-7), then y, then z.  The sample is fine iff known and
 *   F < 1 (an unknown sample, F >= 1 and NaN are coarse).
 * March, with s_f = vs * 0.5f and s_c = trunc * 0.5f: A = the sample at t_a = t_lo; while t_a < t_hi:
 *   t_b = fminf(t_a + (A fine ? s_f : s_c), t_hi), and t_b = t_hi if that is not > t_a;  B = the sample at t_b;
 *   if A is coarse and B fine, the coarse step is taken back: t_b = fminf(t_a + s_f, t_hi) (t_hi if not > t_a), B = the
 *   sample there;  if A and B are known and (F_a < 0) != (F_b < 0) the march ends: a hit if F_b < 0 (F == 0 counts as
 *   outside, as in meshing), else a back face (a miss);  otherwise t_a = t_b, A = B.  t_a strictly increases and stays at
 *   most t_hi, so the loop ends; every pair of consecutive samples ending in a fine sample is at most s_f apart, so each
 *   sign change of F between known samples is bracketed by samples one fine step apart, at grazing angles too.
 * Hit: s = F_a / (F_a - F_b);  depth = fma(s, t_b - t_a, t_a);  colour per channel __float2int_rn(lerp(s, C_a, C_b))
 *   clamped to 0..255, C the trilinear colour at each sample;  n = lerp(s, G_a, G_b) per component, G the trilinear
 *   interpolation (same order) of um_tsdf_mesh's per-voxel gradient, l = sqrt(fma(n.z, n.z, fma(n.y, n.y, n.x * n.x))),
 *   normal = n / l (world coordinates, towards free space), (0, 0, 0) when l == 0.  A miss writes 0 to all three outputs.
 * Outputs: depth [n, h, w] fp32, rgb [n, h, w, 3] uint8, normal [n, h, w, 3] fp32, every pixel written.  near finite and
 * >= 0, far > near (+inf: the box alone limits the ray), voxel_size and trunc positive and finite, fx, fy finite and
 * nonzero, cx, cy finite, n <= 65535; the outputs overlap each other, the volume and c2w nowhere.  Blocks of 16 x 8
 * pixels; no atomics, no host synchronisation (graph-capturable). */
int um_tsdf_raycast(const float* tsdf, const float* weight, const float* color, int32_t X, int32_t Y, int32_t Z,
                    const float* origin, float voxel_size, float trunc, const float* c2w, int32_t n, int32_t h, int32_t w,
                    float fx, float fy, float cx, float cy, float near, float far, float* depth, uint8_t* rgb,
                    float* normal, void* stream);

/* ---- tracking a camera against the fused volume: point-to-plane ICP (KinectFusion, Newcombe et al., ISMAR 2011) ------
 * n frames (at most 65535), each a live depth map and an initial camera-to-world pose P_ref, are tracked independently
 * in the same launches.  fp32 operations are each rounded on their own (__fmaf_rn, __fdiv_rn, ...); fp64 operations are
 * __dmul_rn / __dadd_rn / __dsub_rn / __ddiv_rn / __dsqrt_rn, in the order written, except cos and sin (CUDA's).
 * Depth pyramid (um_icp_downsample): level l+1 of an h x w map has floor(h/2) x floor(w/2) pixels; pixel (x, y) reads
 *   the depths d0..d3 at (2x, 2y), (2x+1, 2y), (2x, 2y+1), (2x+1, 2y+1); a depth is valid iff finite and > 0.
 *   lo = the fminf of the valid ones in that order; out = the fp32 sum, in that order from 0, of the valid d with
 *   d - lo <= trunc, divided by their count (a float); 0 if none is valid.  The level's intrinsics are fx/2, fy/2,
 *   (cx - 0.5f)/2 and (cy - 0.5f)/2 in fp32 (pixel x is centred at x on every level), computed by the caller.
 * Live normals (um_icp_normals, written to a buffer [n, h, w, 3]): the vertex of depth d at pixel (x, y) is
 *   v = (d * ((x - cx) / fx), d * ((y - cy) / fy), d).  With e1 = v(x+1, y) - v and e2 = v(x, y+1) - v (per component),
 *   c_a = e1_b * e2_e - e1_e * e2_b for (a, b, e) = (x, y, z), (y, z, x), (z, x, y); l = sqrt(fma(c.z, c.z, fma(c.y, c.y,
 *   c.x * c.x))), facing = fma(c.z, v.z, fma(c.y, v.y, c.x * v.x)); normal = c / (facing > 0 ? -l : l), so that n.v <= 0.
 *   0 where x + 1 = w, y + 1 = h, one of the three depths is invalid, or l is 0 or not finite.
 * Model maps: um_tsdf_raycast at the level's intrinsics from c2w_ref, the fp32 rows of P_ref, unchanged.  A model pixel is
 *   valid iff its depth D > 0 and its normal m is not (0, 0, 0).
 * State (um_icp_init; DEVICE fp64 [n, UM_ICP_STATE]): [0, 12) the estimate T = (R | t), [12, 24) P_ref, both [3, 4]
 *   row-major camera-to-world; [24] the number of degenerate recorded solves.  Init, per frame f < n_valid:
 *   P_ref = C * P (rows i < 3: (C_i0 P_0j + C_i1 P_1j) + C_i2 P_2j, plus C_i3 when j = 3) with the DEVICE fp64 [4, 4]
 *   correction C, or P itself when C is NULL; T = P_ref; state[24] = 0; c2w_ref = (float)P_ref rows; w2c_ref = the rigid
 *   inverse of P_ref: (R^T, -((R_0i t_0 + R_1i t_1) + R_2i t_2)) in fp64, each entry rounded to fp32.  poses: fp64
 *   [n, 4, 4] row-major (the last row is not read).
 * Association (um_icp_reduce), one thread per live pixel in 16 x 8 tiles, at the current T (rounded to fp32 rows):
 *   skip unless d is valid and the live normal n is not 0;  p_a = fma(T_a2, v.z, fma(T_a1, v.y, fma(T_a0, v.x, T_a3))),
 *   n_w,a = fma(T_a2, n.z, fma(T_a1, n.y, T_a0 * n.x));  c = w2c_ref applied to p exactly as um_tsdf_integrate projects
 *   a voxel, and its nearest pixel (xi, yi) by integration's rule (c.z > 0, floor(u + 0.5f) inside the frame);  skip
 *   unless the model pixel there is valid;  with xc = (xi - cx) / fx, yc = (yi - cy) / fy and M = c2w_ref:
 *   dir_a = fma(M_a0, xc, fma(M_a1, yc, M_a2)) (the ray cast's), q_a = fma(D, dir_a, M_a3), e = p - q, pc = p - M_.3;
 *   an inlier iff sqrt(fma(e.z, e.z, fma(e.y, e.y, e.x * e.x))) <= max_distance and fma(n_w.z, m.z, fma(n_w.y, m.y,
 *   n_w.x * m.x)) >= cos_max_angle;  r = fma(m.z, e.z, fma(m.y, e.y, m.x * e.x));  a = (pc x m (as c above), m), the
 *   Jacobian of r for dT applied on the left about the reference centre.
 *   Terms (fp32 products, then exact conversion to fp64; 0 unless an inlier): k < 21 the upper triangle of a a^T row by
 *   row (a_0 a_0 .. a_0 a_5, a_1 a_1, ..), 21 + i a_i r, 27 r r, 28 the inlier count (1), 29 the valid live pixel count
 *   (1 for every pixel with valid d and n, inlier or not).  Sums, no atomics (the same result from run to run): per warp
 *   v += shfl_down(v, o) for o = 16, 8, 4, 2, 1 (lane 0's: pixels outside the frame add 0), then the block's 4 warps in
 *   order; partials [n, nb, UM_ICP_TERMS] fp64, nb = ceil(w/16) ceil(h/8), block b = by ceil(w/16) + bx.  um_icp_solve and
 *   um_icp_accept sum a frame's partials with one warp of 32 lanes per term: lane l adds blocks l, l + 32, l + 64, ...
 *   in order from 0.0, then v += shfl_down(v, o) for o = 16, 8, 4, 2, 1 gives lane 0 the sum.
 * Solve (um_icp_solve, one block per frame): A (6 x 6, symmetric) and b from the sums.  Degenerate unless inliers >=
 *   min_inliers and every Cholesky pivot of the Jacobi-scaled system is >= min_pivot (a NaN fails).  s_i = 1/sqrt(A_ii),
 *   or 1 where A_ii is not > 0 (an unknown no residual constrains keeps its zero pivot);
 *   Ahat_ij = (A_ij s_i) s_j;  for j = 0..5: pivot = Ahat_jj - L_j0^2 - .. - L_j,j-1^2 (subtracted in order), L_jj =
 *   sqrt(pivot), L_ij = (Ahat_ij - L_i0 L_j0 - ..) / L_jj;  L z = -(b_i s_i), L^T y = z (back substitution from i = 5,
 *   k ascending), x_i = y_i s_i.  A degenerate solve leaves T unchanged and, with `record` (the finest level), adds 1 to
 *   state[24].  Otherwise x = (w, tau): th = sqrt((w0^2 + w1^2) + w2^2); dR = I if th == 0, else with k = w / th,
 *   dR_ij = ((i == j ? cos th : 0) + sin th [k]x_ij) + ((1 - cos th) k_i) k_j;  R <- dR R, t <- ((dR (t - c)) + c) + tau
 *   with c = P_ref's translation (matrix products summed (x0 + x1) + x2).
 * Schedule (the caller's): for each level, coarse to fine, a fixed number of (um_icp_reduce, um_icp_solve) iterations;
 *   fixed counts keep the launch sequence static, so it can be captured in a CUDA graph.
 * Acceptance (um_icp_accept, after one more um_icp_reduce at level 0): tracked iff state[24] == 0 and inliers >=
 *   min_inlier_fraction * valid (fp64).  A frame that is not tracked gets T = P_ref back.  Outputs: pose_out fp32
 *   [n, 4, 4] ((float)T, last row 0 0 0 1), tracked uint8 [n], inliers int64 [n], rmse fp32 [n] ((float)sqrt(sum r^2 /
 *   inliers), 0 without inliers) and w2c fp32 [n, 3, 4] (T's rigid inverse, as init's), the rows um_tsdf_integrate reads.
 *   With a correction (n == 1, poses given), a tracked frame sets C = T P^-1, P^-1 = (R_P^T, -R_P^T t_P) in fp64 (rows
 *   i < 3 as in init); a frame that is not tracked leaves C as it is.
 * Every loop has a fixed trip count.  n_valid (DEVICE int32): frames >= min(max(n_valid, 0), n) are untouched by init,
 * reduce, solve and accept, so one captured graph serves a short last step.  Pointers are fp32 unless stated; no output
 * overlaps an input or another output. */
#define UM_ICP_TERMS 30
#define UM_ICP_STATE 32
int um_icp_downsample(const float* src, float* dst, int32_t n, int32_t h, int32_t w, float trunc, void* stream);
int um_icp_normals(const float* depth, float* normal, int32_t n, int32_t h, int32_t w, float fx, float fy, float cx,
                   float cy, void* stream);
int um_icp_init(const double* poses, const double* correction, int32_t n, const int32_t* n_valid, double* state,
                float* c2w, float* w2c, void* stream);
int um_icp_reduce(const float* depth, const float* live_normal, const float* model_depth, const float* model_normal,
                  const double* state, const float* c2w, const float* w2c, int32_t n, int32_t h, int32_t w, float fx,
                  float fy, float cx, float cy, float max_distance, float cos_max_angle, const int32_t* n_valid,
                  double* partials, void* stream);
int um_icp_solve(const double* partials, int32_t nb, int32_t n, const int32_t* n_valid, double min_inliers,
                 double min_pivot, int32_t record, double* state, void* stream);
int um_icp_accept(const double* partials, int32_t nb, int32_t n, const int32_t* n_valid, double min_inlier_fraction,
                  const double* poses, double* correction, double* state, float* pose_out, uint8_t* tracked,
                  int64_t* inliers, float* rmse, float* w2c, void* stream);

/* ---- point clouds: exact nearest neighbours, voxel down-sampling and the 3D metrics of a reconstruction -------------
 * Points are fp32 [n, 3] (x, y, z), at most 2^31 - 1 per set.  fp64 operations are __dsub_rn / __ddiv_rn / ... in the
 * order written.
 * Grid (origin o, cell size c > 0, dims g[3] >= 1, all fp64 / int32 by value): the cell coordinate of a point along axis a
 *   is t_a = ((double)p_a - o_a) / c, its cell k_a = floor(t_a) clamped to [0, g_a - 1], and its key
 *   (k_z * g_y + k_y) * g_x + k_x (int64, x fastest).  um_cloud_keys writes the keys.
 * Table (um_cloud_ranges): given the keys sorted stably with their input positions (order), start[c] / end[c] (int32
 *   [g_x g_y g_z], zeroed by the entry) are the first and one-past-last sorted positions of cell c (0 and 0 for an empty
 *   cell; keys outside the table are not entered), and sorted[i] = (x, y, z, bits of (int32) order[i]) fp32 [n, 4].
 * Down-sampling (Open3D's VoxelDownSample): with v the voxel size, o = min_bound - v / 2 in fp64 (min_bound the set's
 *   per-axis minimum) and g_a = floor((max_bound_a - o_a) / v) + 1 computed as t is, every point lies in the grid, so the
 *   clamp never applies.  um_cloud_down_sample_count writes the offsets table (see Offsets tables) of the
 *   runs of equal keys over the n sorted positions a run can start at, nb = ceil(n / 256), the total M.
 *   um_cloud_down_sample: run m (in key order) writes out[m] = (float)(s / count) per axis, s the fp64 sum from 0.0 of
 *   (double)p over the run in sorted order, which a stable sort makes the input order.
 * Nearest neighbour (um_cloud_nearest, one query q per thread) over the table of an indexed set P whose grid box holds
 *   it (o at or below its minimum, g_a c at or above its extent): dx = q.x - p.x, dy, dz likewise (fp32), s =
 *   fmaf(dz, dz, fmaf(dy, dy, dx * dx)); the neighbour is the p of least s, ties to the least input index; distance =
 *   sqrtf(s) correctly rounded, index int64.  This equals a brute-force fp32 scan bit for bit whatever c is.
 *   Search: cells of Chebyshev rings r = 0, 1, ... around the query's clamped cell j, clamped to the table.  Per axis the
 *   gap of cell k is G_a(k) = max(0, max(k - t_a, t_a - (k + 1), 0) - (2^-20 + 2^-45 |t_a|)) * c (fp64).
 *   Proof that a skipped cell cannot hold p with s <= best: a point of cell k has exact cell coordinate T in
 *   [k - 2^-29, k + 1 + 2^-29] (two fp64 roundings of a value below 2^22 cells, the box holding the set); the query's
 *   t_a = ((double)q_a - o_a) * rcp(c) (rcp correctly rounded: three roundings) is within 2^-51 |t| of its exact value, and the gap's own rounding is below 2^-31 + 2^-53 |t| cells, so the exact
 *   |q_a - p_a| >= G_a(k).  The fp32 s is at least (1 - 5 * 2^-24) times the exact squared distance less 6 * 2^-150 (five
 *   roundings, each within 2^-24 relative or 2^-150 absolute).  So a region whose fp64 bound B = sum of G_a^2 satisfies
 *   B * (1 - 2^-20) - 2^-140 > best (the fp64 rounding of B is below 2^-50 relative) holds no p with s <= best.
 *   A cell is skipped when its own B passes that test; the search stops before ring r when the bound of every cell at
 *   Chebyshev distance >= r, min over axes a and sides +-1 with j_a +- r inside the table of G_a(j_a +- r)^2 + the
 *   other two axes' G_b(j_b)^2 (G is monotone away from j and least at j), passes it, or when no such side is left (the
 *   rings covered the table).  A query outside the box starts from its nearest box cell; its t carries its distance.
 *   With distance / index, writes them [nq]; with partial_sum / partial_count (fp64 / int64 [ceil(nq / 256)]) instead,
 *   per block of 256 queries the sum of (double)d (per warp a shfl_down tree 16, 8, 4, 2, 1 from lane 0, then the 8
 *   warps in order) and the count of d < threshold (fp32, strict).
 * Stats (um_cloud_stats, one warp): lane l adds the partials of blocks l, l + 32, ... in order from 0.0, then a
 *   shfl_down tree (16, 8, 4, 2, 1); out[0] = the sum of d, out[1] = the count as a double (exact).  No atomics
 *   anywhere: every result is the same from run to run.
 * Every pointer is DEVICE memory; no output overlaps an input or another output. */
int um_cloud_keys(const float* points, int64_t n, double ox, double oy, double oz, double cell, int32_t gx, int32_t gy,
                  int32_t gz, int64_t* keys, void* stream);
int um_cloud_ranges(const int64_t* sorted_keys, const int64_t* order, const float* points, int64_t n, int32_t gx,
                    int32_t gy, int32_t gz, int32_t* start, int32_t* end, float* sorted_points, void* stream);
int um_cloud_down_sample_count(const int64_t* sorted_keys, int64_t n, int64_t* offsets, void* stream);
int um_cloud_down_sample(const int64_t* sorted_keys, const int64_t* order, const float* points, int64_t n,
                         const int64_t* offsets, int64_t m, float* out, void* stream);
int um_cloud_nearest(const float* queries, int64_t nq, const float* sorted_points, const int32_t* start,
                     const int32_t* end, int64_t n, double ox, double oy, double oz, double cell, int32_t gx, int32_t gy,
                     int32_t gz, float threshold, float* distance, int64_t* index, double* partial_sum,
                     int64_t* partial_count, void* stream);
int um_cloud_stats(const double* partial_sum, const int64_t* partial_count, int64_t nb, double* out, void* stream);

/* ---- triangle meshes: rasterisation, visibility of points and the 2D depth metrics ----------------------------------
 * A mesh is points fp32 [P, 3] and faces int32 [T, 3] (indices in [0, P), at most 2^31 - 1 faces), seen by n <= 65535
 * pinhole cameras of h x w pixels (h w <= 2^31 - 1), intrinsics fx, fy (finite, nonzero), cx, cy (finite), through the
 * fp32 world-to-camera rows w2c [n, 3, 4] (row-major, as um_tsdf_integrate reads them); near finite and > 0, far > near
 * (+inf: no limit).  fp32 operations are each rounded on their own (__fmaf_rn, __fdiv_rn, ...), fp64 ones are __dadd_rn,
 * __dsub_rn, __dmul_rn, __ddiv_rn, floor and ceil, in the order written.
 * Per view and pixel (x, y), in fp32:
 *   xc = (x - cx) / fx, yc = (y - cy) / fy: the ray through the pixel centre along d = (xc, yc, 1) in camera coordinates
 *   (um_tsdf_raycast's convention); its parameter t along d is the camera z-depth.
 *   Vertex V of point p: V.x = fma(M02, p.z, fma(M01, p.y, fma(M00, p.x, M03))), likewise V.y (row 1) and V.z (row 2).
 *   Cross product a x b = (a.y b.z - a.z b.y, a.z b.x - a.x b.z, a.x b.y - a.y b.x), each product rounded, then the
 *   difference.  Face (i0, i1, i2) with vertices A, B, C has edges AB (i0 -> i1), BC (i1 -> i2) and CA (i2 -> i0); the
 *   edge i -> j has the canonical cross product K = V_lo x V_hi (lo, hi = i, j in ascending order) times +1 if i <= j,
 *   else -1, so two faces that share an edge get exactly opposite edge values (the rasteriser is watertight by
 *   construction).  E = fma(K.x, xc, fma(K.y, yc, K.z)) per edge (K the signed product).
 *   Coverage: E_AB, E_BC, E_CA all >= 0 or all <= 0, and S = (E_AB + E_BC) + E_CA != 0.  Faces are two-sided (no
 *   culling).  A face whose vertices coincide in camera space (a repeated index included) has S = 0 exactly and is never
 *   hit.  A hit on the line of the ray behind the camera has t < 0 and fails the depth test.
 *   Depth: det = fma(A.z, K_BC.z, fma(A.y, K_BC.y, A.x * K_BC.x)), t = det / S; a hit iff t is finite and
 *   near <= t <= far.  The winner is the hit of least t; among equal t the least face index (a strict < over the
 *   faces in ascending index).
 *   Colour (when colors, uint8 [P, 3], is given): bA = E_BC / S, bB = E_CA / S, bC = E_AB / S (the 3D barycentrics of
 *   the hit point, so perspective-correct); per channel fma(bC, col_C, fma(bB, col_B, bA * col_A)), __float2int_rn,
 *   clamped to 0..255.
 *   Outputs: depth fp32 [n, h, w] (t, 0 for a miss), face int32 [n, h, w] (-1 for a miss), rgb uint8 [n, h, w, 3] (0 for
 *   a miss; optional).
 * Rectangle (part of the definition: a face covers only the pixels of its rectangle), per (view, face) in fp64:
 *   the vertices c = ((M_r0 p.x + M_r1 p.y) + M_r2 p.z) + M_r3 per row r (the fp32 entries and coordinates converted
 *   exactly);  none if every vertex has c.z < near or every vertex has c.z > far;  else the triangle clipped to
 *   c.z >= near: for each edge P -> Q (AB, BC, CA) keep P if P.z >= near, and if exactly one of P, Q has z >= near add
 *   (P.x + s (Q.x - P.x), P.y + s (Q.y - P.y), near) with s = (near - P.z) / (Q.z - P.z);  each kept point projects to
 *   u = fx (x / z) + cx, v = fy (y / z) + cy;  the rectangle is x in [floor(min u) - 1, ceil(max u) + 1] and y in
 *   [floor(min v) - 1, ceil(max v) + 1] clamped to the frame (none if that is empty or a bound is NaN).  The exact hit
 *   point of a ray with t >= near lies in the clipped triangle, so the rectangle holds every pixel whose exact ray hits
 *   it; the 1-pixel margin absorbs the fp32 rounding of coverage and depth for the geometry tested
 *   (tests/test_raster_cpu.py shows that dropping it changes no output there), but it is not proved for arbitrarily
 *   degenerate geometry (slivers, vertices at extreme magnitudes, faces grazing the near plane).
 * Launches (16 x 16 pixel tiles, tiles = ceil(h/16) ceil(w/16) per view):
 *   um_mesh_bin_count writes the offsets table (see Offsets tables) of the tiles the faces' rectangles
 *   touch, over the (view, face) pairs in blocks of 256 faces of one view, view-major: nb = n ceil(T/256), the total E.
 *   um_mesh_bin (E entries): for each (view, face) in that order, per touched tile row by row, keys[e] = view tiles +
 *   tile (int64) and values[e] = face << 16 | (x0 | x1 << 4 | y0 << 8 | y1 << 12), the rectangle within the tile.
 *   The caller sorts keys stably with their positions (order), so each tile's entries stay in ascending face order.
 *   um_mesh_ranges: start / end int32 [n tiles] (zeroed by the entry) hold the first and one-past-last sorted position
 *   of each tile's entries.
 *   um_mesh_raster: one CTA per (tile, view) and one thread per pixel; the entries values[order[e]] of the tile are
 *   staged 256 at a time in shared memory (the signed canonical cross products, det, face and rectangle), and each thread
 *   walks them in order.  Every pixel is written.
 *   No atomics anywhere: every output is the same from run to run.
 * Visibility (um_visible_points, one thread per point, views in order): the point is transformed and projected exactly as
 *   um_tsdf_integrate projects a voxel centre (c.z > 0, nearest pixel floor(u + 0.5f) inside the frame); view t sees it
 *   iff the depth D = depth[t, yi, xi] is finite, D > 0 and c.z <= D + tolerance (fp32).  visible[i] (uint8) = 1 iff some
 *   view sees point i.
 * Depth metrics (um_depth_metrics) of pred and gt fp32 [n, h, w]: a pixel is valid iff p is finite and > 0, masked iff
 *   valid and g finite with 0 < g < max_depth.  Over masked pixels, with fp64 d = (double)p - (double)g: terms 0 count,
 *   1 |d|, 2 |d| / g, 3 (d d) / g, 4 d d, 5 (log p - log g)^2 (CUDA's fp64 log of the fp32 values), 6..8 the count of
 *   max(g / p, p / g) (fp32, correctly rounded divisions) < 1.25, 1.5625, 1.953125; term 9 the count of valid pixels
 *   (masked or not).  Per block of 256 pixels of a frame, per term a shfl_down tree (16, 8, 4, 2, 1) per warp, then the
 *   8 warps in order: partials fp64 [n, nb, UM_DEPTH_METRIC_TERMS], nb = ceil(h w / 256); then one warp per (frame,
 *   term): lane l adds blocks l, l + 32, ... in order from 0.0, then a shfl_down tree: out fp64 [n, UM_DEPTH_METRIC_TERMS].
 * Every pointer is DEVICE memory; no output overlaps an input or another output. */
#define UM_DEPTH_METRIC_TERMS 10
int um_mesh_bin_count(const float* points, int64_t n_points, const int32_t* faces, int64_t n_faces, const float* w2c,
                      int32_t n, int32_t h, int32_t w, float fx, float fy, float cx, float cy, float near, float far,
                      int64_t* offsets, void* stream);
int um_mesh_bin(const float* points, int64_t n_points, const int32_t* faces, int64_t n_faces, const float* w2c, int32_t n,
                int32_t h, int32_t w, float fx, float fy, float cx, float cy, float near, float far,
                const int64_t* offsets, int64_t n_entries, int64_t* keys, int64_t* values, void* stream);
int um_mesh_ranges(const int64_t* sorted_keys, int64_t n_entries, int32_t n, int32_t h, int32_t w, int32_t* start,
                   int32_t* end, void* stream);
int um_mesh_raster(const float* points, int64_t n_points, const int32_t* faces, int64_t n_faces, const uint8_t* colors,
                   const float* w2c, int32_t n, int32_t h, int32_t w, float fx, float fy, float cx, float cy, float near,
                   float far, const int64_t* order, const int64_t* values, int64_t n_entries, const int32_t* start,
                   const int32_t* end, float* depth, int32_t* face, uint8_t* rgb, void* stream);
int um_visible_points(const float* points, int64_t n_points, const float* depth, int32_t n, int32_t h, int32_t w,
                      const float* w2c, float fx, float fy, float cx, float cy, float tolerance, uint8_t* visible,
                      void* stream);
int um_depth_metrics(const float* pred, const float* gt, int32_t n, int32_t h, int32_t w, float max_depth,
                     double* partials, double* out, void* stream);

/* ---- multi-view geometric consistency of depth maps, and valid depths as coloured world points ---------------------
 * n depth maps depth fp32 [n, h, w] of one frame size with one pinhole camera fx, fy (finite, nonzero), cx, cy (finite);
 * camera-to-world rows c2w and world-to-camera rows w2c fp32 [n, 3, 4] (row-major, as um_tsdf_raycast and
 * um_tsdf_integrate read them).  A depth is valid iff it is finite and > 0.  fp32 operations are each rounded on their own
 * (__fmaf_rn, __fdiv_rn, __fsqrt_rn, ...), in the order written.  Rows M applied to a point p:
 *   M p = (fma(M02, p.z, fma(M01, p.y, fma(M00, p.x, M03))), likewise rows 1 and 2).
 * Back-projection of pixel coordinates (u, v) at depth z: B(u, v, z) = ((u - cx) / fx * z, (v - cy) / fy * z, z), so pixel
 * (x, y) is the ray through its centre (um_tsdf_raycast's and um_mesh_raster's convention).
 * Consistency (um_depth_consistency): refs int32 [R] are the reference maps and sources int32 [R, S] their sources in
 * order; an entry outside [0, n) is "no source" (and a reference outside [0, n) has no valid depth), so no table reads out
 * of bounds.  One thread per reference pixel (x, y) of reference r with d = depth[r, y, x]; if d is valid, per source s:
 *   c = w2c[s] (c2w[r] B(x, y, d));  the source does not count unless c.z > 0;
 *   u = fma(fx, c.x / c.z, cx), v = fma(fy, c.y / c.z, cy);  it does not count unless 0 <= u <= w - 1 and
 *   0 <= v <= h - 1 (a NaN does not count);
 *   x0 = floor(u), y0 = floor(v), x1 = min(x0 + 1, w - 1), y1 = min(y0 + 1, h - 1), ax = u - x0, ay = v - y0 (exact);
 *   the taps D00 = depth[s, y0, x0], D01 = [s, y0, x1], D10 = [s, y1, x0], D11 = [s, y1, x1] must all be valid;
 *   top = fma(ax, D01 - D00, D00), bot = fma(ax, D11 - D10, D10), ds = fma(ay, bot - top, top)  (bilinear);
 *   c' = w2c[r] (c2w[s] B(u, v, ds));  it does not count unless c'.z > 0;
 *   u' = fma(fx, c'.x / c'.z, cx), v' = fma(fy, c'.y / c'.z, cy), dx = u' - x, dy = v' - y;
 *   it is consistent iff sqrt(fma(dy, dy, dx * dx)) < max_pixel and |c'.z - d| / d < max_relative.
 * views uint8 [R, h, w] = the number of consistent sources (0 for an invalid d); out fp32 [R, h, w] = d where
 * views >= min_views, else 0.  S 1 .. 255, min_views 1 .. S, max_pixel and max_relative positive and finite, R 1 .. 65535.
 * No atomics, no host synchronisation (graph-capturable); the same output from run to run.
 * Points (um_depth_points_count, um_depth_points): every valid depth d = depth[t, y, x] gives the world point
 * c2w[t] B(x, y, d) and the colour frames[t, y, x] (uint8 [n, h, w, 3]), ordered by frame, then row-major pixel.
 * um_depth_points_count writes the offsets table (see Offsets tables) of the points over the n h w pixels
 * (frame-major), nb = ceil(n h w / 256), the total P; the caller allocates points fp32 [P, 3] and colors uint8 [P, 3]
 * (P <= 2^31 - 1), and um_depth_points (n_points = P) writes them, and with P = 0 launches nothing.  n 1 .. 65535, h w <= 2^31 - 1, n h w <= 2^39.
 * Every pointer is DEVICE memory; no output overlaps an input or another output. */
int um_depth_consistency(const float* depth, int32_t n, int32_t h, int32_t w, float fx, float fy, float cx, float cy,
                         const float* c2w, const float* w2c, const int32_t* refs, int32_t r, const int32_t* sources,
                         int32_t s, float max_pixel, float max_relative, int32_t min_views, uint8_t* views, float* out,
                         void* stream);
int um_depth_points_count(const float* depth, int32_t n, int32_t h, int32_t w, int64_t* offsets, void* stream);
int um_depth_points(const float* depth, const uint8_t* frames, int32_t n, int32_t h, int32_t w, float fx, float fy,
                    float cx, float cy, const float* c2w, const int64_t* offsets, int64_t n_points, float* points,
                    uint8_t* colors, void* stream);

/* Middlebury colour coding of n planar flows [n, 2, h, w] -> uint8 RGB pictures: pixel (y, x) of image i is written at
 * out + i * image_stride + y * row_stride + 3 * x (strides in BYTES; row_stride >= 3w), so a picture can land inside a larger
 * frame (e.g. next to the video frame).  Per image: |u| or |v| > 1e7 are unknown (black, excluded from the maximum), the
 * maximum radius is a float32 reduction, the rest float64, as numpy evaluates the reference; zero flow is white.
 * max_scratch: DEVICE buffer of n floats (receives the per-image maximum radius).  n <= 65535.
 * Replaces flow_to_image (utils/flow_viz.py:240-275; called at evaluate_flow.py:768 for videos). */
int um_flow_to_image(const float* flow, uint8_t* out, int64_t row_stride, int64_t image_stride, float* max_scratch,
                     int32_t n, int32_t h, int32_t w, void* stream);

/* Disparity colouring of n contiguous fp32 disparities [n, h, w] -> uint8 BGR pictures (cv2's channel order), written at
 * out + i * image_stride + y * row_stride + 3 * x (strides in BYTES, as for um_flow_to_image).  Per image, as numpy
 * evaluates vis_disparity on float32: g = uint8(((d - min) / (max - min)) * 255), each operation a correctly rounded fp32
 * operation, truncated; the pixel is cv2's COLORMAP_INFERNO table at g.  A NaN normalised value gives g = 0, so a constant
 * image, a NaN anywhere in the image or +-inf in it paints the whole image INFERNO[0].
 * minmax_scratch: DEVICE buffer of 2n words (the per-image min / max keys; reset inside the call, graph-capturable).
 * n <= 65535.
 * Replaces vis_disparity (utils/visualization.py:11-16), called on every predicted disparity by inference_stereo
 * (evaluate_stereo.py:820-841). */
int um_disparity_to_image(const float* disp, uint8_t* out, int64_t row_stride, int64_t image_stride, float* minmax_scratch,
                          int32_t n, int32_t h, int32_t w, void* stream);

/* Depth colouring of n contiguous fp32 depths [n, h, w] -> uint8 RGB pictures (PIL's channel order) of the inverse depth,
 * written at out + i * image_stride + y * row_stride + 3 * x (strides in BYTES, as for um_flow_to_image).  Per image, as
 * numpy 1.19 / matplotlib 3.5.1 evaluate viz_depth_tensor(1. / depth): inv = 1 / depth (correctly rounded fp32); vmin =
 * min(inv); vmax = a * (1 - g) + b * g in float64, with a, b the exact order statistics of inv at ranks k and
 * min(k + 1, N - 1), k = floor(0.95 * (N - 1)) and g its fraction (np.percentile(inv, 95)); t = (inv - vmin) /
 * fp32(vmax - vmin) in fp32; the pixel is uint8(floor(255 * plasma[c])) at index trunc(256 * t), clamped to 0..255, and
 * black for a NaN t.  vmax <= vmin gives index 0 everywhere; a NaN in the image, or a NaN vmax, paints it all black.
 * scratch: DEVICE buffer of 2056 * n 32-bit words (per image four 512-bin radix-select histograms and the selection
 * state; reset inside the call).  One memset and nine kernels whatever the data, no host synchronisation: graph-capturable.
 * n <= 65535.
 * Replaces viz_depth_tensor (utils/visualization.py:92-107), called on every predicted depth (and the backward one with
 * pred_bidir_depth) by inference_depth (evaluate_depth.py:403-417). */
int um_depth_to_image(const float* depth, uint8_t* out, int64_t row_stride, int64_t image_stride, void* scratch, int32_t n,
                      int32_t h, int32_t w, void* stream);

/* um_depth_to_image per item: depth i = fp32 [h_i, w_i] at depth + items[i].offset (numel floats in all) -> its RGB picture
 * at out + 3 * items[i].offset bytes, rows of 3 w_i bytes.  Picture i is bit-identical to um_depth_to_image of depth i
 * alone: the radix select runs over the item's own N_i = h_i w_i pixels (k = floor(0.95 (N_i - 1))), and the NaN, constant
 * and vmax <= vmin rules are the same.  scratch: DEVICE buffer of 2056 * n 32-bit words, reset inside the call.  One
 * memset and nine kernels, grids sized by the capacity (h_max, w_max).  Replaces viz_depth_tensor on each predicted depth
 * of inference_depth for frames of different sizes (evaluate_depth.py:338-417). */
int um_depth_to_image_ragged(const float* depth, int64_t numel, const um_ragged_item* items, uint8_t* out, void* scratch,
                             int32_t n, int32_t h_max, int32_t w_max, void* stream);

/* ---- leaderboard submission payloads -------------------------------------------------------------------------
 * One launch from the model's planar output pred = DEVICE fp32 [batch, C, h, w] at the inference size (C = 2 flow, 1
 * disparity) to each sample's file payload, without the header: sample i at out + i * sample_stride (bytes).  Geometry:
 *   UM_SUBMIT_CROP:   value (Y, X) = pred[i, c, top + Y, left + X], the InputPadder unpad (top + out_h <= h, left + out_w <= w);
 *   UM_SUBMIT_RESIZE: the align-corners bilinear resize to (out_h, out_w) of um_resize_bilinear, then the reference's two
 *                     rounded steps (x * out_w) / w for u and disparity, (x * out_h) / h for v (evaluate_flow.py:67-70,
 *                     evaluate_stereo.py:87); top / left unused.
 * Formats (payload bytes per sample):
 *   UM_SUBMIT_FLO             writeFlow (utils/frame_utils.py:70-99): interleaved (u, v) fp32 little-endian, row-major; 8 h w
 *   UM_SUBMIT_KITTI_FLOW_PNG  writeFlowKITTI (:117-121): PNG scanlines of RGB uint16 big-endian, R = q(64 u + 32768),
 *                             G = q(64 v + 32768), B = 1 (fp32 multiply, then fp32 add); (1 + 6 w) h
 *   UM_SUBMIT_KITTI_DISP_PNG  (disp * 256.).astype(np.uint16) (evaluate_stereo.py:91): PNG scanlines of grey uint16
 *                             big-endian, q(256 d) in fp32; (1 + 2 w) h
 *   UM_SUBMIT_PFM             write_pfm (utils/file_io.py:98-127): fp32 little-endian, rows bottom to top; 4 h w
 * q is numpy's float -> uint16 cast on x86-64: truncate toward zero to int32, NaN / +-inf / anything outside the int32
 * range -> INT32_MIN, keep the low 16 bits (so 65536 -> 0, -1.5 -> 65535, NaN -> 0).  PNG scanlines carry the "Up" filter
 * (each byte minus the byte above it, mod 256, filter byte 2; row 0 unfiltered, filter byte 0): the host only deflates.
 * out_w / out_h are the sizes in the payload; every operation is a correctly rounded fp32 intrinsic (no contraction).  The
 * crop copies values bit for bit; a NaN out of the resize arithmetic is the device's canonical 0x7fffffff.
 * FLO needs 8-byte and PFM 4-byte alignment of out and sample_stride.  No host synchronisation: graph-capturable. */
#define UM_SUBMIT_CROP 0
#define UM_SUBMIT_RESIZE 1
#define UM_SUBMIT_FLO 0
#define UM_SUBMIT_KITTI_FLOW_PNG 1
#define UM_SUBMIT_KITTI_DISP_PNG 2
#define UM_SUBMIT_PFM 3
int um_encode_submission(const float* pred, int32_t batch, int32_t channels, int32_t h, int32_t w, int32_t geometry,
                         int32_t top, int32_t left, int32_t out_h, int32_t out_w, int32_t format, uint8_t* out,
                         int64_t sample_stride, void* stream);

/* ---- evaluation statistics -----------------------------------------------------------------------------------
 * One pass from a batch of predictions at ground-truth resolution to a [batch, S] float64 table of per-sample sufficient
 * statistics (pixel counts, counts over thresholds, fp64 sums), from which the host forms the metrics of the reference's
 * validate_* loops (evaluate_flow.py:160-638, evaluate_stereo.py:302-708, evaluate_depth.py:22-293).
 *   pred: [B, C, h, w] read through element strides (pred_sb, pred_sc, pred_sy, pred_sx) -- e.g. the unpadded window of the
 *         padded model output; C = 2 for flow (pred_sc = distance between the u and v planes), 1 otherwise (pred_sc unused);
 *   gt: contiguous [B, C, h, w]; valid, noc_valid: contiguous [B, h, w] or NULL;
 *   scratch: DEVICE buffer of batch * UM_EVAL_PARTS * S doubles; out: DEVICE [batch, S] doubles.
 * Per-pixel values are correctly rounded fp32 in the reference's order of operations, so every count is the reference's
 * count on the same prediction (logf may differ from numpy's float32 log by 1 ulp: the log-error sum only).  One caveat: the
 * reference's flow epe / |gt| come from torch's CPU float sqrt, which is not correctly rounded (torch 2.11: one ulp off on
 * about 0.7% of inputs); a flow count can then differ only where such a value lies within one ulp of a threshold.  Sums are
 * reduced in a fixed order over a fixed grid (UM_EVAL_PARTS CTAs per sample, then one ordered pass): bit-reproducible,
 * no host synchronisation.  Threshold constants are the reference's python scalars rounded to float32, as torch / numpy
 * compare them with float32 arrays. */
#define UM_EVAL_FLOW 0
#define UM_EVAL_STEREO 1
#define UM_EVAL_DEPTH 2
#define UM_EVAL_PARTS 128
/* Flow, mask_mode selects the evaluation mask M; epe = sqrt(du*du + dv*dv), mag the same of the GT: */
#define UM_EVAL_MASK_ALL 0         /* every pixel (Sintel, Chairs)                                                   */
#define UM_EVAL_MASK_VALID 1       /* valid >= 0.5 (KITTI)                                                           */
#define UM_EVAL_MASK_VALID_MAX 2   /* valid * (mag < max_val) >= 0.5 (Things, evaluate_flow.py:298-303)              */
enum um_eval_flow_cols {
  UM_EVF_N = 0,          /* pixels in M                                                                               */
  UM_EVF_EPE,            /* sum of epe over M                                                                         */
  UM_EVF_1PX, UM_EVF_3PX, UM_EVF_5PX,   /* counts of epe > 1, 3, 5                                                   */
  UM_EVF_OUTLIER,        /* KITTI outliers: epe > 3 & epe / mag > 0.05 (evaluate_flow.py:593)                         */
  UM_EVF_S0_10_N, UM_EVF_S0_10_EPE,     /* (n, sum epe) with mag < 10                                                */
  UM_EVF_S10_40_N, UM_EVF_S10_40_EPE,   /* 10 <= mag <= 40                                                           */
  UM_EVF_S40_N, UM_EVF_S40_EPE,         /* mag > 40                                                                  */
  UM_EVF_MATCHED_N, UM_EVF_MATCHED_EPE, /* noc_valid given: noc_valid > 0.5 & in-image (compute_out_of_boundary_mask) */
  UM_EVF_UNMATCHED_N, UM_EVF_UNMATCHED_EPE,   /* the rest of M                                                       */
  UM_EVAL_FLOW_COLS
};
/* Stereo: e = |gt - pred|, M = gt > 0 (& gt < max_val when max_val > 0). */
enum um_eval_stereo_cols {
  UM_EVS_N = 0, UM_EVS_ABS,               /* n, sum e                                                                */
  UM_EVS_D1,                              /* e > 3 & e / gt > 0.05 (loss/stereo_metric.py:d1_metric)                 */
  UM_EVS_1PX, UM_EVS_2PX, UM_EVS_3PX,     /* e > 1, 2, 3                                                             */
  UM_EVAL_STEREO_COLS
};
/* Depth: d = gt - pred, M = gt > eval_min & gt < eval_max (& valid > 0.5 when valid is given); loss/depth_loss.py:compute_errors. */
enum um_eval_depth_cols {
  UM_EVD_N = 0,
  UM_EVD_ABS_REL,        /* sum |d| / gt                                                                              */
  UM_EVD_SQ_REL,         /* sum d^2 / gt                                                                              */
  UM_EVD_SQ,             /* sum d^2                                                                                   */
  UM_EVD_LOG_SQ,         /* sum (log gt - log pred)^2                                                                 */
  UM_EVD_A1, UM_EVD_A2, UM_EVD_A3,        /* max(gt/pred, pred/gt) < 1.25, 1.25^2, 1.25^3                            */
  UM_EVAL_DEPTH_COLS
};
int um_eval_stats(const float* pred, int64_t pred_sb, int64_t pred_sc, int64_t pred_sy, int64_t pred_sx, const float* gt,
                  const float* valid, const float* noc_valid, int32_t task, int32_t mask_mode, float max_val, float eval_min,
                  float eval_max, int32_t batch, int32_t h, int32_t w, double* scratch, double* out, void* stream);

/* ---- tensor-core implicit-GEMM convolution / Linear layer (fp16 hi/lo split operands, fp32 accumulate) ----------
 * Replaces the nn.Conv2d calls of BasicUpdateBlock (reg_refine.py:6-119), refine_proj (unimatch.py:315) and, as a
 * 1x1 convolution over a [rows/16, 16] grid, nn.Linear (transformer.py:58-60,137,141).
 * Activations: channel-last fp16 planes [2 (hi,lo)][B][H][W][cin_p], cin_p % 64 == 0, padding channels zero.
 * Weights: fp16 planes [2][cout_p][ktot], K ordered (source, tap = ky*kw+kx, ci), ktot = sum_s kh*kw*cin_p[s].
 * Stride 1, 2, 4 or 8 (TMA element strides), zero padding (pad_h, pad_w).  Up to two sources are accumulated (= convolution of their concatenation). */
#define UM_ACT_NONE 0
#define UM_ACT_RELU 1
#define UM_ACT_TANH 2
#define UM_ACT_SIGMOID 3
#define UM_ACT_GELU 4      /* exact erf form (nn.GELU default, transformer.py:34) */
#define UM_CONV_LINEAR 0   /* y = act(acc + bias) -> out_f32 and/or out_split                                          */
#define UM_CONV_GRU_ZR 1   /* cout 256: z = sigmoid(y[0:128]) -> out_f32; sigmoid(y[128:256]) * aux0 -> out_split       */
#define UM_CONV_GRU_Q 2    /* cout 128: (1 - aux1) * aux0 + aux1 * tanh(y) -> out_f32 and/or out_split (reg_refine.py:41-42) */
#define UM_CONV_LN 3       /* cout 128, no bias: aux0 (optional residual) + LayerNorm(acc) * gamma + beta, eps 1e-5
                              (transformer.py:137-144) -> out_f32 and/or out_split                                       */
typedef struct um_conv_desc {
  const void* src[2];
  int32_t cin_p[2];
  int32_t nsrc;
  int32_t batch, h, w;
  const void* weights;
  const float* bias;          /* [cout] or NULL */
  int32_t kh, kw, pad_h, pad_w;
  int32_t cout, cout_p, bn;   /* bn = output-channel tile (16, 64, 96, 128, 192 or 256); cout_p % bn == 0.  bn = 256 / 192 run
                               * as two 128- / 96-wide tiles (register accumulators of two warpgroups). */
  int32_t mode, act;
  float* out_f32;             /* [B,H,W,*] row stride ld_f32 floats, written at channel offset off_f32; or NULL */
  int64_t ld_f32;
  int32_t off_f32;
  int32_t cp_split;           /* channels of the split destination buffer */
  void* out_split;            /* fp16 planes [2][B][H][W][cp_split], written at channel offset off_split; or NULL */
  int32_t off_split;
  int32_t stride;             /* 1, 2, 4 or 8; output is [B, (h+2*pad_h-kh)/stride+1, (w+2*pad_w-kw)/stride+1, cout] */
  const float* aux0;          /* GRU: h   [B,H,W,128] row stride ld_aux0;  LN: residual or NULL */
  int64_t ld_aux0;
  const float* aux1;          /* GRU_Q: z [B,H,W,128] row stride ld_aux1 */
  int64_t ld_aux1;
  const float* gamma;         /* LN: [128] */
  const float* beta;          /* LN: [128] */
  /* batch == 1 only: distance in halves between the hi and the lo plane of the sources / of out_split when the planes are
   * row ranges of larger buffers (0 = densely stacked planes) */
  int64_t src_plane_stride, split_plane_stride;
  /* Window-major operand planes for um_window_attention_planes (a 128 -> cout Linear layer, bn 128, batch 1, pixels =
   * token rows): output channels [win_c0, win_c1) (128-aligned; operand o = (c - win_c0) / 128) are written as fp16
   * (hi, lo) rows of win_dst[o][2][win_streams][kh*kw][win_lp][128] at the row the window split / cyclic shift of
   * win_geom assigns to the token (attention.py:72-83 as address arithmetic); rows >= win_streams*h*w are skipped and
   * the padding rows [lw, win_lp) of every window are never written.  NULL = off. */
  void* win_dst;
  int32_t win_c0, win_c1, win_lp, win_streams;
  um_attn_geom win_geom;
  /* Optional fp32 tensor [B,H,W,>= cout] (row stride ld_pre floats) added to the accumulator before the post-operation: the
   * part of a convolution whose input channels do not change between calls (SepConvGRU over cat[h, inp, motion]: `inp`, and
   * in the first half `h`, are the same in every refinement iteration, unimatch.py:315-333) is computed once by the caller
   * and only the channels that changed are convolved per call.  Not for UM_CONV_LN; bn >= 32; cout % 32 == 0. */
  const float* pre;
  int64_t ld_pre;
} um_conv_desc;
int um_conv2d_tc(const um_conv_desc* desc, void* stream);

/* Fused transformer FFN (transformer.py:137-144, TransformerLayer.mlp + norm2 + residual) on token rows:
 *   out = residual + LayerNorm( GELU( [src0 | src1] W1^T ) W2^T ) * gamma + beta        (no biases, eps 1e-5)
 * src0 / src1: fp16 (hi, lo) planes [2][>= rows][128] (source, message), planes src_plane_stride halves apart;
 * w1: prepared planes [2][hidden][256] (K ordered source | message), w2: [2][128][hidden] (um_conv2d_tc weight layout);
 * residual: fp32 rows (row stride ld_res) or NULL; out_f32 (row stride ld_f32) and/or out_split planes [2][>= rows][128].
 * The hidden activation never leaves the SM: one kernel, hidden channels produced 64 at a time into register accumulators,
 * GELU'd, split and consumed as the register A operand of the second GEMM.
 * rows must be a multiple of 256 (callers with other row counts use two um_conv2d_tc launches),
 * hidden a multiple of 128. */
typedef struct um_ffn_desc {
  const void* src[2];
  int64_t src_plane_stride;
  int64_t rows;
  const void* w1;
  const void* w2;
  int32_t hidden;
  const float* residual;
  int64_t ld_res;
  const float* gamma;
  const float* beta;
  float* out_f32;
  int64_t ld_f32;
  void* out_split;
  int64_t split_plane_stride;
} um_ffn_desc;
int um_ffn_tc(const um_ffn_desc* desc, void* stream);

/* Direct 7x7 convolution (padding 3, stride 1 or 2) for inputs with 1-3 channels, exact fp32: the image stem
 * (backbone.py:55, with normalize_img of utils.py:23-31 folded in as x*scale[c]+shift[c]; scale/shift are HOST arrays of 3
 * floats or NULL) and refine.encoder.convf1 (reg_refine.py:62,70).  nchw != 0: planar sources in0 (images [0, n_half)) and
 * in1 (the rest), i.e. the two views without a concatenation copy; else one channel-last source [n,h,w,cin].
 * Output channel-last fp32 (row stride ld_out) and/or fp16 (hi, lo) planes of width cp; cout a multiple of 16, <= 128. */
int um_conv7x7_small(const float* in0, const float* in1, int32_t nchw, int32_t n_half, int32_t n, int32_t h, int32_t w,
                     int32_t cin, int32_t stride, const float* weight, const float* bias, int32_t cout, int32_t relu,
                     const float* scale, const float* shift, float* out_f32, int64_t ld_out, void* out_split, int32_t cp,
                     void* stream);

/* InstanceNorm2d (eps 1e-5, no affine, biased variance; backbone.py:7,41) on channel-last fp32 [n, hw, c] maps.
 * stats: [n][2][c] = mean, 1/sqrt(var+eps); scratch: um_instance_norm_scratch_floats(n, c) floats.
 * apply: y = IN(a) (stats_a may be NULL = identity), optional ReLU, optional + res (itself optionally normalised by
 * stats_res), optional ReLU; written as fp32 and/or fp16 (hi, lo) planes [2][n*hw][cp] at channel offset off. */
int64_t um_instance_norm_scratch_floats(int32_t n, int32_t c);
int um_instance_norm_stats(const float* x, int64_t ld, int32_t n, int32_t hw, int32_t c, float* scratch, float* stats,
                           void* stream);
int um_instance_norm_apply(const float* a, int64_t ld_a, const float* stats_a, int32_t relu_a, const float* res,
                           int64_t ld_res, const float* stats_res, int32_t relu_out, float* out_f32, int64_t ld_o,
                           void* out_split, int32_t cp, int32_t off, int32_t n, int32_t hw, int32_t c, void* stream);

/* fp32 rows [rows, channels] (row stride ld) -> fp16 (hi, lo) planes of a [>= rows, cp] buffer at channel offset off;
 * the lo plane starts dst_plane_stride halves after the hi plane (0 = rows * cp, densely stacked). */
int um_split_planes(const float* src, int64_t rows, int32_t channels, int64_t ld, void* dst, int32_t cp, int32_t off,
                    int64_t dst_plane_stride, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* UNIMATCH_SM100_H_ */
