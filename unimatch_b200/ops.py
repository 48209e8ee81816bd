"""ctypes binding of libunimatch_sm100.so + registration of every entry point as a torch custom op
(`torch.ops.unimatch_sm100.*`, CUDA only).

There is no CPU or PyTorch fallback on this path: if the shared library is missing it is built with nvcc,
and if that is impossible the import fails; an op called with CPU tensors raises (no CPU kernel is registered).
The C ABI is declared in include/unimatch_sm100.h.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libunimatch_sm100.so")

MASK_NONE, MASK_SWIN, MASK_CAUSAL = 0, 1, 2
VALUE_TENSOR, VALUE_COORDS, VALUE_XCOORD = 0, 1, 2
POST_NONE, POST_MINUS_OWN, POST_OWN_MINUS = 0, 1, 2


FORCE_CUDA_CORES = 1
_force_cuda_cores = False      # diagnostic switch (tests): route every attention shape to the exact-fp32 CUDA-core kernel


def set_force_cuda_cores(flag):
    global _force_cuda_cores
    _force_cuda_cores = bool(flag)


EVAL_FLOW, EVAL_STEREO, EVAL_DEPTH = 0, 1, 2
EVAL_MASK_ALL, EVAL_MASK_VALID, EVAL_MASK_VALID_MAX = 0, 1, 2
EVAL_PARTS = 128                      # UM_EVAL_PARTS: partial rows per sample in the scratch buffer
# columns of the [B, S] statistics table (include/unimatch_sm100.h, enum um_eval_*_cols)
EVAL_FLOW_COLS = ("n", "epe", "1px", "3px", "5px", "outlier", "s0_10_n", "s0_10_epe", "s10_40_n", "s10_40_epe", "s40_n",
                  "s40_epe", "matched_n", "matched_epe", "unmatched_n", "unmatched_epe")
EVAL_STEREO_COLS = ("n", "abs", "d1", "1px", "2px", "3px")
EVAL_DEPTH_COLS = ("n", "abs_rel", "sq_rel", "sq", "log_sq", "a1", "a2", "a3")
EVAL_COLS = {EVAL_FLOW: EVAL_FLOW_COLS, EVAL_STEREO: EVAL_STEREO_COLS, EVAL_DEPTH: EVAL_DEPTH_COLS}
# the [B, 32] scene-flow table (include/unimatch_sm100.h, um_scene_flow_stats): column of (set, region, metric, kind)
SF_SETS, SF_REGIONS, SF_METRICS, SF_KINDS = ("occ", "noc"), ("bg", "fg"), ("d1", "d2", "fl", "sf"), ("n", "outliers")
SF_COLS = 32


def sf_col(s, r, m, k):
    """UM_SF_COL: column of set s (0 occ, 1 noc), region r (0 bg, 1 fg), metric m (0 D1, 1 D2, 2 Fl, 3 SF) and kind k
    (0 valid pixels, 1 outliers)"""
    return ((s * 2 + r) * 4 + m) * 2 + k


ACT_NONE, ACT_RELU, ACT_TANH, ACT_SIGMOID, ACT_GELU = 0, 1, 2, 3, 4
CONV_LINEAR, CONV_GRU_ZR, CONV_GRU_Q, CONV_LN = 0, 1, 2, 3


class AttnGeom(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in ("h", "w", "kh", "kw", "sh", "sw", "mask_mode")]


class ConvDesc(ctypes.Structure):
    _fields_ = [("src", ctypes.c_void_p * 2), ("cin_p", ctypes.c_int32 * 2), ("nsrc", ctypes.c_int32),
                ("batch", ctypes.c_int32), ("h", ctypes.c_int32), ("w", ctypes.c_int32),
                ("weights", ctypes.c_void_p), ("bias", ctypes.c_void_p),
                ("kh", ctypes.c_int32), ("kw", ctypes.c_int32), ("pad_h", ctypes.c_int32), ("pad_w", ctypes.c_int32),
                ("cout", ctypes.c_int32), ("cout_p", ctypes.c_int32), ("bn", ctypes.c_int32),
                ("mode", ctypes.c_int32), ("act", ctypes.c_int32),
                ("out_f32", ctypes.c_void_p), ("ld_f32", ctypes.c_int64), ("off_f32", ctypes.c_int32),
                ("cp_split", ctypes.c_int32), ("out_split", ctypes.c_void_p), ("off_split", ctypes.c_int32),
                ("stride", ctypes.c_int32),
                ("aux0", ctypes.c_void_p), ("ld_aux0", ctypes.c_int64), ("aux1", ctypes.c_void_p), ("ld_aux1", ctypes.c_int64),
                ("gamma", ctypes.c_void_p), ("beta", ctypes.c_void_p),
                ("src_plane_stride", ctypes.c_int64), ("split_plane_stride", ctypes.c_int64),
                ("win_dst", ctypes.c_void_p), ("win_c0", ctypes.c_int32), ("win_c1", ctypes.c_int32),
                ("win_lp", ctypes.c_int32), ("win_streams", ctypes.c_int32), ("win_geom", AttnGeom),
                ("pre", ctypes.c_void_p), ("ld_pre", ctypes.c_int64)]


class RaggedItem(ctypes.Structure):
    """um_ragged_item: one image of a ragged batch (offset in elements of the packed buffer, size, resize scale, flags)"""
    _fields_ = [("offset", ctypes.c_int64), ("h", ctypes.c_int32), ("w", ctypes.c_int32), ("scale", ctypes.c_float),
                ("flags", ctypes.c_int32)]


RAGGED_FLIP_X, RAGGED_TRANSPOSE = 1, 2
RAGGED_ITEM_BYTES = ctypes.sizeof(RaggedItem)      # 24


class FfnDesc(ctypes.Structure):
    _fields_ = [("src", ctypes.c_void_p * 2), ("src_plane_stride", ctypes.c_int64), ("rows", ctypes.c_int64),
                ("w1", ctypes.c_void_p), ("w2", ctypes.c_void_p), ("hidden", ctypes.c_int32),
                ("residual", ctypes.c_void_p), ("ld_res", ctypes.c_int64), ("gamma", ctypes.c_void_p), ("beta", ctypes.c_void_p),
                ("out_f32", ctypes.c_void_p), ("ld_f32", ctypes.c_int64), ("out_split", ctypes.c_void_p),
                ("split_plane_stride", ctypes.c_int64)]


_P, _I, _L, _F = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_float
_G, _FP, _RC = ctypes.POINTER(AttnGeom), ctypes.POINTER(ctypes.c_float), ctypes.c_int
_PP = ctypes.POINTER(ctypes.c_void_p)

# name -> (restype, argtypes) of every function include/unimatch_sm100.h declares
_SIGNATURES = {
    "um_abi_version": (_RC, []),
    "um_build_info": (ctypes.c_char_p, []),
    "um_last_error": (ctypes.c_char_p, []),
    "um_launch_count": (_L, []),
    "um_window_attention": (_RC, [_P, _P, _P, _P, _I, _I, _L, _L, _L, _L, _G, _P, _L, _I, _P]),
    "um_window_attention_workspace": (_L, [_G, _I]),
    "um_attention_planes_lp": (_I, [_G]),
    "um_window_attention_planes": (_RC, [_P, _P, _P, _P, _L, _P, _L, _I, _I, _G, _P]),
    "um_softmax_expectation": (_RC, [_P, _P, _P, _P, _I, _I, _I, _L, _L, _I, _I, _I, _G, _P, _L, _I, _P]),
    "um_softmax_expectation_workspace": (_L, [_G, _I, _I]),
    "um_local_corr_softmax": (_RC, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _P]),
    "um_local_corr_volume": (_RC, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P]),
    "um_flow_warp": (_RC, [_P, _P, _P, _I, _I, _I, _I, _P]),
    "um_fb_consistency": (_RC, [_P, _P, _F, _F, _P, _P, _I, _I, _I, _P]),
    "um_fb_consistency_ragged": (_RC, [_P, _L, _P, _F, _F, _P, _L, _P, _I, _I, _I, _P]),
    "um_fb_consistency_error": (_RC, [_P, _P, _F, _F, _P, _P, _P, _I, _I, _I, _P]),
    "um_chain_tracks": (_RC, [_P, _P, _I, _I, _I, _P, _P, _P, _P, _P]),
    "um_track_points_forward": (_RC, [_P, _P, _I, _I, _I, _I, _P, _I, _I, _P, _P, _P, _P, _P]),
    "um_track_points_backward": (_RC, [_P, _P, _I, _I, _I, _P, _I, _I, _P, _P, _P]),
    "um_multi_flow_tracks": (_RC, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P]),
    "um_warp_disparity": (_RC, [_P, _P, _P, _P, _I, _I, _I, _P]),
    "um_scene_flow_stats": (_RC, [_P, _P, _P, _PP, _PP, _PP, _PP, _P, _I, _I, _I, _P, _P, _P]),
    "um_propagate_local": (_RC, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _L, _L, _P]),
    "um_depth_corr_softmax": (_RC, [_P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P]),
    "um_add_position": (_RC, [_P, _P, _P, _I, _I, _I, _I, _I, _P]),
    "um_convex_upsample": (_RC, [_P, _P, _P, _I, _I, _I, _I, _I, _F, _P]),
    "um_upsample2x": (_RC, [_P, _P, _I, _I, _I, _I, _F, _P]),
    "um_resize_bilinear": (_RC, [_P, _P, _I, _I, _I, _I, _I, _I, _FP, _I, _P]),
    "um_frames_to_planar": (_RC, [_P, _P, _I, _I, _I, _I, _I, _I, _P]),
    "um_frames_to_planar_ragged": (_RC, [_P, _L, _P, _P, _I, _I, _I, _I, _I, _P]),
    "um_frames_to_planar_normalized": (_RC, [_P, _P, _I, _I, _I, _I, _I, _FP, _FP, _P]),
    "um_frames_to_planar_normalized_ragged": (_RC, [_P, _L, _P, _P, _I, _I, _I, _I, _I, _FP, _FP, _P]),
    "um_resize_bilinear_ragged": (_RC, [_P, _P, _L, _P, _I, _I, _I, _I, _I, _P]),
    "um_disparity_to_image_ragged": (_RC, [_P, _L, _P, _P, _P, _I, _I, _I, _P]),
    "um_flow_to_image": (_RC, [_P, _P, _L, _L, _P, _I, _I, _I, _P]),
    "um_flow_to_image_ragged": (_RC, [_P, _L, _P, _P, _L, _P, _P, _I, _I, _I, _P]),
    "um_disparity_to_image": (_RC, [_P, _P, _L, _L, _P, _I, _I, _I, _P]),
    "um_depth_to_image": (_RC, [_P, _P, _L, _L, _P, _I, _I, _I, _P]),
    "um_depth_to_image_ragged": (_RC, [_P, _L, _P, _P, _P, _I, _I, _I, _P]),
    "um_encode_submission": (_RC, [_P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P, _L, _P]),
    "um_eval_stats": (_RC, [_P, _L, _L, _L, _L, _P, _P, _P, _I, _I, _F, _F, _F, _I, _I, _I, _P, _P, _P]),
    "um_conv2d_tc": (_RC, [ctypes.POINTER(ConvDesc), _P]),
    "um_ffn_tc": (_RC, [ctypes.POINTER(FfnDesc), _P]),
    "um_conv7x7_small": (_RC, [_P, _P, _I, _I, _I, _I, _I, _I, _I, _P, _P, _I, _I, _FP, _FP, _P, _L, _P, _I, _P]),
    "um_instance_norm_scratch_floats": (_L, [_I, _I]),
    "um_instance_norm_stats": (_RC, [_P, _L, _I, _I, _I, _P, _P, _P]),
    "um_instance_norm_apply": (_RC, [_P, _L, _P, _I, _P, _L, _P, _I, _P, _L, _P, _I, _I, _I, _I, _I, _P]),
    "um_split_planes": (_RC, [_P, _L, _I, _L, _P, _I, _I, _L, _P]),
}
SYMBOLS = list(_SIGNATURES)


def _load():
    from .csrc.build import build, have_nvcc
    if have_nvcc():
        build()                         # no-op when the in-tree .so matches the sources (content stamp)
    elif not os.path.exists(LIB_PATH):  # no library and no compiler: the product path has no fallback
        raise ImportError("libunimatch_sm100.so is missing and nvcc is not available to build it")
    lib = ctypes.CDLL(LIB_PATH)
    missing = [s for s in SYMBOLS if not hasattr(lib, s)]
    if missing:
        raise ImportError("libunimatch_sm100.so lacks symbols %s (stale build? run python unimatch_b200/csrc/build.py --force)" % missing)
    for name, (restype, argtypes) in _SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
    return lib


LIB = _load()


def build_info():
    return LIB.um_build_info().decode()


def launch_count():
    return int(LIB.um_launch_count())


def _check(rc, name):
    if rc != 0:
        raise RuntimeError("%s failed (%d): %s" % (name, rc, LIB.um_last_error().decode()))


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _f32c(t, name, rows_ok=False):
    if not t.is_cuda:
        raise RuntimeError("%s: expected a CUDA tensor (libunimatch_sm100 has no CPU path)" % name)
    if t.dtype != torch.float32:
        raise RuntimeError("%s: expected float32" % name)
    if rows_ok:
        if t.stride(-1) != 1:
            raise RuntimeError("%s: last dim must be contiguous" % name)
    elif not t.is_contiguous():
        raise RuntimeError("%s: expected a contiguous tensor" % name)
    return t


def _rows(t, name):
    """[N, L, 128] view with uniform row stride: returns ld (floats)."""
    _f32c(t, name, rows_ok=True)
    if t.dim() != 3 or t.shape[-1] != 128:
        raise RuntimeError("%s: expected [N, L, 128]" % name)
    ld = t.stride(1)
    if t.shape[0] > 1 and t.stride(0) != ld * t.shape[1]:
        raise RuntimeError("%s: batch stride must equal L * row stride" % name)
    return ld


_lib = torch.library.Library("unimatch_sm100", "DEF")


def _define(schema, impl):
    _lib.define(schema)
    name = schema.split("(")[0]
    _lib.impl(name, impl, "CUDA")
    return getattr(torch.ops.unimatch_sm100, name)


# ---- attention ------------------------------------------------------------------------------------------
def _window_attention(q, k, v, kv_shift, h, w, kh, kw, sh, sw, mask_mode):
    ldq, ldk, ldv = _rows(q, "q"), _rows(k, "k"), _rows(v, "v")
    n, l, _ = q.shape
    out = torch.empty((n, l, 128), device=q.device, dtype=torch.float32)
    g = AttnGeom(h, w, kh, kw, sh, sw, mask_mode)
    flags = FORCE_CUDA_CORES if _force_cuda_cores else 0
    ws_bytes = 0 if flags else int(LIB.um_window_attention_workspace(ctypes.byref(g), n))
    ws = torch.empty((ws_bytes,), device=q.device, dtype=torch.uint8) if ws_bytes else None
    _check(LIB.um_window_attention(_p(q), _p(k), _p(v), _p(out), n, kv_shift, ldq, ldk, ldv, 128, ctypes.byref(g),
                                   _p(ws), ws_bytes, flags, _stream()), "um_window_attention")
    return out


window_attention = _define(
    "window_attention(Tensor q, Tensor k, Tensor v, int kv_shift, int h, int w, int kh, int kw, int sh, int sw, "
    "int mask_mode) -> Tensor", _window_attention)


def attention_planes_lp(h, w, kh, kw, sh, sw, mask_mode):
    """Padded window length of the tensor-core attention's operand planes; 0 = this geometry runs on the CUDA-core kernel."""
    g = AttnGeom(h, w, kh, kw, sh, sw, mask_mode)
    return int(LIB.um_attention_planes_lp(ctypes.byref(g)))


def _planes_ok(t, name, n, nwin, lp):
    if t.dtype != torch.float16 or not t.is_contiguous() or t.numel() != 2 * n * nwin * lp * 128:
        raise RuntimeError("%s: expected contiguous fp16 planes [2, %d, %d, %d, 128]" % (name, n, nwin, lp))


def _window_attention_planes(qp, kp, vp, n, kv_shift, h, w, kh, kw, sh, sw, mask_mode, out_f32, out_split):
    g = AttnGeom(h, w, kh, kw, sh, sw, mask_mode)
    lp = int(LIB.um_attention_planes_lp(ctypes.byref(g)))
    if lp == 0:
        raise RuntimeError("window_attention_planes: geometry is not built for the tensor-core kernel")
    for t, nm in ((qp, "q_planes"), (kp, "k_planes"), (vp, "v_planes")):
        _planes_ok(t, nm, n, kh * kw, lp)
    ldo, plane = 0, 0
    if out_f32 is not None:
        ldo = _rows(out_f32, "out_f32")
    if out_split is not None:
        if out_split.dtype != torch.float16 or not out_split.is_contiguous() or out_split.shape[0] != 2 or out_split.shape[-1] != 128:
            raise RuntimeError("window_attention_planes: out_split must be contiguous fp16 planes [2, rows, 128]")
        plane = out_split[0].numel()
    _check(LIB.um_window_attention_planes(_p(qp), _p(kp), _p(vp), _p(out_f32), ldo, _p(out_split), plane, n, kv_shift,
                                          ctypes.byref(g), _stream()), "um_window_attention_planes")


window_attention_planes = _define(
    "window_attention_planes(Tensor q_planes, Tensor k_planes, Tensor v_planes, int n_streams, int kv_shift, int h, int w, "
    "int kh, int kw, int sh, int sw, int mask_mode, Tensor(a!)? out_f32, Tensor(b!)? out_split) -> ()",
    _window_attention_planes)


def _softmax_expectation(q, k, values, n_streams, kv_shift, vdim, value_mode, post_op, h, w, kh, kw, mask_mode):
    ldq, ldk = _rows(q, "q"), _rows(k, "k")
    n_total, l, _ = q.shape
    if values is not None:
        _f32c(values, "values")
    out = torch.empty((n_streams, l, vdim), device=q.device, dtype=torch.float32)
    g = AttnGeom(h, w, kh, kw, 0, 0, mask_mode)
    flags = FORCE_CUDA_CORES if _force_cuda_cores else 0
    ws_bytes = 0 if flags else int(LIB.um_softmax_expectation_workspace(ctypes.byref(g), n_total, value_mode))
    ws = torch.empty((ws_bytes,), device=q.device, dtype=torch.uint8) if ws_bytes else None
    _check(LIB.um_softmax_expectation(_p(q), _p(k), _p(values), _p(out), n_streams, n_total, kv_shift, ldq, ldk, vdim,
                                      value_mode, post_op, ctypes.byref(g), _p(ws), ws_bytes, flags, _stream()),
           "um_softmax_expectation")
    return out


softmax_expectation = _define(
    "softmax_expectation(Tensor q, Tensor k, Tensor? values, int n_streams, int kv_shift, int vdim, int value_mode, "
    "int post_op, int h, int w, int kh, int kw, int mask_mode) -> Tensor", _softmax_expectation)


# ---- local matching ---------------------------------------------------------------------------------------
def _local_corr_softmax(f0, f1, h, w, ry, rx, stereo):
    _f32c(f0, "f0"), _f32c(f1, "f1")
    b = f0.shape[0]
    out = torch.empty((b, h, w, 1 if stereo else 2), device=f0.device, dtype=torch.float32)
    _check(LIB.um_local_corr_softmax(_p(f0), _p(f1), _p(out), b, h, w, ry, rx, int(stereo), _stream()),
           "um_local_corr_softmax")
    return out


local_corr_softmax = _define("local_corr_softmax(Tensor f0, Tensor f1, int h, int w, int ry, int rx, bool stereo) -> Tensor",
                             _local_corr_softmax)


def _local_corr_volume(f0, f1, flow, h, w, radius):
    _f32c(f0, "f0"), _f32c(f1, "f1"), _f32c(flow, "flow")
    b = f0.shape[0]
    k = (2 * radius + 1) ** 2
    out = torch.empty((b, h, w, k), device=f0.device, dtype=torch.float32)
    _check(LIB.um_local_corr_volume(_p(f0), _p(f1), _p(flow), _p(out), b, h, w, radius, flow.shape[-1], _stream()),
           "um_local_corr_volume")
    return out


local_corr_volume = _define("local_corr_volume(Tensor f0, Tensor f1, Tensor flow, int h, int w, int radius) -> Tensor",
                            _local_corr_volume)


def _flow_warp(f, flow, h, w):
    _f32c(f, "f"), _f32c(flow, "flow")
    out = torch.empty_like(f)
    _check(LIB.um_flow_warp(_p(f), _p(flow), _p(out), f.shape[0], h, w, flow.shape[-1], _stream()), "um_flow_warp")
    return out


flow_warp = _define("flow_warp(Tensor f, Tensor flow, int h, int w) -> Tensor", _flow_warp)


def _fb_consistency(fwd_flow, bwd_flow, alpha, beta):
    _f32c(fwd_flow, "fwd_flow"), _f32c(bwd_flow, "bwd_flow")
    if fwd_flow.dim() != 4 or fwd_flow.shape[1] != 2 or fwd_flow.shape != bwd_flow.shape:
        raise ValueError("fb_consistency: flows must be planar [B,2,H,W] of equal shape")
    b, _, h, w = fwd_flow.shape
    fwd_occ = torch.empty((b, h, w), device=fwd_flow.device, dtype=torch.float32)
    bwd_occ = torch.empty_like(fwd_occ)
    _check(LIB.um_fb_consistency(_p(fwd_flow), _p(bwd_flow), float(alpha), float(beta), _p(fwd_occ), _p(bwd_occ), b, h, w,
                                 _stream()), "um_fb_consistency")
    return fwd_occ, bwd_occ


fb_consistency = _define("fb_consistency(Tensor fwd_flow, Tensor bwd_flow, float alpha, float beta) -> (Tensor, Tensor)",
                         _fb_consistency)


def _fb_consistency_error(fwd_flow, bwd_flow, alpha, beta):
    """fb_consistency's masks plus the forward residual [B,H,W] they compare (include/unimatch_sm100.h,
    um_fb_consistency_error)"""
    _f32c(fwd_flow, "fwd_flow"), _f32c(bwd_flow, "bwd_flow")
    if fwd_flow.dim() != 4 or fwd_flow.shape[1] != 2 or fwd_flow.shape != bwd_flow.shape:
        raise ValueError("fb_consistency_error: flows must be planar [B,2,H,W] of equal shape")
    b, _, h, w = fwd_flow.shape
    fwd_occ = torch.empty((b, h, w), device=fwd_flow.device, dtype=torch.float32)
    bwd_occ, fwd_err = torch.empty_like(fwd_occ), torch.empty_like(fwd_occ)
    _check(LIB.um_fb_consistency_error(_p(fwd_flow), _p(bwd_flow), float(alpha), float(beta), _p(fwd_occ), _p(bwd_occ),
                                       _p(fwd_err), b, h, w, _stream()), "um_fb_consistency_error")
    return fwd_occ, bwd_occ, fwd_err


fb_consistency_error = _define("fb_consistency_error(Tensor fwd_flow, Tensor bwd_flow, float alpha, float beta) -> "
                               "(Tensor, Tensor, Tensor)", _fb_consistency_error)


def _chain_tracks(flow, occ, pos, vis):
    """flow: contiguous fp32 [n, 2, h, w]; occ: contiguous fp32 [n, h, w] or None (nothing occluded); pos / vis: the running
    state, contiguous fp32 [h, w, 2] and uint8 [h, w], advanced in place.  Returns the state after each flow, [n, h, w, 2]
    and [n, h, w] (include/unimatch_sm100.h, um_chain_tracks)."""
    _f32c(flow, "flow"), _f32c(pos, "pos")
    if flow.dim() != 4 or flow.shape[1] != 2:
        raise RuntimeError("chain_tracks: expected planar flows [n, 2, h, w]")
    n, _, h, w = flow.shape
    if occ is not None:
        _f32c(occ, "occ")
        if tuple(occ.shape) != (n, h, w) or occ.device != flow.device:
            raise RuntimeError("chain_tracks: occ must be [n, h, w] on the flows' device")
    if tuple(pos.shape) != (h, w, 2) or pos.device != flow.device:
        raise RuntimeError("chain_tracks: pos must be [h, w, 2] on the flows' device")
    if vis.dtype != torch.uint8 or tuple(vis.shape) != (h, w) or not vis.is_contiguous() or vis.device != flow.device:
        raise RuntimeError("chain_tracks: vis must be contiguous uint8 [h, w] on the flows' device")
    pos_out = torch.empty((n, h, w, 2), device=flow.device, dtype=torch.float32)
    vis_out = torch.empty((n, h, w), device=flow.device, dtype=torch.uint8)
    _check(LIB.um_chain_tracks(_p(flow), _p(occ), n, h, w, _p(pos), _p(vis), _p(pos_out), _p(vis_out), _stream()),
           "um_chain_tracks")
    return pos_out, vis_out


chain_tracks = _define("chain_tracks(Tensor flow, Tensor? occ, Tensor(a!) pos, Tensor(b!) vis) -> (Tensor, Tensor)",
                       _chain_tracks)


def _point_tables(queries, tracks, visible, device):
    """queries: contiguous fp32 [nq, 3] (t_q, y, x); tracks / visible: contiguous fp32 [nq, nt, 2] and uint8 [nq, nt]"""
    _f32c(queries, "queries"), _f32c(tracks, "tracks")
    if queries.dim() != 2 or queries.shape[1] != 3 or queries.device != device:
        raise RuntimeError("track_points: queries must be [nq, 3] on the flows' device")
    nq = queries.shape[0]
    if tracks.dim() != 3 or tracks.shape[0] != nq or tracks.shape[2] != 2 or tracks.device != device:
        raise RuntimeError("track_points: tracks must be [nq, nt, 2] on the flows' device")
    if (visible.dtype != torch.uint8 or tuple(visible.shape) != tuple(tracks.shape[:2]) or not visible.is_contiguous()
            or visible.device != device):
        raise RuntimeError("track_points: visible must be contiguous uint8 [nq, nt] on the flows' device")
    return nq, tracks.shape[1]


def _flows_and_masks(flow, occ, name):
    _f32c(flow, name)
    if flow.dim() != 4 or flow.shape[1] != 2:
        raise RuntimeError("%s: expected planar flows [n, 2, h, w]" % name)
    if occ is not None:
        _f32c(occ, "occ")
        if tuple(occ.shape) != (flow.shape[0],) + tuple(flow.shape[2:]) or occ.device != flow.device:
            raise RuntimeError("%s: occ must be [n, h, w] on the flows' device" % name)
    return flow.shape[0], flow.shape[2], flow.shape[3]


def _track_points_forward(flow, occ, t0, queries, pos, vis, tracks, visible):
    """flow / occ: the forward flows [n, 2, h, w] and masks [n, h, w] (or None) of pairs t0 .. t0+n-1; queries [nq, 3];
    pos / vis: the running state, contiguous fp32 [nq, 2] and uint8 [nq]; tracks / visible: the tables, written in place
    (include/unimatch_sm100.h, um_track_points_forward)."""
    n, h, w = _flows_and_masks(flow, occ, "track_points_forward")
    nq, nt = _point_tables(queries, tracks, visible, flow.device)
    _f32c(pos, "pos")
    if tuple(pos.shape) != (nq, 2) or pos.device != flow.device:
        raise RuntimeError("track_points_forward: pos must be [nq, 2] on the flows' device")
    if vis.dtype != torch.uint8 or tuple(vis.shape) != (nq,) or vis.device != flow.device:
        raise RuntimeError("track_points_forward: vis must be uint8 [nq] on the flows' device")
    _check(LIB.um_track_points_forward(_p(flow), _p(occ), n, h, w, int(t0), _p(queries), nq, nt, _p(pos), _p(vis),
                                       _p(tracks), _p(visible), _stream()), "um_track_points_forward")


track_points_forward = _define("track_points_forward(Tensor flow, Tensor? occ, int t0, Tensor queries, Tensor(a!) pos, "
                               "Tensor(b!) vis, Tensor(c!) tracks, Tensor(d!) visible) -> ()", _track_points_forward)


def _track_points_backward(flow, occ, queries, tracks, visible):
    """flow / occ: the backward flows [n, 2, h, w] and masks [n, h, w] (or None) of pairs 0 .. n-1, n >= 0; queries [nq, 3];
    tracks / visible: the tables, entries 0 .. t_q of every row written in place (include/unimatch_sm100.h,
    um_track_points_backward)."""
    n, h, w = _flows_and_masks(flow, occ, "track_points_backward")
    nq, nt = _point_tables(queries, tracks, visible, flow.device)
    _check(LIB.um_track_points_backward(_p(flow) if n else None, _p(occ) if n else None, n, h, w, _p(queries), nq, nt,
                                        _p(tracks), _p(visible), _stream()), "um_track_points_backward")


track_points_backward = _define("track_points_backward(Tensor flow, Tensor? occ, Tensor queries, Tensor(a!) tracks, "
                                "Tensor(b!) visible) -> ()", _track_points_backward)


def _multi_flow_tracks(flow, occ, err, src, dst, pos, sig, vis):
    """flow: contiguous fp32 [n, k, 2, h, w], candidate (t, j)'s pair; occ / err: its forward mask and residual, contiguous
    fp32 [n, k, h, w]; src: device int32 [n, k], the state slot of each candidate's source (-1 absent); dst: device int32
    [n], each frame's slot; pos / sig / vis: the state ring, contiguous fp32 [r, h, w, 2], fp32 [r, h, w] and uint8
    [r, h, w], updated in place.  Returns tracks [n, h, w, 2], visible [n, h, w] and sigma^2 [n, h, w]
    (include/unimatch_sm100.h, um_multi_flow_tracks)."""
    _f32c(flow, "flow"), _f32c(occ, "occ"), _f32c(err, "err"), _f32c(pos, "pos"), _f32c(sig, "sig")
    if flow.dim() != 5 or flow.shape[2] != 2:
        raise RuntimeError("multi_flow_tracks: expected planar flows [n, k, 2, h, w]")
    n, k, _, h, w = flow.shape
    dev = flow.device
    for name, t in (("occ", occ), ("err", err)):
        if tuple(t.shape) != (n, k, h, w) or t.device != dev:
            raise RuntimeError("multi_flow_tracks: %s must be [n, k, h, w] on the flows' device" % name)
    for name, t, shape in (("src", src, (n, k)), ("dst", dst, (n,))):
        if t.dtype != torch.int32 or tuple(t.shape) != shape or not t.is_contiguous() or t.device != dev:
            raise RuntimeError("multi_flow_tracks: %s must be contiguous int32 %s on the flows' device" % (name, list(shape)))
    r = pos.shape[0] if pos.dim() == 4 else -1
    if tuple(pos.shape) != (r, h, w, 2) or pos.device != dev:
        raise RuntimeError("multi_flow_tracks: pos must be [r, h, w, 2] on the flows' device")
    if tuple(sig.shape) != (r, h, w) or sig.device != dev:
        raise RuntimeError("multi_flow_tracks: sig must be [r, h, w] like pos")
    if vis.dtype != torch.uint8 or tuple(vis.shape) != (r, h, w) or not vis.is_contiguous() or vis.device != dev:
        raise RuntimeError("multi_flow_tracks: vis must be contiguous uint8 [r, h, w] like pos")
    tracks = torch.empty((n, h, w, 2), device=dev, dtype=torch.float32)
    visible = torch.empty((n, h, w), device=dev, dtype=torch.uint8)
    sigma = torch.empty((n, h, w), device=dev, dtype=torch.float32)
    _check(LIB.um_multi_flow_tracks(_p(flow), _p(occ), _p(err), _p(src), _p(dst), n, k, h, w, r, _p(pos), _p(sig), _p(vis),
                                    _p(tracks), _p(visible), _p(sigma), _stream()), "um_multi_flow_tracks")
    return tracks, visible, sigma


multi_flow_tracks = _define("multi_flow_tracks(Tensor flow, Tensor occ, Tensor err, Tensor src, Tensor dst, Tensor(a!) pos, "
                            "Tensor(b!) sig, Tensor(c!) vis) -> (Tensor, Tensor, Tensor)", _multi_flow_tracks)


def _warp_disparity(disp_next, flow):
    """disp_next: contiguous fp32 [B, h, w], the disparity of left frame t+1; flow: contiguous fp32 [B, 2, h, w], left t ->
    left t+1.  Returns (disp1 fp32 [B, h, w], in_frame uint8 [B, h, w]) (include/unimatch_sm100.h, um_warp_disparity)."""
    _f32c(disp_next, "disp_next"), _f32c(flow, "flow")
    if disp_next.dim() != 3 or flow.dim() != 4 or flow.shape[1] != 2 or tuple(flow.shape[2:]) != tuple(disp_next.shape[1:]) \
            or flow.shape[0] != disp_next.shape[0] or flow.device != disp_next.device:
        raise RuntimeError("warp_disparity: expected disp_next [B, h, w] and a planar flow [B, 2, h, w] on its device")
    b, h, w = disp_next.shape
    disp1 = torch.empty_like(disp_next)
    in_frame = torch.empty((b, h, w), device=disp_next.device, dtype=torch.uint8)
    _check(LIB.um_warp_disparity(_p(disp_next), _p(flow), _p(disp1), _p(in_frame), b, h, w, _stream()), "um_warp_disparity")
    return disp1, in_frame


warp_disparity = _define("warp_disparity(Tensor disp_next, Tensor flow) -> (Tensor, Tensor)", _warp_disparity)


def _propagate_local(q, k, flow, h, w, radius):
    ldq, ldk = _rows(q, "q"), _rows(k, "k")
    _f32c(flow, "flow")
    b = q.shape[0]
    out = torch.empty_like(flow)
    _check(LIB.um_propagate_local(_p(q), _p(k), _p(flow), _p(out), b, h, w, radius, flow.shape[-1], ldq, ldk, _stream()),
           "um_propagate_local")
    return out


propagate_local = _define("propagate_local(Tensor q, Tensor k, Tensor flow, int h, int w, int radius) -> Tensor",
                          _propagate_local)


def _depth_corr_softmax(f0, f1, K, Kinv, pose, cand, h, w, from_argmax):
    for t, n in ((f0, "f0"), (f1, "f1"), (K, "K"), (Kinv, "Kinv"), (pose, "pose"), (cand, "cand")):
        _f32c(t, n)
    b = f0.shape[0]
    out = torch.empty((b, h, w, 1), device=f0.device, dtype=torch.float32)
    _check(LIB.um_depth_corr_softmax(_p(f0), _p(f1), _p(K), _p(Kinv), _p(pose), _p(cand), _p(out), b, h, w,
                                     cand.numel(), int(from_argmax), _stream()), "um_depth_corr_softmax")
    return out


depth_corr_softmax = _define(
    "depth_corr_softmax(Tensor f0, Tensor f1, Tensor K, Tensor Kinv, Tensor pose, Tensor cand, int h, int w, "
    "bool from_argmax) -> Tensor", _depth_corr_softmax)


# ---- glue -------------------------------------------------------------------------------------------------
def _add_position(x, table, h, w):
    _f32c(x, "x"), _f32c(table, "table")
    out = torch.empty_like(x)
    _check(LIB.um_add_position(_p(x), _p(table), _p(out), x.shape[0], h, w, table.shape[0], table.shape[1], _stream()),
           "um_add_position")
    return out


add_position = _define("add_position(Tensor x, Tensor table, int h, int w) -> Tensor", _add_position)


def _convex_upsample(flow, mask, factor, mult):
    _f32c(flow, "flow"), _f32c(mask, "mask")
    b, h, w, fd = flow.shape
    out = torch.empty((b, fd, h * factor, w * factor), device=flow.device, dtype=torch.float32)
    _check(LIB.um_convex_upsample(_p(flow), _p(mask), _p(out), b, h, w, fd, factor, float(mult), _stream()),
           "um_convex_upsample")
    return out


convex_upsample = _define("convex_upsample(Tensor flow, Tensor mask, int factor, float mult) -> Tensor", _convex_upsample)


def _upsample2x(flow, mult):
    _f32c(flow, "flow")
    b, h, w, fd = flow.shape
    out = torch.empty((b, 2 * h, 2 * w, fd), device=flow.device, dtype=torch.float32)
    _check(LIB.um_upsample2x(_p(flow), _p(out), b, h, w, fd, float(mult), _stream()), "um_upsample2x")
    return out


upsample2x = _define("upsample2x(Tensor flow, float mult) -> Tensor", _upsample2x)


def _resize_bilinear(x, h_out, w_out, scale, flip_x):
    _f32c(x, "x")
    if x.dim() != 4 or x.shape[1] > 3:
        raise RuntimeError("resize_bilinear: expected planar [B, C <= 3, H, W]")
    b, c, h, w = x.shape
    out = torch.empty((b, c, h_out, w_out), device=x.device, dtype=torch.float32)
    sc = (ctypes.c_float * c)(*scale) if scale is not None else None
    _check(LIB.um_resize_bilinear(_p(x), _p(out), b, c, h, w, h_out, w_out, sc, int(flip_x), _stream()), "um_resize_bilinear")
    return out


resize_bilinear = _define("resize_bilinear(Tensor x, int h_out, int w_out, float[]? scale, bool flip_x) -> Tensor", _resize_bilinear)


def _frames(frames, name):
    """frames: contiguous CUDA uint8 [T, H, W, 3]; returns (T, H, W)"""
    if not frames.is_cuda or frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[-1] != 3 or not frames.is_contiguous():
        raise RuntimeError("%s: expected contiguous CUDA uint8 frames [T, H, W, 3]" % name)
    return frames.shape[:3]


def _frames_to_planar(frames, h_out, w_out, transpose):
    t, h, w = _frames(frames, "frames_to_planar")
    out = torch.empty((t, 3, h_out, w_out), device=frames.device, dtype=torch.float32)
    _check(LIB.um_frames_to_planar(_p(frames), _p(out), t, h, w, int(transpose), h_out, w_out, _stream()), "um_frames_to_planar")
    return out


frames_to_planar = _define("frames_to_planar(Tensor frames, int h_out, int w_out, bool transpose) -> Tensor", _frames_to_planar)


def _frames_to_planar_normalized(frames, h_out, w_out, mean, std):
    """mean / std: 3 per-channel constants each, passed to the kernel rounded to float32"""
    t, h, w = _frames(frames, "frames_to_planar_normalized")
    if len(mean) != 3 or len(std) != 3:
        raise RuntimeError("frames_to_planar_normalized: expected 3 means and 3 stds")
    out = torch.empty((t, 3, h_out, w_out), device=frames.device, dtype=torch.float32)
    m, s = (ctypes.c_float * 3)(*mean), (ctypes.c_float * 3)(*std)
    _check(LIB.um_frames_to_planar_normalized(_p(frames), _p(out), t, h, w, h_out, w_out, m, s, _stream()),
           "um_frames_to_planar_normalized")
    return out


frames_to_planar_normalized = _define(
    "frames_to_planar_normalized(Tensor frames, int h_out, int w_out, float[] mean, float[] std) -> Tensor",
    _frames_to_planar_normalized)


def _pictures(out, x, name, what):
    """the pictures of x [N, ..., H, W]: uint8 [N, H, W, 3] on x's device with 3-byte pixels, rows and images may be strided"""
    n, h, w = x.shape[0], x.shape[-2], x.shape[-1]
    if out.dtype != torch.uint8 or tuple(out.shape) != (n, h, w, 3) or out.stride(-1) != 1 or (w > 1 and out.stride(2) != 3) \
            or out.device != x.device:
        raise RuntimeError("%s: out must be uint8 [N, H, W, 3] on the %s's device with 3-byte pixels" % (name, what))


def _flow_to_image(flow, out):
    """flow: planar [N, 2, H, W] fp32; out: uint8 [N, H, W, 3] whose pixels are 3 contiguous bytes -- rows and images may be
    strided (a view into a larger picture)."""
    _f32c(flow, "flow")
    if flow.dim() != 4 or flow.shape[1] != 2:
        raise RuntimeError("flow_to_image: expected planar flow [N, 2, H, W]")
    n, _, h, w = flow.shape
    _pictures(out, flow, "flow_to_image", "flow")
    scratch = torch.empty((n,), device=flow.device, dtype=torch.float32)
    _check(LIB.um_flow_to_image(_p(flow), _p(out), out.stride(1), out.stride(0), _p(scratch), n, h, w, _stream()),
           "um_flow_to_image")


flow_to_image = _define("flow_to_image(Tensor flow, Tensor(a!) out) -> ()", _flow_to_image)


def _disparity_to_image(disp, out):
    """disp: contiguous fp32 [N, H, W]; out: uint8 BGR [N, H, W, 3] with 3-byte pixels, rows and images may be strided."""
    _f32c(disp, "disp")
    if disp.dim() != 3:
        raise RuntimeError("disparity_to_image: expected disparities [N, H, W]")
    n, h, w = disp.shape
    _pictures(out, disp, "disparity_to_image", "disparity")
    scratch = torch.empty((2 * n,), device=disp.device, dtype=torch.float32)
    _check(LIB.um_disparity_to_image(_p(disp), _p(out), out.stride(1), out.stride(0), _p(scratch), n, h, w, _stream()),
           "um_disparity_to_image")


disparity_to_image = _define("disparity_to_image(Tensor disp, Tensor(a!) out) -> ()", _disparity_to_image)


# ---- ragged batches (include/unimatch_sm100.h, um_ragged_item) ---------------------------------------------------------
def _ragged_items(items, name):
    """items: the DEVICE descriptor table, uint8 [n, 24] (n um_ragged_item structs); returns n"""
    if not items.is_cuda or items.dtype != torch.uint8 or items.dim() != 2 or items.shape[1] != RAGGED_ITEM_BYTES \
            or not items.is_contiguous() or not 1 <= items.shape[0] <= 65535:
        raise RuntimeError("%s: items must be a contiguous CUDA uint8 table [1..65535, %d]" % (name, RAGGED_ITEM_BYTES))
    return items.shape[0]


def _frames_to_planar_normalized_ragged(frames, items, h_max, w_max, h_out, w_out, mean, std):
    """frames: contiguous CUDA uint8, the packed frames (frame i [h_i, w_i, 3] at byte items[i].offset) -> fp32 [n, 3, h_out,
    w_out]; mean / std as for frames_to_planar_normalized"""
    if not frames.is_cuda or frames.dtype != torch.uint8 or not frames.is_contiguous() or frames.numel() == 0:
        raise RuntimeError("frames_to_planar_normalized_ragged: expected contiguous CUDA uint8 packed frames")
    if len(mean) != 3 or len(std) != 3:
        raise RuntimeError("frames_to_planar_normalized_ragged: expected 3 means and 3 stds")
    n = _ragged_items(items, "frames_to_planar_normalized_ragged")
    out = torch.empty((n, 3, h_out, w_out), device=frames.device, dtype=torch.float32)
    m, s = (ctypes.c_float * 3)(*mean), (ctypes.c_float * 3)(*std)
    _check(LIB.um_frames_to_planar_normalized_ragged(_p(frames), frames.numel(), _p(items), _p(out), n, h_max, w_max, h_out,
                                                     w_out, m, s, _stream()), "um_frames_to_planar_normalized_ragged")
    return out


frames_to_planar_normalized_ragged = _define(
    "frames_to_planar_normalized_ragged(Tensor frames, Tensor items, int h_max, int w_max, int h_out, int w_out, float[] mean, "
    "float[] std) -> Tensor", _frames_to_planar_normalized_ragged)


def _resize_bilinear_ragged(x, items, h_max, w_max, out_numel):
    """x: contiguous fp32 [n, 1, h, w] -> fp32 [out_numel], item i at items[i].offset (the rest left unwritten)"""
    _f32c(x, "x")
    if x.dim() != 4 or x.shape[1] != 1:
        raise RuntimeError("resize_bilinear_ragged: expected planar [n, 1, H, W]")
    n = _ragged_items(items, "resize_bilinear_ragged")
    if x.shape[0] != n or out_numel < 1:
        raise RuntimeError("resize_bilinear_ragged: one item per image and a positive output size")
    out = torch.empty((out_numel,), device=x.device, dtype=torch.float32)
    _check(LIB.um_resize_bilinear_ragged(_p(x), _p(out), out_numel, _p(items), n, x.shape[2], x.shape[3], h_max, w_max,
                                         _stream()), "um_resize_bilinear_ragged")
    return out


resize_bilinear_ragged = _define("resize_bilinear_ragged(Tensor x, Tensor items, int h_max, int w_max, int out_numel) -> Tensor",
                                 _resize_bilinear_ragged)


def _disparity_to_image_ragged(disp, items, out, h_max, w_max):
    """disp: contiguous fp32 packed disparities (item i at items[i].offset); out: contiguous uint8 of at least 3 disp.numel()
    bytes, picture i at 3 items[i].offset"""
    _f32c(disp, "disp")
    if out.dtype != torch.uint8 or not out.is_contiguous() or out.device != disp.device or out.numel() < 3 * disp.numel():
        raise RuntimeError("disparity_to_image_ragged: out must be contiguous uint8 of 3 bytes per disparity on its device")
    n = _ragged_items(items, "disparity_to_image_ragged")
    scratch = torch.empty((2 * n,), device=disp.device, dtype=torch.float32)
    _check(LIB.um_disparity_to_image_ragged(_p(disp), disp.numel(), _p(items), _p(out), _p(scratch), n, h_max, w_max, _stream()),
           "um_disparity_to_image_ragged")


disparity_to_image_ragged = _define("disparity_to_image_ragged(Tensor disp, Tensor items, Tensor(a!) out, int h_max, int w_max) -> ()",
                                    _disparity_to_image_ragged)


def _frames_to_planar_ragged(frames, items, h_max, w_max, h_out, w_out):
    """frames: contiguous CUDA uint8, the packed frames (frame i [h_i, w_i, 3] at byte items[i].offset, read transposed with
    RAGGED_TRANSPOSE) -> fp32 [n, 3, h_out, w_out] in [0, 255]"""
    if not frames.is_cuda or frames.dtype != torch.uint8 or not frames.is_contiguous() or frames.numel() == 0:
        raise RuntimeError("frames_to_planar_ragged: expected contiguous CUDA uint8 packed frames")
    n = _ragged_items(items, "frames_to_planar_ragged")
    out = torch.empty((n, 3, h_out, w_out), device=frames.device, dtype=torch.float32)
    _check(LIB.um_frames_to_planar_ragged(_p(frames), frames.numel(), _p(items), _p(out), n, h_max, w_max, h_out, w_out,
                                          _stream()), "um_frames_to_planar_ragged")
    return out


frames_to_planar_ragged = _define(
    "frames_to_planar_ragged(Tensor frames, Tensor items, int h_max, int w_max, int h_out, int w_out) -> Tensor",
    _frames_to_planar_ragged)


def _flow_to_image_ragged(flow, flow_items, out, picture_items, h_max, w_max):
    """flow: contiguous fp32 packed planar flows (flow i [2, h_i, w_i] at float flow_items[i].offset); out: contiguous uint8,
    picture i [h_i, w_i, 3] at byte picture_items[i].offset"""
    _f32c(flow, "flow")
    if out.dtype != torch.uint8 or not out.is_contiguous() or out.device != flow.device or out.numel() == 0:
        raise RuntimeError("flow_to_image_ragged: out must be contiguous uint8 on the flow's device")
    n = _ragged_items(flow_items, "flow_to_image_ragged")
    if _ragged_items(picture_items, "flow_to_image_ragged") != n:
        raise RuntimeError("flow_to_image_ragged: one picture item per flow item")
    scratch = torch.empty((n,), device=flow.device, dtype=torch.float32)
    _check(LIB.um_flow_to_image_ragged(_p(flow), flow.numel(), _p(flow_items), _p(out), out.numel(), _p(picture_items),
                                       _p(scratch), n, h_max, w_max, _stream()), "um_flow_to_image_ragged")


flow_to_image_ragged = _define(
    "flow_to_image_ragged(Tensor flow, Tensor flow_items, Tensor(a!) out, Tensor picture_items, int h_max, int w_max) -> ()",
    _flow_to_image_ragged)


def _fb_consistency_ragged(flow, flow_items, occ, occ_items, h_max, w_max, alpha, beta):
    """flow: contiguous fp32 packed planar flows; occ: contiguous fp32 packed masks; both tables hold 2n items, pair i's
    forward flow (mask) at [i] and its backward one at [n + i]"""
    _f32c(flow, "flow"), _f32c(occ, "occ")
    n2 = _ragged_items(flow_items, "fb_consistency_ragged")
    if _ragged_items(occ_items, "fb_consistency_ragged") != n2 or n2 % 2 or occ.device != flow.device:
        raise RuntimeError("fb_consistency_ragged: two flow items and two mask items per pair, on one device")
    _check(LIB.um_fb_consistency_ragged(_p(flow), flow.numel(), _p(flow_items), float(alpha), float(beta), _p(occ), occ.numel(),
                                        _p(occ_items), n2 // 2, h_max, w_max, _stream()), "um_fb_consistency_ragged")


fb_consistency_ragged = _define(
    "fb_consistency_ragged(Tensor flow, Tensor flow_items, Tensor(a!) occ, Tensor occ_items, int h_max, int w_max, float alpha, "
    "float beta) -> ()", _fb_consistency_ragged)

DEPTH_TO_IMAGE_SCRATCH_WORDS = 2056      # per image, include/unimatch_sm100.h (um_depth_to_image)


def _depth_to_image(depth, out):
    """depth: contiguous fp32 [N, H, W]; out: uint8 RGB [N, H, W, 3] with 3-byte pixels, rows and images may be strided."""
    _f32c(depth, "depth")
    if depth.dim() != 3:
        raise RuntimeError("depth_to_image: expected depths [N, H, W]")
    n, h, w = depth.shape
    _pictures(out, depth, "depth_to_image", "depth")
    scratch = torch.empty((DEPTH_TO_IMAGE_SCRATCH_WORDS * n,), device=depth.device, dtype=torch.int32)
    _check(LIB.um_depth_to_image(_p(depth), _p(out), out.stride(1), out.stride(0), _p(scratch), n, h, w, _stream()),
           "um_depth_to_image")


depth_to_image = _define("depth_to_image(Tensor depth, Tensor(a!) out) -> ()", _depth_to_image)


def _depth_to_image_ragged(depth, items, out, h_max, w_max):
    """depth: contiguous fp32 packed depths (item i [h_i, w_i] at items[i].offset); out: contiguous uint8 of at least
    3 depth.numel() bytes, RGB picture i at 3 items[i].offset"""
    _f32c(depth, "depth")
    if out.dtype != torch.uint8 or not out.is_contiguous() or out.device != depth.device or out.numel() < 3 * depth.numel():
        raise RuntimeError("depth_to_image_ragged: out must be contiguous uint8 of 3 bytes per depth on its device")
    n = _ragged_items(items, "depth_to_image_ragged")
    scratch = torch.empty((DEPTH_TO_IMAGE_SCRATCH_WORDS * n,), device=depth.device, dtype=torch.int32)
    _check(LIB.um_depth_to_image_ragged(_p(depth), depth.numel(), _p(items), _p(out), _p(scratch), n, h_max, w_max, _stream()),
           "um_depth_to_image_ragged")


depth_to_image_ragged = _define("depth_to_image_ragged(Tensor depth, Tensor items, Tensor(a!) out, int h_max, int w_max) -> ()",
                                _depth_to_image_ragged)

# include/unimatch_sm100.h (um_encode_submission)
SUBMIT_CROP, SUBMIT_RESIZE = 0, 1
SUBMIT_FLO, SUBMIT_KITTI_FLOW_PNG, SUBMIT_KITTI_DISP_PNG, SUBMIT_PFM = 0, 1, 2, 3
SUBMIT_CHANNELS = {SUBMIT_FLO: 2, SUBMIT_KITTI_FLOW_PNG: 2, SUBMIT_KITTI_DISP_PNG: 1, SUBMIT_PFM: 1}


def submission_payload_bytes(fmt, h, w):
    """Payload bytes of one (h, w) sample in format `fmt` (PNG formats: filtered scanlines, one filter byte per row)."""
    if fmt == SUBMIT_FLO:
        return 8 * h * w
    if fmt == SUBMIT_PFM:
        return 4 * h * w
    if fmt == SUBMIT_KITTI_FLOW_PNG:
        return h * (1 + 6 * w)
    if fmt == SUBMIT_KITTI_DISP_PNG:
        return h * (1 + 2 * w)
    raise RuntimeError("encode_submission: unknown format %r" % (fmt,))


def _encode_submission(pred, fmt, out_h, out_w, resize, top, left):
    """pred: contiguous fp32 [B, C, h, w] at the inference size -> uint8 [B, bytes], each row one sample's file payload.
    `resize`: align-corners resize to (out_h, out_w) with the two-step rescale; otherwise the crop at (top, left)."""
    _f32c(pred, "pred")
    if pred.dim() != 4:
        raise RuntimeError("encode_submission: expected planar predictions [B, C, h, w]")
    if fmt not in SUBMIT_CHANNELS or pred.shape[1] != SUBMIT_CHANNELS[fmt]:
        raise RuntimeError("encode_submission: format %r needs [B, %s, h, w]" % (fmt, SUBMIT_CHANNELS.get(fmt, "?")))
    b, c, h, w = pred.shape
    nbytes = submission_payload_bytes(fmt, out_h, out_w)
    out = torch.empty((b, nbytes), device=pred.device, dtype=torch.uint8)
    _check(LIB.um_encode_submission(_p(pred), b, c, h, w, SUBMIT_RESIZE if resize else SUBMIT_CROP, top, left, out_h, out_w,
                                    fmt, _p(out), nbytes, _stream()), "um_encode_submission")
    return out


encode_submission = _define(
    "encode_submission(Tensor pred, int fmt, int out_h, int out_w, bool resize, int top, int left) -> Tensor",
    _encode_submission)


def _eval_stats(pred, gt, valid, noc_valid, task, mask_mode, max_val, eval_min, eval_max):
    """pred: flow [B, 2, h, w] or disparity / depth [B, h, w], fp32 with any non-overlapping strides (e.g. the unpadded view
    of the padded model output); gt: contiguous, same shape; valid / noc_valid: contiguous [B, h, w] or None.
    Returns the [B, S] float64 statistics table, columns EVAL_COLS[task]."""
    if task not in EVAL_COLS:
        raise RuntimeError("eval_stats: unknown task %d" % task)
    nd = 4 if task == EVAL_FLOW else 3
    if pred.dim() != nd or (nd == 4 and pred.shape[1] != 2):
        raise RuntimeError("eval_stats: expected pred [B, 2, h, w] for flow and [B, h, w] otherwise")
    if not pred.is_cuda or pred.dtype != torch.float32:
        raise RuntimeError("eval_stats: pred must be a float32 CUDA tensor")
    _f32c(gt, "gt")
    if gt.shape != pred.shape or gt.device != pred.device:
        raise RuntimeError("eval_stats: gt must have the prediction's shape and device")
    b, h, w = pred.shape[0], pred.shape[-2], pred.shape[-1]
    for t, name in ((valid, "valid"), (noc_valid, "noc_valid")):
        if t is not None:
            _f32c(t, name)
            if tuple(t.shape) != (b, h, w) or t.device != pred.device:
                raise RuntimeError("eval_stats: %s must be [B, h, w] on the prediction's device" % name)
    sb, sy, sx = pred.stride(0), pred.stride(-2), pred.stride(-1)
    sc = pred.stride(1) if nd == 4 else 0
    cols = len(EVAL_COLS[task])
    scratch = torch.empty((b * EVAL_PARTS * cols,), device=pred.device, dtype=torch.float64)
    out = torch.empty((b, cols), device=pred.device, dtype=torch.float64)
    _check(LIB.um_eval_stats(_p(pred), sb, sc, sy, sx, _p(gt), _p(valid), _p(noc_valid), task, mask_mode, float(max_val),
                             float(eval_min), float(eval_max), b, h, w, _p(scratch), _p(out), _stream()), "um_eval_stats")
    return out


eval_stats = _define(
    "eval_stats(Tensor pred, Tensor gt, Tensor? valid, Tensor? noc_valid, int task, int mask_mode, float max_val, "
    "float eval_min, float eval_max) -> Tensor", _eval_stats)


def _scene_flow_stats(disp0, disp1, flow, gt_disp0, gt_disp1, gt_flow, gt_valid, noc_disp0, noc_disp1, noc_flow, noc_valid,
                      obj_map):
    """Predictions disp0 / disp1 [B, h, w] and flow [B, 2, h, w], the occ ground truth (disparities [B, h, w], flow
    [B, 2, h, w], flow_valid [B, h, w]), the noc ground truth in the same shapes (all four or None) and obj_map [B, h, w] or
    None, all contiguous fp32 on one device.  Returns the [B, SF_COLS] float64 count table (columns `sf_col`)."""
    _f32c(disp0, "disp0")
    if disp0.dim() != 3:
        raise RuntimeError("scene_flow_stats: expected disparities [B, h, w]")
    b, h, w = disp0.shape
    noc = (noc_disp0, noc_disp1, noc_flow, noc_valid)
    if any(t is None for t in noc) and any(t is not None for t in noc):
        raise RuntimeError("scene_flow_stats: the noc set takes all four maps or none")
    for t, name, shape in ((disp1, "disp1", (b, h, w)), (flow, "flow", (b, 2, h, w)), (gt_disp0, "gt_disp0", (b, h, w)),
                           (gt_disp1, "gt_disp1", (b, h, w)), (gt_flow, "gt_flow", (b, 2, h, w)),
                           (gt_valid, "gt_valid", (b, h, w)), (noc_disp0, "noc_disp0", (b, h, w)),
                           (noc_disp1, "noc_disp1", (b, h, w)), (noc_flow, "noc_flow", (b, 2, h, w)),
                           (noc_valid, "noc_valid", (b, h, w)), (obj_map, "obj_map", (b, h, w))):
        if t is None:
            continue
        _f32c(t, name)
        if tuple(t.shape) != shape or t.device != disp0.device:
            raise RuntimeError("scene_flow_stats: %s must be %s on the predictions' device" % (name, list(shape)))

    def pair(occ, noc_t):
        return (ctypes.c_void_p * 2)(occ.data_ptr(), noc_t.data_ptr() if noc_t is not None else None)

    scratch = torch.empty((b * EVAL_PARTS * SF_COLS,), device=disp0.device, dtype=torch.float64)
    out = torch.empty((b, SF_COLS), device=disp0.device, dtype=torch.float64)
    _check(LIB.um_scene_flow_stats(_p(disp0), _p(disp1), _p(flow), pair(gt_disp0, noc_disp0), pair(gt_disp1, noc_disp1),
                                   pair(gt_flow, noc_flow), pair(gt_valid, noc_valid), _p(obj_map), b, h, w, _p(scratch),
                                   _p(out), _stream()), "um_scene_flow_stats")
    return out


scene_flow_stats = _define(
    "scene_flow_stats(Tensor disp0, Tensor disp1, Tensor flow, Tensor gt_disp0, Tensor gt_disp1, Tensor gt_flow, "
    "Tensor gt_valid, Tensor? noc_disp0, Tensor? noc_disp1, Tensor? noc_flow, Tensor? noc_valid, Tensor? obj_map) -> Tensor",
    _scene_flow_stats)


# ---- tensor-core convolution / Linear ---------------------------------------------------------------------------
def prep_conv_weight(w, cin_splits, cout_p):
    """[Cout, sum(cin_splits), KH, KW] fp32 -> fp16 planes [2, cout_p, ktot], K ordered (source, tap, ci) with every
    source's channels padded to a multiple of 64 (host-side, once per weight)."""
    cout, _, kh, kw = w.shape
    cols, off = [], 0
    for c in cin_splits:
        cp = (c + 63) // 64 * 64
        ws = w[:, off:off + c].permute(0, 2, 3, 1)                      # [Cout, KH, KW, c]
        ws = torch.nn.functional.pad(ws, (0, cp - c)).reshape(cout, kh * kw * cp)
        cols.append(ws)
        off += c
    m = torch.cat(cols, dim=1)
    m = torch.nn.functional.pad(m, (0, 0, 0, cout_p - cout)).float()
    hi = m.half()
    lo = (m - hi.float()).half()
    return torch.stack((hi, lo), dim=0).contiguous()


def split_buffer(batch, h, w, cp, device):
    """Zero-initialised fp16 (hi, lo) activation planes [2, B, h, w, cp]."""
    return torch.zeros((2, batch, h, w, cp), device=device, dtype=torch.float16)


def _split_planes(src, dst, off):
    _f32c(src, "src", rows_ok=True)
    s2 = src.flatten(0, -2)
    rows, c = s2.shape
    cp = dst.shape[-1]
    if dst.dtype != torch.float16 or not dst.is_contiguous() or dst.shape[0] != 2 or dst[0].numel() < rows * cp:
        raise RuntimeError("split_planes: dst must be contiguous fp16 planes [2, >= rows, cp]")
    _check(LIB.um_split_planes(_p(s2), rows, c, s2.stride(0), _p(dst), cp, off, dst[0].numel(), _stream()), "um_split_planes")


split_planes = _define("split_planes(Tensor src, Tensor(a!) dst, int off) -> ()", _split_planes)


def _conv2d_tc(src0, src1, weights, bias, kh, kw, pad_h, pad_w, cout, bn, mode, act, out_f32, off_f32, out_split,
               off_split, aux0, aux1, gamma=None, beta=None, stride=1, rows=0, win_dst=None, win_geom=None, win_c0=0,
               win_c1=0, win_streams=0, pre=None):
    """`rows` > 0: the sources / out_split are [2, R, cp] plane buffers of token rows and the layer runs over their first
    `rows` rows as a [rows/16, 16] pixel grid (rows % 16 == 0), the (hi, lo) planes staying R*cp halves apart.
    `win_dst` + `win_geom` (h, w, kh, kw, sh, sw, mask): output channels [win_c0, win_c1) go to the window-major operand
    planes of the tensor-core attention instead (see include/unimatch_sm100.h)."""
    d = ConvDesc()
    if rows:
        if rows % 16 or src0.dim() != 3 or rows > src0.shape[1]:
            raise RuntimeError("conv2d_tc: rows must be a multiple of 16 within the [2, R, cp] source planes")
        b, h, w, cp0 = 1, rows // 16, 16, src0.shape[-1]
        # the (hi, lo) planes may be row ranges of larger buffers (a slab of the token rows): distance = stride of dim 0
        d.src_plane_stride = src0.stride(0)
        if src1 is not None and (src1.shape[1] != src0.shape[1] or src1.stride(0) != src0.stride(0)):
            raise RuntimeError("conv2d_tc: both sources must have the same number of rows and the same plane stride")
        if out_split is not None:
            d.split_plane_stride = out_split.stride(0)
    else:
        _, b, h, w, cp0 = src0.shape
    d.src[0] = src0.data_ptr(); d.cin_p[0] = cp0
    d.nsrc = 1
    if src1 is not None:
        d.src[1] = src1.data_ptr(); d.cin_p[1] = src1.shape[-1]; d.nsrc = 2
    d.batch, d.h, d.w = b, h, w
    d.weights = weights.data_ptr()
    d.bias = bias.data_ptr() if bias is not None else None
    d.kh, d.kw, d.pad_h, d.pad_w = kh, kw, pad_h, pad_w
    d.stride = stride
    d.cout, d.cout_p, d.bn = cout, weights.shape[1], bn
    d.mode, d.act = mode, act
    if out_f32 is not None:
        _f32c(out_f32, "out_f32", rows_ok=True)
        d.out_f32 = out_f32.data_ptr(); d.ld_f32 = out_f32.stride(-2); d.off_f32 = off_f32
    if out_split is not None:
        d.out_split = out_split.data_ptr(); d.cp_split = out_split.shape[-1]; d.off_split = off_split
    if aux0 is not None:
        d.aux0 = aux0.data_ptr(); d.ld_aux0 = aux0.stride(-2)
    if aux1 is not None:
        d.aux1 = aux1.data_ptr(); d.ld_aux1 = aux1.stride(-2)
    if gamma is not None:
        d.gamma = gamma.data_ptr(); d.beta = beta.data_ptr()
    if pre is not None:
        _f32c(pre, "pre", rows_ok=True)
        d.pre = pre.data_ptr(); d.ld_pre = pre.stride(-2)
    if win_dst is not None:
        g = AttnGeom(*win_geom)
        lp = int(LIB.um_attention_planes_lp(ctypes.byref(g)))
        nops = (win_c1 - win_c0) // 128
        if win_dst.dtype != torch.float16 or not win_dst.is_contiguous() or lp == 0 or \
                win_dst.numel() != nops * 2 * win_streams * g.kh * g.kw * lp * 128:
            raise RuntimeError("conv2d_tc: win_dst must be contiguous fp16 planes [ops, 2, streams, windows, lp, 128]")
        d.win_dst = win_dst.data_ptr(); d.win_geom = g; d.win_lp = lp
        d.win_c0, d.win_c1, d.win_streams = win_c0, win_c1, win_streams
    _check(LIB.um_conv2d_tc(ctypes.byref(d), _stream()), "um_conv2d_tc")


conv2d_tc = _define(
    "conv2d_tc(Tensor src0, Tensor? src1, Tensor weights, Tensor? bias, int kh, int kw, int pad_h, int pad_w, int cout, "
    "int bn, int mode, int act, Tensor(a!)? out_f32, int off_f32, Tensor(b!)? out_split, int off_split, Tensor? aux0, "
    "Tensor? aux1, Tensor? gamma=None, Tensor? beta=None, int stride=1, int rows=0, Tensor(c!)? win_dst=None, "
    "int[]? win_geom=None, int win_c0=0, int win_c1=0, int win_streams=0, Tensor? pre=None) -> ()", _conv2d_tc)


def ffn_tc_supported(rows):
    """The fused FFN kernel works on pairs of 128-row tiles."""
    return rows > 0 and rows % 256 == 0


def _ffn_tc(src0, src1, w1, w2, residual, gamma, beta, out_f32, out_split, rows):
    """out = residual + LayerNorm(GELU([src0 | src1] W1^T) W2^T) over the first `rows` token rows (transformer.py:137-144).
    src0 / src1 / out_split: fp16 (hi, lo) planes [2, R, 128]; w1 / w2: prepared weight planes (prep_conv_weight);
    residual / out_f32: fp32 [R, 128]."""
    for t, name in ((src0, "src0"), (src1, "src1")):
        if t.dtype != torch.float16 or t.dim() != 3 or t.shape[0] != 2 or t.shape[-1] != 128 or t.stride(-1) != 1 or \
                t.stride(1) != 128 or rows > t.shape[1]:
            raise RuntimeError("ffn_tc: %s must be fp16 planes [2, R >= rows, 128]" % name)
    if src1.stride(0) != src0.stride(0):
        raise RuntimeError("ffn_tc: both sources must have the same plane stride")
    hidden = w1.shape[1]
    if w1.shape[0] != 2 or w1.shape[2] != 256 or tuple(w2.shape) != (2, 128, hidden) or not w1.is_contiguous() or not w2.is_contiguous():
        raise RuntimeError("ffn_tc: w1 must be [2, hidden, 256] and w2 [2, 128, hidden] prepared planes")
    d = FfnDesc()
    d.src[0] = src0.data_ptr(); d.src[1] = src1.data_ptr(); d.src_plane_stride = src0.stride(0)
    d.rows = rows; d.w1 = w1.data_ptr(); d.w2 = w2.data_ptr(); d.hidden = hidden
    if residual is not None:
        _f32c(residual, "residual", rows_ok=True)
        d.residual = residual.data_ptr(); d.ld_res = residual.stride(-2)
    d.gamma = gamma.data_ptr(); d.beta = beta.data_ptr()
    if out_f32 is not None:
        _f32c(out_f32, "out_f32", rows_ok=True)
        d.out_f32 = out_f32.data_ptr(); d.ld_f32 = out_f32.stride(-2)
    if out_split is not None:
        if out_split.dtype != torch.float16 or out_split.shape[0] != 2 or out_split.shape[-1] != 128 or out_split.stride(1) != 128:
            raise RuntimeError("ffn_tc: out_split must be fp16 planes [2, R, 128]")
        d.out_split = out_split.data_ptr(); d.split_plane_stride = out_split.stride(0)
    _check(LIB.um_ffn_tc(ctypes.byref(d), _stream()), "um_ffn_tc")


ffn_tc = _define(
    "ffn_tc(Tensor src0, Tensor src1, Tensor w1, Tensor w2, Tensor? residual, Tensor gamma, Tensor beta, "
    "Tensor(a!)? out_f32, Tensor(b!)? out_split, int rows) -> ()", _ffn_tc)


# ---- instance norm -----------------------------------------------------------------------------------------------
def _instance_norm_stats(x):
    """x: fp32 [N, h, w, C] channel-last (last dim contiguous) -> stats [N, 2, C] (mean, rstd)."""
    _f32c(x, "x", rows_ok=True)
    n, c = x.shape[0], x.shape[-1]
    hw = x[0].numel() // c
    scratch = torch.empty((int(LIB.um_instance_norm_scratch_floats(n, c)),), device=x.device, dtype=torch.float32)
    stats = torch.empty((n, 2, c), device=x.device, dtype=torch.float32)
    _check(LIB.um_instance_norm_stats(_p(x), x.stride(-2), n, hw, c, _p(scratch), _p(stats), _stream()),
           "um_instance_norm_stats")
    return stats


instance_norm_stats = _define("instance_norm_stats(Tensor x) -> Tensor", _instance_norm_stats)


def _instance_norm_apply(a, stats_a, relu_a, res, stats_res, relu_out, out_f32, out_split, off):
    _f32c(a, "a", rows_ok=True)
    n, c = a.shape[0], a.shape[-1]
    hw = a[0].numel() // c
    _check(LIB.um_instance_norm_apply(_p(a), a.stride(-2), _p(stats_a), int(relu_a), _p(res),
                                      res.stride(-2) if res is not None else 0, _p(stats_res), int(relu_out), _p(out_f32),
                                      out_f32.stride(-2) if out_f32 is not None else 0, _p(out_split),
                                      out_split.shape[-1] if out_split is not None else 0, off, n, hw, c, _stream()),
           "um_instance_norm_apply")


instance_norm_apply = _define(
    "instance_norm_apply(Tensor a, Tensor? stats_a, bool relu_a, Tensor? res, Tensor? stats_res, bool relu_out, "
    "Tensor(a!)? out_f32, Tensor(b!)? out_split, int off) -> ()", _instance_norm_apply)


# ---- 7x7 convolutions on 1-3 input channels -----------------------------------------------------------------------
def _conv7x7_small(in0, in1, nchw, weight, bias, stride, relu, scale, shift, out_f32, out_split):
    _f32c(in0, "in0"), _f32c(weight, "weight")
    if nchw:
        n0, cin, h, w = in0.shape
        n = n0 + (in1.shape[0] if in1 is not None else 0)
    else:
        n, h, w, cin = in0.shape
        n0 = n
    cout = weight.shape[0]
    sc = (ctypes.c_float * 3)(*scale) if scale is not None else None
    sh = (ctypes.c_float * 3)(*shift) if shift is not None else None
    _check(LIB.um_conv7x7_small(_p(in0), _p(in1), int(nchw), n0, n, h, w, cin, stride, _p(weight), _p(bias), cout, int(relu),
                                sc, sh, _p(out_f32), out_f32.stride(-2) if out_f32 is not None else 0, _p(out_split),
                                out_split.shape[-1] if out_split is not None else 0, _stream()), "um_conv7x7_small")


conv7x7_small = _define(
    "conv7x7_small(Tensor in0, Tensor? in1, bool nchw, Tensor weight, Tensor? bias, int stride, bool relu, float[]? scale, "
    "float[]? shift, Tensor(a!)? out_f32, Tensor(b!)? out_split) -> ()", _conv7x7_small)
