"""Batched inference drivers around the drop-in module (SURVEY.md section 8f rows 2-4).

Mirrors what the reference's own drivers do around `model(...)` -- `InputPadder` (utils/utils.py:6-24), the
resize-to-multiple / resize-back / rescale logic of `inference_flow` (evaluate_flow.py:711-755), `inference_stereo`
(evaluate_stereo.py:712-843, including the horizontal-flip trick for right / bidirectional disparity, :789-796, :829-836) and
`inference_depth` (evaluate_depth.py:297-419), and the forward-backward consistency check (geometry.py:75-96,
evaluate_flow.py:774-792) -- but on BATCHES of pairs that are already device tensors, with every resize (flow-component /
disparity rescale and flips folded in) as one `um_resize_bilinear` launch and the occlusion test as one fused kernel
(`um_fb_consistency`).

`BatchedFlowRunner` is the serving-side driver (evaluate_flow.py:686-760 runs one frame pair at a time): frames are padded to a
fixed bucket, host batches are staged through two pinned buffers and copied on a side stream while the previous batch
computes, and the fixed-shape forward is replayed as a CUDA graph.

Video (`main_flow.py --inference_video`, evaluate_flow.py:642-831): `infer_flow_video` runs the consecutive pairs of a frame
sequence with every frame encoded ONCE (pair (t, t+1) and pair (t+1, t+2) share frame t+1's feature pyramid; the encoder is
per-image, so the result is what `infer_flow` gives on the pairs, up to fp32 summation order), `VideoFlowRunner` streams host uint8 frames through the same
path with one upload per new frame and the previous step's last pyramid carried over, and `flow_to_image` is the Middlebury
colouring of utils/flow_viz.py on the device.  The leaderboard files (.flo, PNG, PFM) are written by `submission.py`,
and the plain inference commands' files (decoding and the `save_video` mp4 included) by `inference_io.py`.
Dense point tracks over a video (composing the reference's `flow_warp` and `forward_backward_consistency_check`,
geometry.py:41-96, frame after frame): `chain_tracks` chains device forward flows from every pixel of a first frame with the
forward occlusion masks as visibility (`um_chain_tracks`), and `VideoTrackRunner` runs that launch inside the
`VideoFlowRunner` step, so only the tracks are downloaded.  Query point tracks (TAP-Vid's question: N points, each given
at its own frame, tracked forward and backward in time through every frame of the clip): `track_points` for device flows a
caller holds, and `PointTrackRunner`, which chains them next to the `VideoFlowRunner` step and downloads only the tables
(`um_track_points_forward` / `um_track_points_backward`).  Multi-flow dense tracks (each new frame matched against several
earlier frames and the first, keeping the most certain visible candidate, so tracks come back after an occlusion):
`multi_flow_tracks` for device flows a caller holds and `MultiFlowTrackRunner`, which encodes each frame once and gathers
the source pyramids from a device ring (`um_fb_consistency_error`, `um_multi_flow_tracks`).

Posed sequences (`inference_depth`, evaluate_depth.py:297-419): `infer_depth_sequence` runs the consecutive pairs of a frame
sequence with absolute camera poses, every frame encoded once and the relative poses computed on the host as the reference
does; `DepthSequenceRunner` streams host (uint8 frame, pose) items through the same path, replayed as a CUDA graph;
`depth_to_image` is the reference's `viz_depth_tensor(1. / depth)` (inverse depth scaled by its exact 95th percentile,
matplotlib's `plasma` map, evaluate_depth.py:403-417) on the device.  Writing files (PNG) stays out of scope.

Stereo (`inference_stereo`, evaluate_stereo.py:711-843): `StereoRunner` streams host uint8 (left, right) pairs of one frame
size, normalised and resized on the device, through the same path as `infer_stereo`, replayed as a CUDA graph;
`MixedSizeStereoRunner` does the same for pairs of any size, as the reference takes each file at its own size: pairs are
batched by the size the model sees, and the input conversion, the resize back and the colouring read each pair's own size
from a device descriptor table (the `*_ragged` kernels), so one CUDA graph per inference size serves every pair that maps
to it.  `disparity_to_image` is the reference's `vis_disparity` (min-max scaling, cv2's INFERNO map) on the device.
Writing files (PNG, PFM) stays out of scope.

Flow pairs of mixed sizes (`inference_flow`, evaluate_flow.py:686-799, which takes each pair at its own size and
orientation): `MixedSizeFlowRunner` streams host uint8 (image1, image2) pairs of any size, landscape or portrait, batched by
the size the model sees after the portrait transpose; the conversion, the resize back with the two component scales and the
transpose back, the forward-backward occlusion check and the Middlebury colouring all read each pair's geometry from the
device descriptor table (`um_frames_to_planar_ragged`, `um_resize_bilinear_ragged`, `um_fb_consistency_ragged`,
`um_flow_to_image_ragged`).  It shares its buckets, graphs, packing and statistics with `MixedSizeStereoRunner`
(`_MixedSizeRunner`).

Posed depth pairs of mixed sizes (`inference_depth`, evaluate_depth.py:338-417, which takes each pair at its own size):
`MixedSizeDepthRunner` streams host (frame t, frame t+1, relative pose) items, batched by frame t's inference size, through
the same machinery; the conversion, the resize back and the colouring (`um_depth_to_image_ragged`) read each frame's size
from the descriptor table.

Stereo scene flow (KITTI 2015's disp_0 / disp_1 / flow, the stereo and flow networks together): `infer_scene_flow` runs one
stereo forward over the 2B pairs of B stereo quadruples (left0, right0, left1, right1), one flow forward on (left0, left1)
and one `um_warp_disparity`, which samples the disparity of frame t+1 where the flow carries each pixel of frame t;
`warp_disparity` is that kernel for device tensors a caller holds, and `SceneFlowRunner` streams host stereo frames with
each frame's stereo computed and its left view encoded once, in one CUDA graph per staging slot.
"""
import collections
import itertools
import math
import operator

import numpy as np
import torch
import torch.nn.functional as F

from . import ops  # noqa: F401  (registers torch.ops.unimatch_sm100.*)
from .synthetic import IMAGENET_MEAN, IMAGENET_STD

_OPS = torch.ops.unimatch_sm100


class InputPadder:
    """Replicate-pads [..., H, W] tensors so that H and W are divisible by `padding_factor`; same constructor, `pad` and
    `unpad` as the reference class (utils/utils.py:6-24): centred padding for mode 'sintel', bottom-only in height otherwise."""

    def __init__(self, dims, mode="sintel", padding_factor=8):
        self.ht, self.wd = dims[-2:]
        ph, pw = (-self.ht) % padding_factor, (-self.wd) % padding_factor
        top = ph // 2 if mode == "sintel" else 0
        self._pad = [pw // 2, pw - pw // 2, top, ph - top]

    def pad(self, *inputs):
        return [F.pad(x, self._pad, mode="replicate") for x in inputs]

    def unpad(self, x):
        h, w = x.shape[-2:]
        left, right, top, bottom = self._pad
        return x[..., top:h - bottom, left:w - right]


def forward_backward_consistency_check(fwd_flow, bwd_flow, alpha=0.01, beta=0.5):
    """geometry.py:75-96: (fwd_occ, bwd_occ), float [B,H,W], 1 = occluded.  One fused kernel over the planar flows."""
    if fwd_flow.dim() != 4 or bwd_flow.dim() != 4 or fwd_flow.size(1) != 2 or bwd_flow.size(1) != 2:
        raise ValueError("forward_backward_consistency_check expects [B,2,H,W] flows")
    return _OPS.fb_consistency(fwd_flow.contiguous(), bwd_flow.contiguous(), float(alpha), float(beta))


def _inference_size(ori, padding_factor, inference_size):
    if inference_size is None:
        return (int(math.ceil(ori[0] / padding_factor)) * padding_factor, int(math.ceil(ori[1] / padding_factor)) * padding_factor)
    return (int(inference_size[0]), int(inference_size[1]))


def _batches(samples, batch, shape_of, max_open=None):
    """Lists of samples of equal `shape_of(sample)`, at most `batch` long: one open batch per shape, flushed when full and,
    at the end, in the order the shapes were first opened.  With `max_open`, opening a batch that makes more than
    `max_open` open flushes the oldest open batch first, so at most `max_open` partial batches are held."""
    if batch < 1:
        raise ValueError("batch must be positive")
    if max_open is not None and max_open < 1:
        raise ValueError("max_open must be positive")
    open_batches = {}
    for s in samples:
        key = shape_of(s)
        if key not in open_batches and max_open is not None and len(open_batches) >= max_open:
            yield open_batches.pop(next(iter(open_batches)))
        open_batches.setdefault(key, []).append(s)
        if len(open_batches[key]) == batch:
            yield open_batches.pop(key)
    for key in list(open_batches):
        yield open_batches.pop(key)


def _resize(x, size, scale=None, flip=False):
    """[B, C<=3, H, W] -> [B, C, *size] bilinear, align_corners=True, optional per-channel scale and horizontal flip."""
    return _OPS.resize_bilinear(x.float().contiguous(), int(size[0]), int(size[1]), scale, bool(flip))


def _hflip(x):
    """torchvision hflip of a [B, C, H, W] tensor as the same kernel at unchanged size."""
    return _resize(x, x.shape[-2:], None, True)


@torch.no_grad()
def infer_flow(model, image1, image2, *, padding_factor, inference_size=None, pred_bidir_flow=False,
               fwd_bwd_consistency_check=False, **model_kwargs):
    """`inference_flow` (evaluate_flow.py:711-755, :774-792) for a batch of pairs `[B,3,H,W]` in [0,255].

    Portrait inputs are transposed (the model is trained with width > height), images are resized to the nearest
    multiple of `padding_factor` (or to `inference_size`), the flow is resized back and its components rescaled.
    Returns {'flow': [B,2,H,W]} plus 'flow_bwd' when `pred_bidir_flow` and 'fwd_occ' / 'bwd_occ' ([B,H,W], 1 = occluded)
    when `fwd_bwd_consistency_check`.  `model_kwargs` are forwarded to `model(...)` (attn_type, attn_splits_list, ...)."""
    _check_flow_args(pred_bidir_flow, fwd_bwd_consistency_check)
    model_kwargs = _task_kwargs(model_kwargs, "flow", "infer_flow")
    transposed = image1.size(-2) > image1.size(-1)
    if transposed:
        image1, image2 = image1.transpose(-2, -1), image2.transpose(-2, -1)
    ori = tuple(image1.shape[-2:])
    size = _inference_size(ori, padding_factor, inference_size)
    if size != ori:
        image1, image2 = _resize(image1, size), _resize(image2, size)
    flow = model(image1.contiguous(), image2.contiguous(), pred_bidir_flow=pred_bidir_flow, **model_kwargs)["flow_preds"][-1]
    return _flow_outputs(flow, ori, size, transposed, pred_bidir_flow, fwd_bwd_consistency_check)


def _task_kwargs(model_kwargs, task, name):
    """A copy of the model keywords without 'task' (the model's own default is "flow"; the stereo and depth paths pass
    their task themselves), refused unless it names `task`."""
    model_kwargs = dict(model_kwargs)
    if model_kwargs.pop("task", task) != task:
        raise ValueError("%s drives the %s task only" % (name, task))
    return model_kwargs


def _check_returns(return_value, visualize, option, name):
    if not return_value and not visualize:
        raise ValueError("%s: nothing to return: %s=False needs visualize=True" % (name, option))


def _check_flow_args(pred_bidir_flow, fwd_bwd_consistency_check):
    if fwd_bwd_consistency_check and not pred_bidir_flow:
        raise ValueError("fwd_bwd_consistency_check needs pred_bidir_flow=True (evaluate_flow.py:774-792)")


def _check_stereo_views(pred_bidir_disp, pred_right_disp, name):
    if pred_bidir_disp and pred_right_disp:
        raise ValueError("%s: choose one of pred_bidir_disp / pred_right_disp" % name)


def _flow_outputs(flow, ori, size, transposed, pred_bidir_flow, fwd_bwd_consistency_check):
    """The model's flow at the inference size -> the driver's outputs at the original size (evaluate_flow.py:750-792)."""
    if size != ori:                                      # resize back + rescale (u, v) by the size ratios, one launch
        flow = _resize(flow, ori, [ori[1] / size[1], ori[0] / size[0]])
    if transposed:
        flow = flow.transpose(-2, -1)       # axes only -- the reference leaves the (u, v) components in place (evaluate_flow.py:757-758)
    out = {"flow": flow}
    if pred_bidir_flow:
        half = flow.shape[0] // 2
        out["flow"], out["flow_bwd"] = flow[:half], flow[half:]
        if fwd_bwd_consistency_check:
            out["fwd_occ"], out["bwd_occ"] = forward_backward_consistency_check(out["flow"], out["flow_bwd"])
    return out


def flow_to_image(flow, out=None):
    """utils/flow_viz.py:240-275 (`flow_to_image`, what the video driver paints, evaluate_flow.py:768) on the device for a
    batch: planar flow [N,2,H,W] -> uint8 RGB [N,H,W,3], per-image normalisation by the largest radius.  `out` may be a view
    into larger pictures ([N,H,W,3] with 3-byte pixels and any row / image stride), e.g. the flow half of a frame + flow
    picture.  One max-reduction pass and one colouring pass."""
    if flow.dim() != 4 or flow.shape[1] != 2:
        raise ValueError("flow_to_image expects planar flows [N,2,H,W]")
    n, _, h, w = flow.shape
    if out is None:
        out = torch.empty((n, h, w, 3), device=flow.device, dtype=torch.uint8)
    _OPS.flow_to_image(flow.float().contiguous(), out)
    return out


def _frames_hw(frames, name):
    """(H, W) of a device sequence of T >= 2 frames: uint8 channel-last [T,H,W,3] as decoded, or float planar [T,3,H,W]."""
    if not torch.is_tensor(frames) or frames.dim() != 4 or frames.shape[0] < 2:
        raise ValueError("%s needs at least two frames [T>=2, H, W, 3] uint8 or [T>=2, 3, H, W] float" % name)
    if frames.dtype == torch.uint8:
        if frames.shape[-1] != 3:
            raise ValueError("%s: uint8 frames are channel-last [T, H, W, 3]" % name)
        return int(frames.shape[1]), int(frames.shape[2])
    if frames.dtype.is_floating_point and frames.shape[1] == 3:
        return int(frames.shape[2]), int(frames.shape[3])
    raise ValueError("%s: frames must be uint8 [T, H, W, 3] or float [T, 3, H, W]" % name)


def _frame_geometry(h, w, padding_factor, inference_size, task):
    """(transposed, original size as the model sees it, inference size) of a frame sequence.  Portrait frames are transposed
    for the flow model, which is trained with width > height (evaluate_flow.py:713-723); depth frames are not
    (evaluate_depth.py:364-376)."""
    transposed = task == "flow" and h > w
    ori = (w, h) if transposed else (h, w)
    return transposed, ori, _inference_size(ori, padding_factor, inference_size)


def _frames_to_model(frames, task, transposed, size):
    """Frames -> planar float32 [T,3,*size] model input.  uint8 [T,H,W,3] as decoded: one fused kernel (transpose and resize
    for flow; ImageNet normalisation and resize for depth, evaluate_depth.py:353-376).  Float [T,3,H,W], in [0,255] for flow
    and normalised for depth: the resize kernel, or the frames as they are at the inference size."""
    if frames.dtype == torch.uint8:
        if task == "depth":
            return _OPS.frames_to_planar_normalized(frames.contiguous(), int(size[0]), int(size[1]), list(IMAGENET_MEAN),
                                                    list(IMAGENET_STD))
        return _OPS.frames_to_planar(frames.contiguous(), int(size[0]), int(size[1]), bool(transposed))
    if transposed:
        frames = frames.transpose(-2, -1)
    return _resize(frames, size) if tuple(frames.shape[-2:]) != tuple(size) else frames.float().contiguous()


@torch.no_grad()
def infer_flow_video(model, frames, *, padding_factor, inference_size=None, pred_bidir_flow=False, pred_bwd_flow=False,
                     fwd_bwd_consistency_check=False, **model_kwargs):
    """`inference_flow(..., inference_video=...)` (evaluate_flow.py:686-792) on a device frame sequence: `frames` is
    uint8 [T,H,W,3] (channel-last, as decoded) or float [T,3,H,W] in [0,255].  Returns what
    `infer_flow(model, frames[:-1], frames[1:], ...)` returns for the T-1 consecutive pairs, with every frame encoded once
    (equal up to fp32 summation order, see `UniMatch.encode_frames`).
    `pred_bwd_flow`: each pair runs in swapped order (evaluate_flow.py:735-736), i.e. the flow from frame t+1 to frame t."""
    _check_flow_args(pred_bidir_flow, fwd_bwd_consistency_check)
    model_kwargs = _task_kwargs(model_kwargs, "flow", "infer_flow_video")
    h, w = _frames_hw(frames, "infer_flow_video")
    transposed, ori, size = _frame_geometry(h, w, padding_factor, inference_size, "flow")
    feats = model.encode_frames(_frames_to_model(frames, "flow", transposed, size))
    first, second = [f[:-1] for f in feats], [f[1:] for f in feats]
    if pred_bwd_flow:
        first, second = second, first
    flow = model.forward_encoded(first, second, pred_bidir_flow=pred_bidir_flow, **model_kwargs)["flow_preds"][-1]
    return _flow_outputs(flow, ori, size, transposed, pred_bidir_flow, fwd_bwd_consistency_check)


@torch.no_grad()
def infer_stereo(model, left, right, *, padding_factor=16, inference_size=None, pred_bidir_disp=False, pred_right_disp=False,
                 **model_kwargs):
    """`inference_stereo` (evaluate_stereo.py:776-836) for a batch of ImageNet-normalised pairs `[B,3,H,W]`.

    `pred_bidir_disp`: the right-view disparity comes from the SAME network on the mirrored, swapped pair, batched with the
    original pair (hflip trick, :789-792) and mirrored back (:829-836); `pred_right_disp`: only that.  Returns
    {'disp': [B,H,W]} (+ 'disp_right' for the bidirectional case); disparities are rescaled by the width ratio."""
    _check_stereo_views(pred_bidir_disp, pred_right_disp, "infer_stereo")
    ori = tuple(left.shape[-2:])
    size = _inference_size(ori, padding_factor, inference_size)
    if size != ori:
        left, right = _resize(left, size), _resize(right, size)
    return _stereo_outputs(model, left, right, ori, size, pred_bidir_disp, pred_right_disp, model_kwargs)


def _stereo_forward(model, left, right, pred_bidir_disp, pred_right_disp, model_kwargs):
    """Normalised pairs at the inference size -> the model's disparities [B or 2B, 1, H, W] at that size: the hflip batching
    of the right view (evaluate_stereo.py:789-796) and the forward."""
    if pred_bidir_disp:
        left, right = torch.cat((left, _hflip(right)), dim=0), torch.cat((right, _hflip(left)), dim=0)
    elif pred_right_disp:
        left, right = _hflip(right), _hflip(left)
    model_kwargs["task"] = "stereo"
    disp = model(left.float().contiguous(), right.float().contiguous(), **model_kwargs)["flow_preds"][-1]     # [B or 2B, H, W]
    return disp.unsqueeze(1)


def _stereo_outputs(model, left, right, ori, size, pred_bidir_disp, pred_right_disp, model_kwargs):
    """Normalised pairs at the inference size -> the stereo driver's outputs at the original size: the hflip batching, the
    forward, and the resize back with the width rescale and the flip back (evaluate_stereo.py:789-836)."""
    resized = size != ori
    b = left.shape[0]
    disp = _stereo_forward(model, left, right, pred_bidir_disp, pred_right_disp, model_kwargs)
    sc = [ori[1] / float(size[1])] if resized else None
    if pred_bidir_disp:
        main = _resize(disp[:b], ori, sc) if resized else disp[:b]
        other = _resize(disp[b:], ori, sc, flip=True)              # resize back, rescale and mirror back in one pass
        return {"disp": main.squeeze(1), "disp_right": other.squeeze(1)}
    if resized or pred_right_disp:
        disp = _resize(disp, ori, sc, flip=pred_right_disp)
    return {"disp": disp.squeeze(1)}


@torch.no_grad()
def _stereo_from_frames(model, frames_u8, *, padding_factor=16, inference_size=None, pred_bidir_disp=False,
                        pred_right_disp=False, **model_kwargs):
    """`infer_stereo` on B pairs given as 2B device uint8 frames [2B,H,W,3] as decoded, the B left frames then the B right
    ones.  One `um_frames_to_planar_normalized` launch normalises them as the stereo data pipeline does
    (dataloader/stereo/transforms.py:20-63: x / 255, - mean, / std in float32) and resizes them to the inference size, so the
    model sees what `infer_stereo` sees on frames normalised on the host."""
    ori = (int(frames_u8.shape[1]), int(frames_u8.shape[2]))
    size = _inference_size(ori, padding_factor, inference_size)
    planes = _OPS.frames_to_planar_normalized(frames_u8.contiguous(), int(size[0]), int(size[1]), list(IMAGENET_MEAN),
                                              list(IMAGENET_STD))
    b = frames_u8.shape[0] // 2
    return _stereo_outputs(model, planes[:b], planes[b:], ori, size, pred_bidir_disp, pred_right_disp, model_kwargs)


def disparity_to_image(disp, out=None):
    """`vis_disparity` (utils/visualization.py:11-16, what the stereo driver paints, evaluate_stereo.py:820-841) on the device
    for a batch: disparities [N,H,W] -> uint8 BGR pictures [N,H,W,3] (cv2's channel order, ready for cv2.imwrite), each image
    min-max scaled to 0..255 and coloured with cv2's INFERNO map; a single disparity [H,W] gives one picture [H,W,3].  `out`
    may be a view into larger pictures (3-byte pixels, any row / image stride).  One min / max pass and one colouring pass."""
    return _to_image(disp, out, _OPS.disparity_to_image, "disparity_to_image", "disparities")


def _to_image(x, out, op, name, what):
    """float maps [N,H,W] or [H,W] -> uint8 pictures [..., 3] through the colouring op `op(maps [N,H,W], out [N,H,W,3])`"""
    if not torch.is_tensor(x) or x.dim() not in (2, 3) or not x.dtype.is_floating_point or 0 in x.shape:
        raise ValueError("%s expects float %s [N,H,W] or [H,W]" % (name, what))
    shape = tuple(x.shape) + (3,)
    if out is None:
        out = torch.empty(shape, device=x.device, dtype=torch.uint8)
    elif not torch.is_tensor(out) or tuple(out.shape) != shape or out.dtype != torch.uint8:
        raise ValueError("%s: out must be uint8 %s" % (name, list(shape)))
    if x.dim() == 2:
        op(x[None].float().contiguous(), out[None])
    else:
        op(x.float().contiguous(), out)
    return out


@torch.no_grad()
def infer_depth(model, img_ref, img_tgt, intrinsics, pose, *, padding_factor=16, inference_size=None, min_depth=0.5,
                max_depth=10.0, num_depth_candidates=64, depth_from_argmax=False, pred_bidir_depth=False, **model_kwargs):
    """`inference_depth` (evaluate_depth.py:360-400) for a batch of ImageNet-normalised view pairs `[B,3,H,W]`,
    intrinsics `[B,3,3]` and relative poses `[B,4,4]` (target <- reference).  `min_depth` / `max_depth` are metric depths;
    the model receives their inverses, as in the reference (:389-390).  Returns {'depth': [B,H,W]} (+ 'depth_bwd')."""
    ori = tuple(img_ref.shape[-2:])
    size = _inference_size(ori, padding_factor, inference_size)
    resized = size != ori
    if resized:
        img_ref, img_tgt = _resize(img_ref, size), _resize(img_tgt, size)
    model_kwargs["task"] = "depth"
    depth = model(img_ref.float().contiguous(), img_tgt.float().contiguous(), intrinsics=intrinsics, pose=pose,
                  min_depth=1.0 / max_depth, max_depth=1.0 / min_depth, num_depth_candidates=num_depth_candidates,
                  depth_from_argmax=depth_from_argmax, pred_bidir_depth=pred_bidir_depth, **model_kwargs)["flow_preds"][-1]
    return _depth_outputs(depth, ori, size, pred_bidir_depth)


def depth_to_image(depth, out=None):
    """`viz_depth_tensor(1. / depth)` (utils/visualization.py:92-107, what the depth driver paints, evaluate_depth.py:403-417)
    on the device for a batch: depths [N,H,W] -> uint8 RGB pictures [N,H,W,3] (PIL's channel order) of the inverse depth,
    scaled from its minimum to its exact 95th percentile (np.percentile's linear interpolation) and coloured with
    matplotlib's `plasma`; a single depth [H,W] gives one picture [H,W,3].  `out` may be a view into larger pictures (3-byte
    pixels, any row / image stride).  A radix select of the two order statistics, then one colouring pass; see
    oracle/depth_viz.py for the arithmetic and the edge cases (NaN, zero or negative depths)."""
    return _to_image(depth, out, _OPS.depth_to_image, "depth_to_image", "depths")


def _colour_outputs(out, key, colour, keep):
    """Adds the picture of every output in `out` (all named `key`*) as 'vis'* ('disp_right' -> 'vis_right'), colouring with
    `colour`; the outputs themselves are dropped unless `keep`."""
    for k in list(out):
        out[k.replace(key, "vis")] = colour(out[k])
        if not keep:
            del out[k]
    return out


def _depth_outputs(depth, ori, size, pred_bidir_depth):
    """The model's depth at the inference size -> the driver's outputs at the original size (evaluate_depth.py:397-417)."""
    if size != ori:
        depth = _resize(depth.unsqueeze(1), ori).squeeze(1)
    if pred_bidir_depth:
        half = depth.shape[0] // 2
        return {"depth": depth[:half], "depth_bwd": depth[half:]}
    return {"depth": depth}


# ---------------------------------------------------------------------------------------------- depth over posed sequences
def _intrinsics33(intrinsics, name):
    """The sequence's one intrinsics matrix (the reference reads one file per sequence, evaluate_depth.py:331, :343) as float32 [3,3]."""
    if not (torch.is_tensor(intrinsics) or isinstance(intrinsics, np.ndarray)) or tuple(intrinsics.shape) != (3, 3):
        raise ValueError("%s: intrinsics must be one [3,3] matrix (tensor or numpy array)" % name)
    if not (intrinsics.dtype.is_floating_point if torch.is_tensor(intrinsics) else np.issubdtype(intrinsics.dtype, np.floating)):
        raise ValueError("%s: intrinsics must be floating point" % name)
    return torch.as_tensor(intrinsics).float()


def _pose44(pose, name):
    """An absolute camera pose on the host as float32 [4,4], as the reference loads it (np.loadtxt(...).astype(np.float32))."""
    if torch.is_tensor(pose) and pose.is_cuda:
        raise ValueError("%s: camera poses are host arrays (numpy or CPU tensors)" % name)
    p = np.asarray(pose)
    if p.shape != (4, 4) or not np.issubdtype(p.dtype, np.floating):
        raise ValueError("%s: a camera pose must be a floating-point [4,4] matrix" % name)
    return p.astype(np.float32)


def _relative_poses(poses, bidir):
    """Relative poses of the consecutive pairs of a list of absolute float32 poses [4,4], computed on the host with the
    reference's own expression, pair by pair (evaluate_depth.py:344-350): inv(pose[t+1]) @ pose[t] in numpy float32.  With
    `bidir` the inverses of those (np.linalg.inv) follow, for the backward streams: float32 [n,4,4] or [2n,4,4], the layout
    `UniMatch.depth_cameras` takes."""
    return _with_inverses([np.linalg.inv(poses[t + 1]) @ poses[t] for t in range(len(poses) - 1)], bidir)


def _world_to_camera(poses):
    """World-to-camera matrices of absolute float32 camera-to-world poses [4,4]: np.linalg.inv(pose) in numpy float32, the
    path `_relative_poses` takes, as the float32 [n,3,4] rows `um_tsdf_integrate` reads."""
    return np.ascontiguousarray(np.stack([np.linalg.inv(p) for p in poses]).astype(np.float32)[:, :3])


def _camera_to_world(poses):
    """The float32 [n,3,4] camera-to-world rows `um_tsdf_raycast` reads: the top three rows of absolute float32 poses [4,4]."""
    return np.ascontiguousarray(np.stack([np.asarray(p, np.float32) for p in poses])[:, :3])


def _with_inverses(rel, bidir):
    """Relative poses [4,4] stacked as float32 [n,4,4], followed with `bidir` by their inverses (np.linalg.inv)."""
    if bidir:
        rel = rel + [np.linalg.inv(r) for r in rel]
    return np.stack(rel).astype(np.float32)


@torch.no_grad()
def infer_depth_sequence(model, frames, intrinsics, poses, *, padding_factor=16, inference_size=None, min_depth=0.5,
                         max_depth=10.0, num_depth_candidates=64, depth_from_argmax=False, pred_bidir_depth=False,
                         **model_kwargs):
    """`inference_depth` (evaluate_depth.py:297-419) on a posed frame sequence with every frame encoded once.

    `frames`: device uint8 [T,H,W,3] as decoded (normalised and resized by one kernel) or ImageNet-normalised float
    [T,3,H,W]; `intrinsics`: the sequence's [3,3] matrix (not rescaled when the frames are resized, as in the reference);
    `poses`: the absolute camera poses [T,4,4] on the host.  The T-1 consecutive pairs (t, t+1) get the relative pose
    inv(pose[t+1]) @ pose[t], computed on the host in numpy float32 as the reference does (and its inverse there too when
    `pred_bidir_depth`).  Returns what `infer_depth` returns on those pairs: {'depth': [T-1,H,W]} (+ 'depth_bwd'), equal up to
    fp32 summation order (see `UniMatch.encode_frames`)."""
    model_kwargs = _task_kwargs(model_kwargs, "depth", "infer_depth_sequence")
    h, w = _frames_hw(frames, "infer_depth_sequence")
    T = frames.shape[0]
    if len(poses) != T:
        raise ValueError("infer_depth_sequence: %d frames need %d poses, got %d" % (T, T, len(poses)))
    abs_poses = [_pose44(p, "infer_depth_sequence") for p in poses]
    K = _intrinsics33(intrinsics, "infer_depth_sequence")
    _, ori, size = _frame_geometry(h, w, padding_factor, inference_size, "depth")
    dev = frames.device
    feats = model.encode_frames(_frames_to_model(frames, "depth", False, size), task="depth")
    rel = torch.from_numpy(_relative_poses(abs_poses, pred_bidir_depth)).to(dev)
    cams = model.depth_cameras(K.to(dev)[None].repeat(T - 1, 1, 1), rel, model.upsample_factor, 1.0 / max_depth,
                               1.0 / min_depth, num_depth_candidates, pred_bidir_depth)
    depth = model.forward_encoded([f[:-1] for f in feats], [f[1:] for f in feats], task="depth", cameras=cams,
                                  min_depth=1.0 / max_depth, max_depth=1.0 / min_depth, depth_from_argmax=depth_from_argmax,
                                  pred_bidir_depth=pred_bidir_depth, **model_kwargs)["flow_preds"][-1]
    return _depth_outputs(depth, ori, size, pred_bidir_depth)


class _PipelinedRunner:
    """Two staging slots, host->device copies on a side stream, one CUDA graph per slot, device->host copies behind the step.

    Subclasses provide `_stage_host(slot, chunk)` (fill the slot's pinned buffers and enqueue their H2D copies on the current
    stream, which is the copy stream), `_reset_inputs(slot)` and `_step(slot)` (the fixed-shape device work).  When `_step`
    returns a dict of device tensors whose first axis is the batch, the default `_download(slot, out)` (enqueue the D2H
    copies of a step's outputs into pinned buffers) and `_results(slot, n)` (one dict of host tensors per item) apply.
    Runners whose steps are not all one shape override `_chunks` (how items form steps), `_prepare_graphs` and
    `_device_step` (which graph replays a step); all capture through `_capture_graphs`."""

    def _init_pipeline(self, device, use_graph):
        self.dev = torch.device(device)
        self.copy_stream = torch.cuda.Stream(device=self.dev)
        self.graphs = [None, None]
        self.static_out = [None, None]
        self.use_graph = use_graph
        self.out_pin = [None, None]
        self._held_buffers = []
        self._staged = [None, None]                    # completion event of each slot's last H2D copies

    def _download(self, slot, out):
        if self.out_pin[slot] is None:
            self.out_pin[slot] = {k: torch.empty(v.shape, dtype=v.dtype).pin_memory() for k, v in out.items()}
        for k, v in out.items():
            self.out_pin[slot][k].copy_(v, non_blocking=True)

    def _results(self, slot, n):
        for i in range(n):
            yield {k: v[i] for k, v in self.out_pin[slot].items()}

    def _capture_graphs(self, step, reset):
        """One CUDA graph of `step(slot)` per staging slot, after the slots in `reset` are reset to valid inputs and two
        eager warm-up rounds of both slots on a side stream (they build the module's cached operand planes outside the
        capture).  Returns (graphs, outputs, held buffers): the graphs hold the raw addresses of the module's cached planes,
        and calls at other shapes may evict them from the module's caches, so the runner keeps them alive for as long as
        it may replay."""
        with torch.cuda.device(self.dev):
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for slot in reset:
                    self._reset_inputs(slot)
                for _ in range(2):
                    for slot in range(2):
                        step(slot)
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            graphs, outs = [], []
            for slot in range(2):
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    outs.append(step(slot))
                graphs.append(g)
            held = [b for m in self._graph_models() for b in m.cached_buffers()]
            torch.cuda.synchronize()
        return graphs, outs, held

    def _graph_models(self):
        """The modules a step calls, whose cached planes its graphs hold"""
        return (self.model,)

    def _stage(self, slot, chunk):
        """host side of one batch, then the H2D copies on the side stream; returns their completion event.  The slot's
        pinned buffers are refilled only once their previous copies have been read out (the copy stream may still be
        queued behind earlier device work)."""
        if self._staged[slot] is not None:
            self._staged[slot].synchronize()
        with torch.cuda.stream(self.copy_stream):
            self._stage_host(slot, chunk)
            ev = torch.cuda.Event()
            ev.record(self.copy_stream)
        self._staged[slot] = ev
        return ev

    def _prepare_graphs(self):
        """Before the first step: the one-shape runners capture both slots' graphs here."""
        if self.use_graph and self.graphs[0] is None:
            self.graphs, self.static_out, self._held_buffers = self._capture_graphs(self._step, (0, 1))

    def _chunks(self, items):
        """The steps' items: `self.batch` at a time, read as each step is staged."""
        it = iter(items)
        while True:
            chunk = list(itertools.islice(it, self.batch))
            if not chunk:
                return
            yield chunk

    def _device_step(self, slot, chunk):
        """Enqueue the device work of the step staged in `slot`; returns its outputs."""
        if self.use_graph:
            self.graphs[slot].replay()
            return self.static_out[slot]
        return self._step(slot)

    def _pipeline(self, items, start=None):
        """Yields the results of `items` taken one chunk (`_chunks`) at a time.  `start()` runs (eagerly, on the main
        stream) before the first step, after `_prepare_graphs`."""
        self._prepare_graphs()
        chunks = self._chunks(items)

        def next_chunk():
            return next(chunks, [])

        cur = next_chunk()
        if not cur:
            return
        main = torch.cuda.current_stream()
        if start is not None:
            start()
        self.copy_stream.wait_stream(main)
        ready = self._stage(0, cur)
        slot = 0
        done_ev, done_n = None, 0
        while cur:
            main.wait_event(ready)
            out = self._device_step(slot, cur)
            fwd_done = torch.cuda.Event()
            fwd_done.record(main)
            nxt = next_chunk()
            if nxt:                                        # stage the next batch while this one computes
                ready = self._stage(slot ^ 1, nxt)
            if done_ev is not None:                        # hand out the previous batch's results
                done_ev.synchronize()
                yield from self._results(slot ^ 1, done_n)
            with torch.cuda.stream(self.copy_stream):      # D2H of this batch's results behind its step
                self.copy_stream.wait_event(fwd_done)
                self._download(slot, out)
                done_ev = torch.cuda.Event()
                done_ev.record(self.copy_stream)
            done_n = len(cur)
            cur, slot = nxt, slot ^ 1
        done_ev.synchronize()
        yield from self._results(slot ^ 1, done_n)

    @torch.no_grad()
    def run(self, pairs):
        with torch.cuda.device(self.dev):
            yield from self._pipeline(pairs)


class BatchedFlowRunner(_PipelinedRunner):
    """Fixed-bucket, double-buffered, graph-replayed flow inference for a stream of host frame pairs.

    * bucket: every pair is replicate-padded (`InputPadder`, mode 'sintel') from `frame_size` up to a multiple of
      `padding_factor`; batches are always `batch` pairs (a short last batch is padded with copies of its last pair), so the
      device sees ONE shape and the forward can be captured once;
    * prefetch: two pinned host staging buffers and two device input buffers; the host->device copy of batch i+1 runs on
      a side stream while batch i computes, the device->host copy of result i overlaps batch i+1;
    * replay: the forward on the static input buffer is captured in a CUDA graph after two eager warm-up runs (which also
      build the module's cached operand planes outside the capture).

    `run(pairs)` takes an iterable of (img1, img2) CPU tensors `[3,H,W]` in [0,255] and yields unpadded flows `[2,H,W]`
    (CPU, pinned staging reused -- copy them if you keep them)."""

    def __init__(self, model, frame_size, batch, device, padding_factor=32, use_graph=True, **model_kwargs):
        self.model, self.kw, self.batch = model, dict(model_kwargs), int(batch)
        self._init_pipeline(device, use_graph)
        self.kw.setdefault("task", "flow")
        self.padder = InputPadder(frame_size, mode="sintel", padding_factor=padding_factor)
        h, w = frame_size
        left, right, top, bottom = self.padder._pad
        self.hp, self.wp = h + top + bottom, w + left + right
        shape = (self.batch, 3, self.hp, self.wp)
        self.pin = [[torch.empty(shape).pin_memory() for _ in range(2)] for _ in range(2)]       # [slot][view]
        self.dev_in = [[torch.empty(shape, device=self.dev) for _ in range(2)] for _ in range(2)]
        self.out_pin = [torch.empty((self.batch, 2, self.hp, self.wp)).pin_memory() for _ in range(2)]

    def _step(self, slot):
        a, b = self.dev_in[slot]
        return self.model(a, b, **self.kw)["flow_preds"][-1]

    def _reset_inputs(self, slot):
        self.dev_in[slot][0].zero_(); self.dev_in[slot][1].zero_()

    def _stage_host(self, slot, chunk):
        """pad into the pinned buffers, then enqueue the H2D copies"""
        for i in range(self.batch):
            img1, img2 = chunk[min(i, len(chunk) - 1)]
            p1, p2 = self.padder.pad(img1[None].float(), img2[None].float())
            self.pin[slot][0][i].copy_(p1[0]); self.pin[slot][1][i].copy_(p2[0])
        for v in range(2):
            self.dev_in[slot][v].copy_(self.pin[slot][v], non_blocking=True)

    def _download(self, slot, flow):
        self.out_pin[slot].copy_(flow, non_blocking=True)

    def _results(self, slot, n):
        for i in range(n):
            yield self.padder.unpad(self.out_pin[slot][i])


class StereoRunner(_PipelinedRunner):
    """Streaming stereo inference over host (left, right) uint8 frame pairs: `inference_stereo` (evaluate_stereo.py:711-843)
    as a stream.

    * upload: a step stages `batch` pairs into one pinned uint8 [2B,H,W,3] buffer (the B left frames, then the B right ones,
      as decoded) and copies it on a side stream while the previous step computes (3.1 MB per 544x960 pair, against 12.5 MB
      for the two float32 images);
    * device work of a step, captured once per staging slot in a CUDA graph: `_stereo_from_frames` (ImageNet normalisation
      and resize to the inference size in one `um_frames_to_planar_normalized` launch, the hflip batching of
      `pred_bidir_disp` / `pred_right_disp`, the forward, the resize back with the width rescale) and, with `visualize`,
      `disparity_to_image` on 'disp' (and 'disp_right');
    * download: 'disp' [H,W] (+ 'disp_right') and, with `visualize`, the uint8 BGR pictures 'vis' [H,W,3] (+ 'vis_right');
      `return_disp=False` with `visualize` sends back only the pictures.

    Sizes, padding, `inference_size` and the bidirectional / right-view semantics are those of `infer_stereo`.  The runner is
    built for one frame size (the reference handles each file at its own size); a short last step is filled with repeats of
    its last pair and the extra results are dropped.  `run(pairs)` takes an iterable of (left, right) host uint8 frames
    [H,W,3] (numpy arrays or tensors, RGB as PIL decodes them) and yields one dict of CPU tensors per pair (pinned staging
    reused -- copy what you keep)."""

    def __init__(self, model, frame_size, batch, device, padding_factor=16, inference_size=None, pred_bidir_disp=False,
                 pred_right_disp=False, visualize=False, return_disp=True, use_graph=True, **model_kwargs):
        _check_stereo_views(pred_bidir_disp, pred_right_disp, "StereoRunner")
        _check_returns(return_disp, visualize, "return_disp", "StereoRunner")
        self.kw = _task_kwargs(model_kwargs, "stereo", "StereoRunner")
        self.model, self.batch = model, int(batch)
        if self.batch < 1:
            raise ValueError("StereoRunner: batch must be positive")
        self.h, self.w = int(frame_size[0]), int(frame_size[1])
        self.geometry = dict(padding_factor=padding_factor, inference_size=inference_size, pred_bidir_disp=bool(pred_bidir_disp),
                             pred_right_disp=bool(pred_right_disp))
        self.visualize, self.return_disp = bool(visualize), bool(return_disp)
        self._init_pipeline(device, use_graph)
        shape = (2 * self.batch, self.h, self.w, 3)
        self.pin = [torch.empty(shape, dtype=torch.uint8).pin_memory() for _ in range(2)]
        self.dev_in = [torch.empty(shape, dtype=torch.uint8, device=self.dev) for _ in range(2)]

    def _step(self, slot):
        out = _stereo_from_frames(self.model, self.dev_in[slot], **self.geometry, **self.kw)
        return _colour_outputs(out, "disp", disparity_to_image, self.return_disp) if self.visualize else out

    def _reset_inputs(self, slot):
        self.dev_in[slot].zero_()

    def _frame(self, img):
        f = torch.as_tensor(img)
        if f.dtype != torch.uint8 or tuple(f.shape) != (self.h, self.w, 3):
            raise ValueError("StereoRunner: frames must be uint8 [%d, %d, 3]" % (self.h, self.w))
        return f

    def _stage_host(self, slot, chunk):
        """the step's left frames, then its right frames, into the pinned buffer; then their one H2D copy"""
        for i in range(self.batch):
            left, right = chunk[min(i, len(chunk) - 1)]
            self.pin[slot][i].copy_(self._frame(left))
            self.pin[slot][self.batch + i].copy_(self._frame(right))
        self.dev_in[slot].copy_(self.pin[slot], non_blocking=True)


# um_ragged_item (include/unimatch_sm100.h) as a numpy record, for building descriptor tables on the host
RAGGED_ITEM = np.dtype([("offset", "<i8"), ("h", "<i4"), ("w", "<i4"), ("scale", "<f4"), ("flags", "<i4")])
assert RAGGED_ITEM.itemsize == ops.RAGGED_ITEM_BYTES


def _frame_table(halves, batch, flags=None):
    """The 2*batch items of a step's packed uint8 frames: `halves` = (sizes of the real pairs' first frames, sizes of their
    second frames), packed back to back in that order, item i of each half with `flags[i]` (0 without `flags`).  The items
    of a short step's filler pairs point at its last pair's frames, so fillers upload nothing.  Returns (items, bytes)."""
    frames = np.zeros(2 * batch, RAGGED_ITEM)
    off = 0
    for half, sizes in enumerate(halves):
        n = len(sizes)
        for i, (h, w) in enumerate(sizes):
            frames[half * batch + i] = (off, h, w, 1.0, flags[i] if flags else 0)
            off += 3 * h * w
        frames[half * batch + n:(half + 1) * batch] = frames[half * batch + n - 1]
    return frames, off


def _scalar_outputs(keys, sizes, batch, scales=None, flags=None):
    """The len(keys)*batch items of a step's packed one-channel outputs: per key in turn, the real pairs' outputs of sizes
    `sizes` back to back, output i with scale `scales[i]` (1 without `scales`) and flags `flags[k]` of its key (0 without
    `flags`); fillers are empty items, which the kernels skip.  Returns (items, elements used, per real pair the
    (key, offset, h, w) of each of its outputs)."""
    outputs = np.zeros(len(keys) * batch, RAGGED_ITEM)
    results = [[] for _ in sizes]
    used = 0
    for k, key in enumerate(keys):
        for i, (h, w) in enumerate(sizes):
            outputs[k * batch + i] = (used, h, w, scales[i] if scales else 1.0, flags[k] if flags else 0)
            results[i].append((key, used, h, w))
            used += h * w
    return outputs, used, results


def _ragged_step_layout(sizes, batch, size, pred_bidir_disp, pred_right_disp):
    """Descriptor tables of one stereo step of `batch` pairs at the inference size `size`, whose real pairs have the
    original sizes `sizes` (1 <= len <= batch).  Returns (frames, outputs, frame_bytes, out_pixels, results):
    * frames: 2*batch items over the packed uint8 frames -- the real pairs' left frames back to back, then their right
      frames; the items of a short step's filler pairs point at its last pair's frames, so fillers upload nothing;
    * outputs: batch items ('disp'), or 2*batch with `pred_bidir_disp` ('disp', then 'disp_right'), packed back to back in
      that order; each scaled by the width ratio rounded to fp32 when its size differs from `size` (1 otherwise, as
      `_stereo_outputs` does), flipped for the right view; fillers are empty items, which the kernels skip;
    * frame_bytes / out_pixels: the used prefixes of the packed buffers;
    * results: per real pair, the (key, offset, h, w) of each of its outputs."""
    frames, nbytes = _frame_table((sizes, sizes), batch)
    keys = ("disp", "disp_right") if pred_bidir_disp else ("disp",)
    scales = [np.float32(w / float(size[1])) if (h, w) != tuple(size) else np.float32(1.0) for h, w in sizes]
    flags = [ops.RAGGED_FLIP_X if (pred_right_disp or key == "disp_right") else 0 for key in keys]
    outputs, used, results = _scalar_outputs(keys, sizes, batch, scales, flags)
    return frames, outputs, nbytes, used, results


class _MixedSizeRunner(_PipelinedRunner):
    """Streaming over host pairs of uint8 frames [h, w, 3] of ANY size up to `max_frame_size`, the part that does not depend
    on the task: steps of up to `batch` pairs of one bucket (`_batches` with `max_open=max_buckets`); per staging slot one
    pinned and one device buffer of packed uint8 frames and a descriptor table (`um_ragged_item`), of which a step uploads
    the used bytes only; one CUDA graph per bucket and staging slot, captured when the bucket first appears, the least
    recently used bucket's graphs and held buffers dropped when `max_buckets` buckets hold graphs; packed outputs of which
    the used prefixes are downloaded; `(index, result)` in completion order; `stats`.

    A subclass sets `value_key` (its value output, 'disp' / 'depth' / 'flow', of `value_planes` channels), stores its
    `visualize` and `return_<value_key>` options (`_returned`) before `_init_mixed`, and provides
    `_step(slot, size)` (the device work on `dev_in[slot]` / `dev_desc[slot]`, returning {buffer: packed device tensor}) and
    either `_step_layout(sizes, size)` (the step's frame and one-channel output tables as `_ragged_step_layout` returns them;
    `sizes` as `_sizes(pairs)` gives them) or its own `_layout(sizes, size)` (the step's descriptor table as one record
    array, the used elements of each output buffer, and per real pair its result views as (key, buffer, offset, shape)).
    The default `_bucket(pair)` (the size the model sees) is the first frame's inference size, and the default
    `_frame_order(pairs)` packs the step's first frames, then its second frames."""

    value_planes = 1

    def _init_mixed(self, model, max_frame_size, batch, device, use_graph, max_buckets, n_desc, views, extra=None):
        """`n_desc`: items of a step's table; `views`: outputs per pair and key (2 when bidirectional).  The output buffers,
        each as (dtype, elements per pixel of capacity and pair): `value_key` when returned, then `extra`, then the uint8
        RGB pictures 'vis' when returned."""
        name = type(self).__name__
        self.model, self.batch, self.max_buckets = model, int(batch), int(max_buckets)
        if self.batch < 1 or self.max_buckets < 1:
            raise ValueError("%s: batch and max_buckets must be positive" % name)
        self.hmax, self.wmax = int(max_frame_size[0]), int(max_frame_size[1])
        if self.hmax < 1 or self.wmax < 1 or self.hmax * self.wmax > 0x7fffffff:
            raise ValueError("%s: max_frame_size must be positive, at most 2^31 - 1 pixels" % name)
        out_buffers = {}
        if self._returned(self.value_key):
            out_buffers[self.value_key] = (torch.float32, self.value_planes * views)
        out_buffers.update(extra or {})
        if self._returned("vis"):
            out_buffers["vis"] = (torch.uint8, 3 * views)
        self.buffers = tuple(out_buffers)
        self._init_pipeline(device, use_graph)
        cap = self.hmax * self.wmax
        self.pin = [torch.empty((2 * self.batch * cap * 3,), dtype=torch.uint8).pin_memory() for _ in range(2)]
        self.dev_in = [torch.empty((2 * self.batch * cap * 3,), dtype=torch.uint8, device=self.dev) for _ in range(2)]
        self.desc_pin = [torch.empty((n_desc, ops.RAGGED_ITEM_BYTES), dtype=torch.uint8).pin_memory() for _ in range(2)]
        self.dev_desc = [torch.zeros((n_desc, ops.RAGGED_ITEM_BYTES), dtype=torch.uint8, device=self.dev) for _ in range(2)]
        self.out_pin = [{k: torch.empty((per * self.batch * cap,), dtype=dt).pin_memory() for k, (dt, per) in out_buffers.items()}
                        for _ in range(2)]
        self.meta = [None, None]                 # host layout of the step staged in each slot
        self.out_meta = [None, None]             # host layout of the step downloaded into each slot's pinned outputs
        self.buckets = collections.OrderedDict()  # inference size -> (graphs, outputs, held buffers), least recent first
        self.stats = {"steps": 0, "pairs": 0, "captures": 0, "h2d_bytes": 0, "d2h_bytes": 0}

    def _returned(self, buffer):
        """whether the runner returns `buffer`: 'vis' with `visualize`, the value buffer unless its constructor option
        `return_disp` / `return_flow` / `return_depth` is False"""
        return self.visualize if buffer == "vis" else getattr(self, "return_" + buffer)

    # ---- host side
    def _frame(self, frame):
        """a host frame as a uint8 [h, w, 3] tensor within the capacity"""
        name = type(self).__name__
        f = torch.as_tensor(frame)
        if f.dtype != torch.uint8 or f.dim() != 3 or f.shape[2] != 3:
            raise ValueError("%s: frames must be uint8 [h, w, 3]" % name)
        if not (1 <= f.shape[0] <= self.hmax and 1 <= f.shape[1] <= self.wmax):
            raise ValueError("%s: a %dx%d frame exceeds max_frame_size %dx%d"
                             % (name, f.shape[0], f.shape[1], self.hmax, self.wmax))
        return f

    def _pair(self, pair):
        first, second = (self._frame(f) for f in pair)
        if first.shape != second.shape:
            raise ValueError("%s: the two frames of a pair must have the same size" % type(self).__name__)
        return first, second

    def _bucket(self, pair):
        return _inference_size(tuple(pair[0].shape[:2]), self.padding_factor, self.inference_size)

    @staticmethod
    def _frame_order(pairs):
        """the step's first frames, then its second frames"""
        return [p[0] for p in pairs] + [p[1] for p in pairs]

    def _chunks(self, items):
        checked = ((i, self._pair(p)) for i, p in items)
        return _batches(checked, self.batch, lambda s: self._bucket(s[1]), self.max_buckets)

    @staticmethod
    def _sizes(pairs):
        """what `_layout` takes of each pair: its size (both frames of a pair share it)"""
        return [tuple(p[0].shape[:2]) for p in pairs]

    def _table(self, sizes, size):
        table, used, results = self._layout(sizes, size)
        return table.view(np.uint8).reshape(-1, ops.RAGGED_ITEM_BYTES), used, results

    def _layout(self, sizes, size):
        """the frame and output tables of `_step_layout`, with each output's value view and its picture's 'vis' view,
        of the buffers the runner returns"""
        frames, outputs, _, used, results = self._step_layout(sizes, size)
        key = self.value_key
        views = [[v for k, off, h, w in outs
                  for v in ((k, key, off, (h, w)), (k.replace(key, "vis"), "vis", 3 * off, (h, w, 3)))
                  if self._returned(v[1])] for outs in results]
        return np.concatenate((frames, outputs)), {key: used, "vis": 3 * used}, views

    def _stage_host(self, slot, chunk):
        """the step's packed frames and descriptor table into pinned memory, then their H2D copies (used bytes only)"""
        pairs = [p for _, p in chunk]
        size = self._bucket(pairs[0])
        table, used, results = self._table(self._sizes(pairs), size)
        nbytes = 0
        for f in self._frame_order(pairs):
            self.pin[slot][nbytes:nbytes + f.numel()].copy_(f.reshape(-1))
            nbytes += f.numel()
        self.desc_pin[slot].copy_(torch.from_numpy(table))
        self.dev_in[slot][:nbytes].copy_(self.pin[slot][:nbytes], non_blocking=True)
        self.dev_desc[slot].copy_(self.desc_pin[slot], non_blocking=True)
        self.meta[slot] = {"size": size, "used": used, "results": [(i, r) for (i, _), r in zip(chunk, results)]}
        self.stats["steps"] += 1
        self.stats["pairs"] += len(chunk)
        self.stats["h2d_bytes"] += nbytes + table.nbytes

    def _download(self, slot, out):
        meta = self.out_meta[slot] = self.meta[slot]
        for k, v in out.items():
            n = meta["used"][k]
            self.out_pin[slot][k][:n].copy_(v[:n], non_blocking=True)
            self.stats["d2h_bytes"] += n * v.element_size()

    def _results(self, slot, n):
        pins = self.out_pin[slot]
        for index, views in self.out_meta[slot]["results"][:n]:
            yield index, {key: pins[buf][off:off + math.prod(shape)].view(shape) for key, buf, off, shape in views}

    # ---- device side
    def _reset_inputs(self, slot):
        """zero frames and a full-capacity descriptor table: valid for any bucket"""
        table, _, _ = self._table([(self.hmax, self.wmax)] * self.batch, (self.hmax, self.wmax))
        self.dev_in[slot].zero_()
        self.dev_desc[slot].copy_(torch.from_numpy(table))

    def _prepare_graphs(self):
        pass                                       # graphs are captured per bucket, when it first appears

    def _capture_bucket(self, slot, size):
        """Both slots' graphs of bucket `size`, while `slot` holds a staged step of that bucket (its inputs are used as they
        are for the eager warm-up) and the other slot is free (reset to valid descriptors)."""
        entry = self._capture_graphs(lambda s: self._step(s, size), (slot ^ 1,))
        self.stats["captures"] += 1
        return entry

    def _device_step(self, slot, chunk):
        size = self.meta[slot]["size"]
        if not self.use_graph:
            return self._step(slot, size)
        entry = self.buckets.get(size)
        if entry is None:
            if len(self.buckets) >= self.max_buckets:
                torch.cuda.synchronize()           # the evicted graphs' last outputs may still be on their way to the host
                self.buckets.popitem(last=False)
            entry = self.buckets[size] = self._capture_bucket(slot, size)
        self.buckets.move_to_end(size)
        graphs, outs, _ = entry
        graphs[slot].replay()
        return outs[slot]

    def _resize_back(self, values, items, colour):
        """The model's one-channel outputs [N, 1, H, W] at the bucket size resized back into the packed `value_key`
        buffer by their output `items` (`um_resize_bilinear_ragged`), and their pictures by the ragged colouring op
        `colour` when 'vis' is returned."""
        packed = _OPS.resize_bilinear_ragged(values.contiguous(), items, self.hmax, self.wmax,
                                             items.shape[0] * self.hmax * self.wmax)
        out = {}
        if self._returned(self.value_key):
            out[self.value_key] = packed
        if self._returned("vis"):
            out["vis"] = torch.empty((3 * packed.numel(),), dtype=torch.uint8, device=self.dev)
            colour(packed, items, out["vis"], self.hmax, self.wmax)
        return out

    @torch.no_grad()
    def run(self, pairs):
        with torch.cuda.device(self.dev):
            yield from self._pipeline(enumerate(pairs))


class MixedSizeStereoRunner(_MixedSizeRunner):
    """Streaming stereo inference over host (left, right) uint8 pairs of ANY size up to `max_frame_size`:
    `inference_stereo` (evaluate_stereo.py:711-843), which takes each pair at its own size, as a stream.

    * buckets: a pair's bucket is the size the model sees, its size rounded up to a multiple of `padding_factor` or
      `inference_size` (so with `inference_size` every pair shares one bucket); a step holds up to `batch` pairs of one
      bucket, formed as the submission drivers form batches (`_batches`: one open step per bucket, sent when full; opening
      more than `max_buckets` sends the oldest open step early; the open steps are sent at the end);
    * upload: each slot has one pinned uint8 buffer of 2 * batch * H_max * W_max * 3 bytes and a small descriptor table
      (`um_ragged_item`); a step packs its left frames, then its right frames, back to back and copies only the used bytes
      and the table on a side stream while the previous step computes; a short step's fillers repeat its last pair
      without uploading it again and their results are dropped;
    * device work of a step, one CUDA graph per bucket and staging slot, captured when the bucket first appears (the least
      recently used bucket's graphs and held buffers are dropped when `max_buckets` buckets hold graphs): the ragged
      conversion (`um_frames_to_planar_normalized_ragged`: ImageNet normalisation and resize of every frame from its own
      size to the bucket's), the hflip batching and forward of `infer_stereo`, the ragged resize back with the width
      rescale and the flip back (`um_resize_bilinear_ragged`) and, with `visualize`, the ragged colouring
      (`um_disparity_to_image_ragged`); the descriptors live in device memory, so a replay reads each step's geometry;
    * download: only the used prefix of the packed disparities (and pictures).

    Sizes, padding, `inference_size` and the bidirectional / right-view semantics are those of `infer_stereo` on each pair.
    `run(pairs)` takes an iterable of (left, right) host uint8 frames [h, w, 3] (numpy arrays or tensors, RGB as PIL decodes
    them; both of a pair the same size) and yields (index, result) as steps complete -- completion order, not input order,
    so a rare bucket does not hold back later results; `index` is the pair's position in the input, each exactly once.
    `result` holds CPU views 'disp' [h, w] (+ 'disp_right') and, with `visualize`, the uint8 BGR pictures 'vis' [h, w, 3]
    (+ 'vis_right'); `return_disp=False` with `visualize` sends back only the pictures.  The views point into reused pinned
    staging -- copy what you keep.  `stats` counts steps, pairs, captures and the bytes copied each way."""

    value_key = "disp"

    def __init__(self, model, max_frame_size, batch, device, padding_factor=16, inference_size=None, pred_bidir_disp=False,
                 pred_right_disp=False, visualize=False, return_disp=True, use_graph=True, max_buckets=4, **model_kwargs):
        name = type(self).__name__
        _check_stereo_views(pred_bidir_disp, pred_right_disp, name)
        _check_returns(return_disp, visualize, "return_disp", name)
        self.kw = _task_kwargs(model_kwargs, "stereo", name)
        self.padding_factor, self.inference_size = padding_factor, inference_size
        self.bidir, self.right = bool(pred_bidir_disp), bool(pred_right_disp)
        self.visualize, self.return_disp = bool(visualize), bool(return_disp)
        views = 2 if self.bidir else 1
        self._init_mixed(model, max_frame_size, batch, device, use_graph, max_buckets, (2 + views) * int(batch), views)

    def _step_layout(self, sizes, size):
        return _ragged_step_layout(sizes, self.batch, size, self.bidir, self.right)

    def _step(self, slot, size):
        b, nf = self.batch, 2 * self.batch
        items = self.dev_desc[slot]
        planes = _OPS.frames_to_planar_normalized_ragged(self.dev_in[slot], items[:nf], self.hmax, self.wmax, int(size[0]),
                                                         int(size[1]), list(IMAGENET_MEAN), list(IMAGENET_STD))
        disp = _stereo_forward(self.model, planes[:b], planes[b:], self.bidir, self.right, dict(self.kw))
        return self._resize_back(disp, items[nf:], _OPS.disparity_to_image_ragged)


def _flow_step_layout(sizes, batch, size, pred_bidir_flow, fwd_bwd_consistency_check):
    """Descriptor tables of one flow step of `batch` pairs at the inference size `size`, whose real pairs have the original
    sizes `sizes` as stored (1 <= len <= batch; portrait pairs, h > w, carry RAGGED_TRANSPOSE: the model sees them
    transposed).  Returns (frames, planes, flows, pictures, masks, frame_bytes, used, results):
    * frames: 2*batch items over the packed uint8 frames -- the real pairs' first frames back to back, then their second
      frames; the items of a short step's filler pairs point at its last pair's frames, so fillers upload nothing;
    * planes: the resize back of the model's [D*batch, 2, H, W] flow (D = 2 with `pred_bidir_flow`: the forward flows, then
      the backward ones) taken as 2*D*batch single-channel images -- the u plane, then the v plane of each flow, packed
      back to back, so that a pair's flow is a contiguous planar [2, h, w]; scaled by the width and the height ratio of the
      pair as the model sees it, rounded to fp32, when that size differs from `size` (1 otherwise, as `_flow_outputs`
      does); fillers are empty items, which the kernels skip;
    * flows / pictures: D*batch items, each flow [2, h, w] (offset in floats) and its RGB picture (offset in bytes);
    * masks: with `fwd_bwd_consistency_check`, 2*batch items, the pairs' 'fwd_occ' [h, w], then their 'bwd_occ';
    * frame_bytes: the used prefix of the packed frames; used: {'flow': floats, 'vis': bytes, 'occ': floats};
    * results: per real pair, the (key, buffer, offset, shape) of each of its outputs."""
    frames, off = _frame_table((sizes, sizes), batch, [ops.RAGGED_TRANSPOSE if h > w else 0 for h, w in sizes])
    keys =("flow", "flow_bwd") if pred_bidir_flow else ("flow",)
    planes = np.zeros(2 * len(keys) * batch, RAGGED_ITEM)
    flows, pictures = np.zeros(len(keys) * batch, RAGGED_ITEM), np.zeros(len(keys) * batch, RAGGED_ITEM)
    masks = np.zeros(2 * batch if fwd_bwd_consistency_check else 0, RAGGED_ITEM)
    results = [[] for _ in sizes]
    used = 0                                                     # floats of flow so far; the pictures take 3 bytes per 2 floats
    for d, key in enumerate(keys):
        for i, (h, w) in enumerate(sizes):
            transposed = h > w
            ori = (w, h) if transposed else (h, w)                 # the pair as the model sees it
            su, sv = (np.float32(ori[1] / size[1]), np.float32(ori[0] / size[0])) if ori != tuple(size) else (1.0, 1.0)
            flags = ops.RAGGED_TRANSPOSE if transposed else 0
            j = d * batch + i
            planes[2 * j], planes[2 * j + 1] = (used, h, w, su, flags), (used + h * w, h, w, sv, flags)
            flows[j], pictures[j] = (used, h, w, 1.0, 0), (3 * (used // 2), h, w, 1.0, 0)
            results[i] += [(key, "flow", used, (2, h, w)), (key.replace("flow", "vis"), "vis", 3 * (used // 2), (h, w, 3))]
            used += 2 * h * w
    used_occ = 0
    for k, key in enumerate(("fwd_occ", "bwd_occ") if fwd_bwd_consistency_check else ()):
        for i, (h, w) in enumerate(sizes):
            masks[k * batch + i] = (used_occ, h, w, 1.0, 0)
            results[i].append((key, "occ", used_occ, (h, w)))
            used_occ += h * w
    return frames, planes, flows, pictures, masks, off, {"flow": used, "vis": 3 * (used // 2), "occ": used_occ}, results


class MixedSizeFlowRunner(_MixedSizeRunner):
    """Streaming optical flow over host (image1, image2) uint8 pairs of ANY size and either orientation up to
    `max_frame_size`: `inference_flow` (evaluate_flow.py:686-799), which takes each pair at its own size, as a stream.

    * buckets: a pair's bucket is the size the model sees -- the pair transposed when it is portrait (h > w,
      evaluate_flow.py:713-717), then rounded up to a multiple of `padding_factor`, or `inference_size` -- so a 480x832 and
      an 832x480 pair share a step; steps are formed as in `MixedSizeStereoRunner` (`_batches`, at most `max_buckets` open);
    * upload: the step's first frames, then its second frames, packed back to back as uint8 (2.4 MB per 480x832 pair,
      against 9.6 MB for two float32 images), the used bytes only, and the descriptor table, on a side stream while the
      previous step computes; `pred_bwd_flow` (the reference's swap, evaluate_flow.py:735-736) only changes which frame of a
      pair is packed first; a short step's fillers repeat its last pair without uploading it again;
    * device work of a step, one CUDA graph per bucket and staging slot: `um_frames_to_planar_ragged` (uint8 -> float planes,
      portrait transpose and resize of every frame from its own size to the bucket's), the forward (with
      `pred_bidir_flow`), `um_resize_bilinear_ragged` back to each pair's own size and orientation with its two component
      scales, `um_fb_consistency_ragged` on the flows at their original size with `fwd_bwd_consistency_check`, and
      `um_flow_to_image_ragged` on 'flow' (and 'flow_bwd') with `visualize`;
    * download: only the used prefixes of the packed flows, masks and pictures.

    Sizes, transpose, rescale and bidirectional semantics are those of `infer_flow` on each pair.  `max_frame_size` bounds
    the frames as stored, so (832, 832) admits both 480x832 and 832x480.  `run(pairs)` takes an iterable of (image1, image2)
    host uint8 frames [h, w, 3] (numpy arrays or tensors; both of a pair the same size) and yields (index, result) as steps
    complete -- completion order, not input order; `index` is the pair's position in the input, each exactly once.
    `result` holds CPU views 'flow' [2, h, w] (+ 'flow_bwd'; 'fwd_occ' / 'bwd_occ' [h, w], 1 = occluded) and, with
    `visualize`, the uint8 RGB pictures 'vis' [h, w, 3] (+ 'vis_bwd'); `return_flow=False` with `visualize` sends back only
    the pictures.  The views point into reused pinned staging -- copy what you keep.  `stats` counts steps, pairs, captures
    and the bytes copied each way."""

    value_key, value_planes = "flow", 2

    def __init__(self, model, max_frame_size, batch, device, padding_factor=32, inference_size=None, pred_bidir_flow=False,
                 pred_bwd_flow=False, fwd_bwd_consistency_check=False, visualize=False, return_flow=True, use_graph=True,
                 max_buckets=4, **model_kwargs):
        name = type(self).__name__
        _check_flow_args(pred_bidir_flow, fwd_bwd_consistency_check)
        self.kw = _task_kwargs(model_kwargs, "flow", name)
        _check_returns(return_flow, visualize, "return_flow", name)
        if not return_flow and fwd_bwd_consistency_check:
            raise ValueError("return_flow=False sends back pictures only: it excludes fwd_bwd_consistency_check")
        self.padding_factor, self.inference_size = padding_factor, inference_size
        self.bidir, self.bwd, self.check = bool(pred_bidir_flow), bool(pred_bwd_flow), bool(fwd_bwd_consistency_check)
        self.visualize, self.return_flow = bool(visualize), bool(return_flow)
        dirs = 2 if self.bidir else 1
        if self.check and min(max_frame_size) < 2:
            raise ValueError("MixedSizeFlowRunner: fwd_bwd_consistency_check needs frames of at least 2x2")
        self._init_mixed(model, max_frame_size, batch, device, use_graph, max_buckets,
                         (2 + 4 * dirs + (2 if self.check else 0)) * int(batch), dirs,
                         {"occ": (torch.float32, 2)} if self.check else None)

    # ---- host side
    def _pair(self, pair):
        first, second = super()._pair(pair)
        if self.check and min(first.shape[:2]) < 2:
            raise ValueError("MixedSizeFlowRunner: fwd_bwd_consistency_check needs frames of at least 2x2")
        return first, second

    def _bucket(self, pair):
        return _frame_geometry(pair[0].shape[0], pair[0].shape[1], self.padding_factor, self.inference_size, "flow")[2]

    def _frame_order(self, pairs):
        """the step's first frames, then its second frames; `pred_bwd_flow` swaps the two of every pair"""
        first, second = (1, 0) if self.bwd else (0, 1)
        return [p[first] for p in pairs] + [p[second] for p in pairs]

    def _layout(self, sizes, size):
        *tables, _, used, results = _flow_step_layout(sizes, self.batch, size, self.bidir, self.check)
        return np.concatenate(tables), used, [[v for v in views if v[1] in self.buffers] for views in results]

    # ---- device side
    def _step(self, slot, size):
        b, cap = self.batch, self.hmax * self.wmax
        nflow = (2 if self.bidir else 1) * b
        frames, planes, flows, pictures, masks = torch.split(self.dev_desc[slot], [2 * b, 2 * nflow, nflow, nflow,
                                                                                    2 * b if self.check else 0])
        x = _OPS.frames_to_planar_ragged(self.dev_in[slot], frames, self.hmax, self.wmax, int(size[0]), int(size[1]))
        flow = self.model(x[:b], x[b:], pred_bidir_flow=self.bidir, **self.kw)["flow_preds"][-1]      # [nflow, 2, H, W]
        packed = _OPS.resize_bilinear_ragged(flow.contiguous().view(2 * nflow, 1, *flow.shape[-2:]), planes, self.hmax,
                                             self.wmax, 2 * nflow * cap)
        out = {}
        if self.return_flow:
            out["flow"] = packed
        if self.check:
            out["occ"] = torch.empty((2 * b * cap,), device=self.dev)
            _OPS.fb_consistency_ragged(packed, flows, out["occ"], masks, self.hmax, self.wmax, 0.01, 0.5)
        if self.visualize:
            out["vis"] = torch.empty((3 * nflow * cap,), dtype=torch.uint8, device=self.dev)
            _OPS.flow_to_image_ragged(packed, flows, out["vis"], pictures, self.hmax, self.wmax)
        return out


class _SequenceRunner(_PipelinedRunner):
    """Consecutive pairs of a stream of host items, each holding one uint8 frame [H,W,3] as decoded, with every frame uploaded
    and encoded once: a step copies `batch` new frames through pinned double buffers on a side stream, converts and encodes
    them on the device (one CUDA graph per staging slot) and runs `_match` on the `batch` pairs (previous step's last frame,
    new frames); the last frame's pyramid (`carry`) is kept for the next step.  A short last step is filled with repeats of
    its last item and the extra results are dropped.  Subclasses set `task` and provide `_match(slot, first, second)`, which
    returns the step's dict of outputs; items with more than a frame override `_frame` and `_begin` (host state of the first
    item) and extend `_stage_host` and `_reset_inputs`."""

    def _init_sequence(self, model, frame_size, batch, device, use_graph, padding_factor, inference_size):
        self.model, self.batch = model, int(batch)
        if self.batch < 1:
            raise ValueError("%s: batch must be positive" % type(self).__name__)
        self._init_pipeline(device, use_graph)
        self.h, self.w = int(frame_size[0]), int(frame_size[1])
        self.transposed, self.ori, self.size = _frame_geometry(self.h, self.w, padding_factor, inference_size, self.task)
        shape = (self.batch, self.h, self.w, 3)
        self.pin = [torch.empty(shape, dtype=torch.uint8).pin_memory() for _ in range(2)]
        self.dev_in = [torch.empty(shape, dtype=torch.uint8, device=self.dev) for _ in range(2)]
        self.carry = None                                  # last frame's feature pyramid, [1,h,w,128] per scale

    @staticmethod
    def _frame(item):
        return item

    def _begin(self, first):
        pass

    # ---- device side
    def _encode(self, frames_u8):
        return self.model.encode_frames(_frames_to_model(frames_u8, self.task, self.transposed, self.size), task=self.task)

    def _step(self, slot):
        new = self._encode(self.dev_in[slot])
        out = self._match(slot, [torch.cat((c, f[:-1]), dim=0) for c, f in zip(self.carry, new)], new)
        for c, f in zip(self.carry, new):                # carry the last frame into the next step
            c.copy_(f[-1:])
        return out

    def _reset_inputs(self, slot):
        self.dev_in[slot].zero_()

    def _prime(self, frame):
        """Encode the sequence's first frame (eagerly) as the carried frame of the first step."""
        for c, g in zip(self.carry, self._encode(frame)):
            c.copy_(g)

    # ---- host side
    def _stage_host(self, slot, chunk):
        """the step's frames into the pinned buffer, then their H2D copy; returns the step's `batch` items"""
        items = [chunk[min(i, len(chunk) - 1)] for i in range(self.batch)]
        for i, item in enumerate(items):
            self.pin[slot][i].copy_(torch.as_tensor(self._frame(item)))
        self.dev_in[slot].copy_(self.pin[slot], non_blocking=True)
        return items

    @torch.no_grad()
    def run(self, items):
        with torch.cuda.device(self.dev):
            it = iter(items)
            first = next(it, None)
            if first is None:
                return
            frame0 = torch.as_tensor(self._frame(first))
            if tuple(frame0.shape) != (self.h, self.w, 3):
                raise ValueError("%s: frames must be uint8 [%d, %d, 3]" % (type(self).__name__, self.h, self.w))
            self._begin(first)
            frame0 = frame0.to(self.dev)[None].contiguous()
            if self.carry is None:                       # eager runs: allocate the carried pyramid
                self.carry = [f.clone() for f in self._encode(frame0)]
            yield from self._pipeline(it, start=lambda: self._prime(frame0))


class VideoFlowRunner(_SequenceRunner):
    """Streaming optical flow over a video: consecutive pairs of host uint8 frames, every frame uploaded and encoded once.

    * upload: each step copies `batch` NEW frames, uint8 [H,W,3] as decoded (1.2 MB per 480x832 frame, against 9.6 MB for
      the two float32 images of a pair);
    * device work of a step: `um_frames_to_planar` (uint8 -> float planes, portrait transpose and resize to the inference
      size in one pass), the encoder on the new frames, the matching path on the `batch` pairs, the flow resized back;
    * download: the flow (and flow_bwd / fwd_occ / bwd_occ when asked) and, with `visualize`, the uint8 Middlebury picture
      (`flow_to_image`; with `concat_frame` the frame and its picture side by side, stacked as the reference's
      `concat_flow_img` does, evaluate_flow.py:818-825).  `return_flow=False` with `visualize` sends back only the picture.
      `visualize_bwd` (with `pred_bidir_flow` and `visualize`) adds the backward flow's picture 'vis_bwd' [H,W,3];
    * `pred_bwd_flow`: every pair runs in swapped order (evaluate_flow.py:735-736), as in `infer_flow_video`; a
      `concat_frame` picture still shows the pair's first frame, as the reference's `concat_flow_img` does.

    Sizes, transpose and rescale semantics are those of `infer_flow_video` (and `infer_flow`); the flows equal
    `infer_flow_video` on the whole sequence up to fp32 summation order.  `run(frames)` takes an iterable of host uint8 frames
    [H,W,3] (numpy arrays or tensors) and yields one dict of CPU tensors per consecutive pair (pinned staging reused -- copy
    what you keep)."""

    task = "flow"

    def __init__(self, model, frame_size, batch, device, padding_factor=32, inference_size=None, use_graph=True,
                 visualize=False, concat_frame=False, pred_bidir_flow=False, fwd_bwd_consistency_check=False,
                 return_flow=True, pred_bwd_flow=False, visualize_bwd=False, **model_kwargs):
        name = type(self).__name__
        _check_flow_args(pred_bidir_flow, fwd_bwd_consistency_check)
        self.kw = _task_kwargs(model_kwargs, "flow", name)
        if concat_frame and not visualize:
            raise ValueError("concat_frame needs visualize=True")
        if visualize_bwd and not (visualize and pred_bidir_flow):
            raise ValueError("visualize_bwd needs visualize=True and pred_bidir_flow=True")
        _check_returns(return_flow, visualize, "return_flow", name)
        self._init_sequence(model, frame_size, batch, device, use_graph, padding_factor, inference_size)
        self.bidir, self.check = bool(pred_bidir_flow), bool(fwd_bwd_consistency_check)
        self.visualize, self.concat, self.return_flow = bool(visualize), bool(concat_frame), bool(return_flow)
        self.bwd, self.visualize_bwd = bool(pred_bwd_flow), bool(visualize_bwd)
        self.concat_axis = 0 if self.h < self.w else 1                                  # evaluate_flow.py:822
        self.carry_frame = torch.zeros((1, self.h, self.w, 3), dtype=torch.uint8, device=self.dev)

    def _match(self, slot, first, second):
        if self.bwd:
            first, second = second, first
        flow = self.model.forward_encoded(first, second, pred_bidir_flow=self.bidir, **self.kw)["flow_preds"][-1]
        out = _flow_outputs(flow, self.ori, self.size, self.transposed, self.bidir, self.check)
        if self.visualize:
            b, h, w = self.batch, self.h, self.w
            if self.concat:
                pics = torch.empty((b, 2 * h, w, 3) if self.concat_axis == 0 else (b, h, 2 * w, 3), dtype=torch.uint8,
                                   device=self.dev)
                frame_half, flow_half = (pics[:, :h], pics[:, h:]) if self.concat_axis == 0 else (pics[:, :, :w], pics[:, :, w:])
                frame_half.copy_(torch.cat((self.carry_frame, self.dev_in[slot][:-1]), dim=0))   # first frame of each pair
            else:
                pics = flow_half = torch.empty((b, h, w, 3), dtype=torch.uint8, device=self.dev)
            flow_to_image(out["flow"], flow_half)
            out["vis"] = pics
            if self.visualize_bwd:
                out["vis_bwd"] = flow_to_image(out["flow_bwd"])
            if not self.return_flow:
                del out["flow"]
                if self.visualize_bwd:
                    del out["flow_bwd"]
        self.carry_frame.copy_(self.dev_in[slot][-1:])
        return out

    def _prime(self, frame):
        super()._prime(frame)
        self.carry_frame.copy_(frame)


def _track_start(h, w, device):
    """Tracks at every pixel of the first frame: pos [H,W,2] = (x, y), all visible."""
    ys, xs = torch.meshgrid(torch.arange(h, device=device, dtype=torch.float32),
                            torch.arange(w, device=device, dtype=torch.float32), indexing="ij")
    return torch.stack((xs, ys), dim=-1).contiguous(), torch.ones((h, w), device=device, dtype=torch.uint8)


def _track_flags(model_kwargs, name, reason):
    """Takes out of a track runner's keywords the `VideoFlowRunner` flags it fixes: the ones that would change which
    flows it chains are refused (`reason` says why), and the bidirectional flow with its occlusion masks is always on."""
    for k in ("pred_bwd_flow", "visualize", "concat_frame", "visualize_bwd"):
        if model_kwargs.pop(k, False):
            raise ValueError("%s: %s is not supported (%s)" % (name, k, reason))
    for k in ("pred_bidir_flow", "fwd_bwd_consistency_check"):
        if not model_kwargs.pop(k, True):
            raise ValueError("%s: %s is always on (the occlusion masks decide visibility)" % (name, k))


@torch.no_grad()
def chain_tracks(flows, occ=None, state=None):
    """Dense point tracks through the forward flows of consecutive pairs, one `um_chain_tracks` launch.

    `flows`: device planar [N,2,H,W], the forward flow of pair (t-1, t) at index t-1 in pixels at the frames' size (e.g.
    `infer_flow_video(...)['flow']`); `occ`: its forward occlusion masks [N,H,W] (`'fwd_occ'`, 1 = occluded) or None
    (nothing occluded).  `state`: (pos fp32 [H,W,2], vis uint8 [H,W]), contiguous on the flows' device and advanced in place,
    or None: the tracks start at every pixel, pos(y, x) = (x, y), all visible.  Per flow, with F the flow and O the mask:
    d = bilinear(F, p), o = bilinear(O, p) (the reference's `bilinear_sample`: pixel coordinates, align_corners=True, zero
    padding), p = p + d, and the track stays visible while o < 0.5 and p lies in [0, W-1] x [0, H-1]; an invisible track stays
    invisible and is still moved.  fp32, with the order of operations of include/unimatch_sm100.h.
    Returns {'tracks': [N,H,W,2] fp32 (x, y), 'visible': [N,H,W] uint8}, the state after each flow.  To continue with the
    flows that follow, pass state=(tracks[-1].clone(), visible[-1].clone())."""
    if flows.dim() != 4 or flows.shape[1] != 2 or flows.shape[0] < 1:
        raise ValueError("chain_tracks expects at least one planar flow [N,2,H,W]")
    n, _, h, w = flows.shape
    if occ is not None and tuple(occ.shape) != (n, h, w):
        raise ValueError("chain_tracks: occ must be [N,H,W] like the flows")
    if state is None:
        state = _track_start(h, w, flows.device)
    pos, vis = state
    if tuple(pos.shape) != (h, w, 2) or tuple(vis.shape) != (h, w):
        raise ValueError("chain_tracks: the state is (pos [H,W,2], vis [H,W]) at the flows' size")
    tracks, visible = _OPS.chain_tracks(flows.float().contiguous(), None if occ is None else occ.float().contiguous(), pos,
                                        vis)
    return {"tracks": tracks, "visible": visible}


class VideoTrackRunner(VideoFlowRunner):
    """Dense point tracks over a video: where each pixel of the first frame of a `run()` is in every later frame, and whether
    it is still visible, chained on the device inside the `VideoFlowRunner` step.

    The step computes the forward and backward flows and the forward-backward occlusion masks (`pred_bidir_flow` and
    `fwd_bwd_consistency_check` are always on) at the frames' original size and orientation, then one `um_chain_tracks`
    launch advances every track through the step's `batch` forward flows in order (semantics: `chain_tracks`).  The track
    state lives in device buffers that persist across steps and is reset at the start of each `run()`, so the tracks do
    not depend on `batch` beyond the encoder's summation order in the flows themselves.
    `run(frames)` yields, per frame t >= 1, 'tracks' fp32 [H,W,2] (x, y in pixels) and 'visible' uint8 [H,W]: 9 bytes per
    pixel downloaded (3.6 MB per 480x832 frame), against 12 for the forward flow and its mask.  `return_flow=True` adds the
    'flow', 'flow_bwd', 'fwd_occ' and 'bwd_occ' that `VideoFlowRunner(pred_bidir_flow=True, fwd_bwd_consistency_check=True)`
    returns.  `pred_bwd_flow`, `visualize`, `concat_frame` and `visualize_bwd` are refused: the tracks run forward from the
    first frame."""

    def __init__(self, model, frame_size, batch, device, padding_factor=32, inference_size=None, use_graph=True,
                 return_flow=False, **model_kwargs):
        _track_flags(model_kwargs, "VideoTrackRunner", "tracks run forward from the first frame")
        super().__init__(model, frame_size, batch, device, padding_factor=padding_factor, inference_size=inference_size,
                         use_graph=use_graph, pred_bidir_flow=True, fwd_bwd_consistency_check=True, **model_kwargs)
        self.return_flow = bool(return_flow)
        self.track_origin, self.track_vis = _track_start(self.h, self.w, self.dev)
        self.track_pos = self.track_origin.clone()

    def _match(self, slot, first, second):
        out = super()._match(slot, first, second)
        tracks, visible = _OPS.chain_tracks(out["flow"].contiguous(), out["fwd_occ"], self.track_pos, self.track_vis)
        out = out if self.return_flow else {}
        out["tracks"], out["visible"] = tracks, visible
        return out

    def _prime(self, frame):
        super()._prime(frame)
        self.track_pos.copy_(self.track_origin)
        self.track_vis.fill_(1)


def _point_queries(queries, h, w, name):
    """Host float32 [N,3] (t_q, y, x) of TAP-Vid's `query_points`, refused unless t_q is a non-negative integer and (x, y)
    is finite and inside [0, W-1] x [0, H-1]."""
    q = torch.as_tensor(queries).detach().to("cpu", torch.float32)
    if q.dim() != 2 or q.shape[1] != 3 or q.shape[0] < 1:
        raise ValueError("%s: queries must be [N, 3] (t_q, y, x) with N >= 1" % name)
    bad = ~torch.isfinite(q).all(dim=1)
    bad |= (q[:, 0] < 0) | (q[:, 0] != torch.floor(q[:, 0]))
    bad |= (q[:, 1] < 0) | (q[:, 1] > h - 1) | (q[:, 2] < 0) | (q[:, 2] > w - 1)
    if bad.any():
        i = int(bad.nonzero()[0])
        raise ValueError("%s: query %d (t_q, y, x) = %s needs a finite (x, y) inside the %dx%d frame and an integer "
                         "t_q >= 0" % (name, i, tuple(q[i].tolist()), h, w))
    return q


def _late_query(q, nframes, name):
    late = (q[:, 0] >= nframes).nonzero()
    if len(late):
        i = int(late[0])
        raise ValueError("%s: query %d is given at frame %d of a clip of %d frames" % (name, i, int(q[i, 0]), nframes))


@torch.no_grad()
def track_points(flows, flows_bwd, fwd_occ, bwd_occ, queries):
    """Query point tracks through device flows a caller already holds, forward and backward in time from each query's frame.

    `flows` / `flows_bwd`: planar [T-1,2,H,W], the forward flow of pair (t, t+1) and its backward flow (frame t+1 -> t) at
    index t, in pixels at the frames' size (e.g. `infer_flow_video(..., pred_bidir_flow=True,
    fwd_bwd_consistency_check=True)`'s 'flow' and 'flow_bwd'); `fwd_occ` / `bwd_occ`: their occlusion masks [T-1,H,W]
    (1 = occluded) or None (nothing occluded).  `queries`: [N,3] (t_q, y, x), TAP-Vid's `query_points` layout, t_q an integer
    frame index and (x, y) pixels with pixel centres at integers, inside the frame.
    At t_q a track is the query, visible.  Forward (t > t_q) it is `chain_tracks`'s step through pair (t-1, t)'s forward
    flow and `fwd_occ`; backward (t < t_q) the same step through pair (t, t+1)'s backward flow and `bwd_occ`.  One
    `um_track_points_forward` and one `um_track_points_backward` launch.
    Returns {'tracks': [N,T,2] fp32 (x, y), 'visible': [N,T] uint8} on the flows' device."""
    if flows.dim() != 4 or flows.shape[1] != 2 or flows.shape[0] < 1:
        raise ValueError("track_points expects the forward flows of at least one pair, planar [T-1,2,H,W]")
    n, _, h, w = flows.shape
    if tuple(flows_bwd.shape) != tuple(flows.shape):
        raise ValueError("track_points: flows_bwd must be [T-1,2,H,W] like the flows")
    for name, occ in (("fwd_occ", fwd_occ), ("bwd_occ", bwd_occ)):
        if occ is not None and tuple(occ.shape) != (n, h, w):
            raise ValueError("track_points: %s must be [T-1,H,W] like the flows" % name)
    q = _point_queries(queries, h, w, "track_points")
    _late_query(q, n + 1, "track_points")
    dev = flows.device
    nq, tmax = q.shape[0], int(q[:, 0].max())
    qd = q.to(dev)
    tracks = torch.empty((nq, n + 1, 2), device=dev, dtype=torch.float32)
    visible = torch.empty((nq, n + 1), device=dev, dtype=torch.uint8)
    pos = torch.empty((nq, 2), device=dev, dtype=torch.float32)
    vis = torch.empty((nq,), device=dev, dtype=torch.uint8)

    def f32(t):
        return None if t is None else t.float().contiguous()
    _OPS.track_points_forward(f32(flows), f32(fwd_occ), 0, qd, pos, vis, tracks, visible)
    _OPS.track_points_backward(f32(flows_bwd[:tmax]), None if bwd_occ is None else f32(bwd_occ[:tmax]), qd, tracks, visible)
    return {"tracks": tracks, "visible": visible}


class PointTrackRunner(VideoFlowRunner):
    """Query point tracks over a video: for N query points, each given at its own frame t_q, where the point is in every
    frame of the clip, before and after t_q, and whether it is visible there (TAP-Vid's question).

    The step is `VideoFlowRunner`'s with `pred_bidir_flow` and `fwd_bwd_consistency_check` always on.  After each step's
    device work (graph replay or eager), on the same stream and outside the graph because the frame offset changes every
    step: one `um_track_points_forward` launch advances every query from its frame through the step's real pairs (the
    repeats that fill a short last step are never chained), and the backward flows and masks of the step's pairs below
    max(t_q) are copied into a device history.  When the stream ends, one `um_track_points_backward` launch walks every
    query from t_q back to frame 0 through that history, and the tables are downloaded once: N x T x 9 bytes.  Semantics:
    `track_points`, which gives the same tracks on the runner's own flows bit for bit.
    The history holds max(t_q) x 12 x H x W bytes (4.8 MB per pair at 480x832), allocated when `track()` starts and
    released when it ends; queries all at frame 0 need none.
    `track(frames, queries)` takes an iterable of at least two host uint8 frames [H,W,3] and queries [N,3] (t_q, y, x) as in
    `track_points`, and returns {'tracks': [N,T,2] fp32, 'visible': [N,T] uint8} on the host; `return_flow=True` adds the
    per-pair 'flow', 'flow_bwd', 'fwd_occ' and 'bwd_occ' [T-1, ...] that `VideoFlowRunner` returns, stacked (for tests and
    short clips).  `pred_bwd_flow`, `visualize`, `concat_frame` and `visualize_bwd` are refused."""

    def __init__(self, model, frame_size, batch, device, padding_factor=32, inference_size=None, use_graph=True,
                 return_flow=False, **model_kwargs):
        _track_flags(model_kwargs, "PointTrackRunner", "the tracks need the forward and backward flows of every pair")
        super().__init__(model, frame_size, batch, device, padding_factor=padding_factor, inference_size=inference_size,
                         use_graph=use_graph, pred_bidir_flow=True, fwd_bwd_consistency_check=True, **model_kwargs)
        self.return_flow = bool(return_flow)
        self._pts = None

    def _reserve(self, nframes):
        """grow the device tables to at least `nframes` columns (doubling), keeping what is written"""
        s = self._pts
        cap = s["tracks"].shape[1]
        if nframes <= cap:
            return
        cap = max(nframes, 2 * cap)
        for k, shape in (("tracks", (s["nq"], cap, 2)), ("visible", (s["nq"], cap))):
            grown = torch.empty(shape, device=self.dev, dtype=s[k].dtype)
            grown[:, :s[k].shape[1]].copy_(s[k])
            s[k] = grown

    def _device_step(self, slot, chunk):
        s = self._pts
        if s is None:
            raise RuntimeError("PointTrackRunner: call track(frames, queries), not run(frames)")
        out = super()._device_step(slot, chunk)
        t0, n = s["pairs"], len(chunk)
        self._reserve(t0 + n + 1)
        keep = min(n, s["tmax"] - t0)
        if keep > 0:                       # backward flows and masks of the pairs below max(t_q)
            s["flow_bwd"][t0:t0 + keep].copy_(out["flow_bwd"][:keep])
            s["bwd_occ"][t0:t0 + keep].copy_(out["bwd_occ"][:keep])
        _OPS.track_points_forward(out["flow"][:n].contiguous(), out["fwd_occ"][:n].contiguous(), t0, s["queries"], s["pos"],
                                  s["vis"], s["tracks"], s["visible"])
        s["pairs"] = t0 + n
        return out if self.return_flow else {}

    @torch.no_grad()
    def track(self, frames, queries):
        q = _point_queries(queries, self.h, self.w, "PointTrackRunner")
        it = iter(frames)
        head = list(itertools.islice(it, 2))
        if len(head) < 2:
            raise ValueError("PointTrackRunner: a clip needs at least two frames")
        nq, tmax = q.shape[0], int(q[:, 0].max())
        size = len(frames) if hasattr(frames, "__len__") else 0
        with torch.cuda.device(self.dev):
            dev, hw = self.dev, (self.h, self.w)
            self._pts = {"nq": nq, "tmax": tmax, "pairs": 0, "queries": q.to(dev),
                         "pos": torch.empty((nq, 2), device=dev), "vis": torch.empty((nq,), device=dev, dtype=torch.uint8),
                         "tracks": torch.empty((nq, max(size, tmax + 1, 2), 2), device=dev),
                         "visible": torch.empty((nq, max(size, tmax + 1, 2)), device=dev, dtype=torch.uint8),
                         "flow_bwd": torch.empty((tmax, 2) + hw, device=dev), "bwd_occ": torch.empty((tmax,) + hw, device=dev)}
            try:
                per_pair = [{k: v.clone() for k, v in r.items()} for r in self.run(itertools.chain(head, it))]
                s = self._pts
                nframes = s["pairs"] + 1
                _late_query(q, nframes, "PointTrackRunner")
                _OPS.track_points_backward(s["flow_bwd"], s["bwd_occ"], s["queries"], s["tracks"], s["visible"])
                res = {"tracks": s["tracks"][:, :nframes].contiguous().cpu(),
                       "visible": s["visible"][:, :nframes].contiguous().cpu()}
            finally:
                self._pts = None
        if self.return_flow:
            res.update({k: torch.stack([r[k] for r in per_pair]) for k in ("flow", "flow_bwd", "fwd_occ", "bwd_occ")})
        return res


MULTI_FLOW_GAPS = (1, 2, 4, 8, 16, 32)


def _multi_flow_gaps(gaps, anchor, name):
    """(the gaps in increasing order, anchor), refused unless the gaps are distinct positive integers and some source
    exists"""
    try:
        g = sorted(operator.index(x) for x in gaps)
    except TypeError:
        raise ValueError("%s: gaps must be integers, got %r" % (name, gaps)) from None
    if any(x < 1 for x in g) or len(set(g)) != len(g):
        raise ValueError("%s: gaps must be distinct positive integers, got %r" % (name, tuple(gaps)))
    if not g and not anchor:
        raise ValueError("%s: no source at all: give gaps or anchor=True" % name)
    return tuple(g), bool(anchor)


def multi_flow_sources(t, gaps=MULTI_FLOW_GAPS, anchor=True):
    """The candidate source frames of frame t >= 1 of a multi-flow track, in candidate-slot order: frame t-g for each g in
    `gaps` in increasing order (-1, absent, where t-g < 0), then frame 0 when `anchor`.  len(gaps) + anchor slots; frame 0
    may appear twice (as gap t and as the anchor).  A frame without any present source is refused."""
    gaps, anchor = _multi_flow_gaps(gaps, anchor, "multi_flow_sources")
    t = operator.index(t)
    if t < 1:
        raise ValueError("multi_flow_sources: frame %d has no sources (frames t >= 1 have)" % t)
    src = [t - g if t >= g else -1 for g in gaps] + ([0] if anchor else [])
    if max(src) < 0:
        raise ValueError("multi_flow_sources: frame %d has no source with gaps %r and anchor=False" % (t, gaps))
    return src


def _multi_flow_state(slots, h, w, device):
    """The state ring (pos [R,H,W,2], sigma^2 [R,H,W], vis [R,H,W] uint8) with frame 0 in slot 0: every pixel at itself,
    certain and visible"""
    pos = torch.empty((slots, h, w, 2), device=device)
    sig = torch.empty((slots, h, w), device=device)
    vis = torch.empty((slots, h, w), device=device, dtype=torch.uint8)
    pos[0], _ = _track_start(h, w, device)
    sig[0] = 0
    vis[0] = 1
    return pos, sig, vis


@torch.no_grad()
def multi_flow_tracks(flows, flows_bwd, gaps=MULTI_FLOW_GAPS, anchor=True):
    """Multi-flow dense point tracks through device flows a caller already holds: every pixel of frame 0, each frame t >= 1
    reached from its sources (`multi_flow_sources(t, gaps, anchor)`: frames t-g and, with `anchor`, frame 0), keeping the
    most certain candidate that is not occluded, so a point comes back after an occlusion (multi-flow tracking after MFT,
    Neoral, Serych and Matas, WACV 2024).

    `flows` / `flows_bwd`: planar [T-1,K,2,H,W], K = len(gaps) + anchor; entry (t-1, k) is the forward flow of pair
    (source k of t, t) and its backward flow, in pixels at the frames' size (e.g. `infer_flow(..., pred_bidir_flow=True)` on
    those pairs).  Entries of absent sources do not affect the result.  Per pair, O = `fwd_occ` of
    `forward_backward_consistency_check` and E the forward residual that mask thresholds (`um_fb_consistency_error`).  From
    source s's state (x_s, sigma2_s, v_s), with `chain_tracks`'s bilinear sampling: x = x_s + F(x_s), sigma2 = sigma2_s +
    E(x_s)^2, valid = v_s and O(x_s) < 0.5 and x inside the frame.  Frame t takes the valid candidate of smallest sigma2
    (the first on ties) and is visible; with none valid, the smallest sigma2 of all, invisible.  Frame 0: x = p,
    sigma2 = 0, visible.  fp32 in the order of operations of include/unimatch_sm100.h.  One `um_fb_consistency_error`
    call, one `um_multi_flow_tracks` launch, and a state of 13 x T x H x W bytes for the call.
    Returns {'tracks': [T-1,H,W,2] fp32 (x, y), 'visible': [T-1,H,W] uint8, 'uncertainty': [T-1,H,W] fp32 sigma^2} for
    frames 1 .. T-1."""
    gaps, anchor = _multi_flow_gaps(gaps, anchor, "multi_flow_tracks")
    k = len(gaps) + anchor
    if flows.dim() != 5 or flows.shape[0] < 1 or flows.shape[1] != k or flows.shape[2] != 2:
        raise ValueError("multi_flow_tracks expects planar flows [T-1,%d,2,H,W] (K = len(gaps) + anchor), got %s"
                         % (k, tuple(flows.shape)))
    if tuple(flows_bwd.shape) != tuple(flows.shape):
        raise ValueError("multi_flow_tracks: flows_bwd must be [T-1,K,2,H,W] like the flows")
    n, _, _, h, w = flows.shape
    dev = flows.device
    src = torch.tensor([multi_flow_sources(t, gaps, anchor) for t in range(1, n + 1)], dtype=torch.int32).to(dev)
    dst = torch.arange(1, n + 1, dtype=torch.int32, device=dev)
    fwd = flows.float().reshape(n * k, 2, h, w).contiguous()
    occ, _, err = _OPS.fb_consistency_error(fwd, flows_bwd.float().reshape(n * k, 2, h, w).contiguous(), 0.01, 0.5)
    pos, sig, vis = _multi_flow_state(n + 1, h, w, dev)
    tracks, visible, sigma = _OPS.multi_flow_tracks(fwd.view(n, k, 2, h, w), occ.view(n, k, h, w), err.view(n, k, h, w),
                                                    src, dst, pos, sig, vis)
    return {"tracks": tracks, "visible": visible, "uncertainty": sigma}


def _ring_slot(frame, slots):
    """Slot of a frame in a ring of `slots`: frame 0 keeps slot 0, frames t >= 1 cycle through the others"""
    return 0 if frame == 0 else 1 + (frame - 1) % (slots - 1)


class MultiFlowTrackRunner(_SequenceRunner):
    """Multi-flow dense point tracks over a video (semantics: `multi_flow_tracks`): where each pixel of the first frame of a
    `run()` is in every later frame, whether it is visible, and how uncertain the estimate is.  Each new frame t is
    matched against its K = len(gaps) + anchor sources (`multi_flow_sources`: t-1, t-2, t-4, ... and frame 0), so a point
    hidden for a while comes back through a longer flow, and a track is a few links long however far the clip goes.

    A step takes `batch` new frames, uploaded and encoded once, and runs batch x K pairs (2 x batch x K flows with
    `pred_bidir_flow`), all inside one CUDA graph per staging slot:
    * the new frames' pyramids go into a device feature ring; the first frame's pyramid has slot 0, never overwritten;
    * the K source pyramids of every new frame are gathered from the ring with `index_select` on a small device table,
      staged with the frames, so one graph serves every step; absent sources of a clip's first frames are filled with a
      present pair and marked absent in the table;
    * `forward_encoded(..., pred_bidir_flow=True)` on the pairs, resized back to the frames' size as `infer_flow` does,
      then `um_fb_consistency_error` (masks and forward residuals) and one `um_multi_flow_tracks` launch over the step's
      frames, whose states live in a device ring.
    A short last step is filled with repeats of its last frame; they write no state and their results are dropped.
    Memory held for the life of the runner: the feature ring of max(gaps) + batch + 1 pyramids (encode_frames' [h,w,128]
    fp32 per scale: about 16 MB each for gmflow-scale2 at 480x832), and a state ring of as many slots, 13 bytes per pixel
    each; plus the activations of a forward over batch x K pairs.
    `run(frames)` resets the state and yields, per frame t >= 1 (frame 0 is not yielded), 'tracks' fp32 [H,W,2] (x, y),
    'visible' uint8 [H,W] and 'uncertainty' fp32 [H,W] (sigma^2): 13 bytes per pixel.  `return_flow=True` adds the frame's
    'flow' / 'flow_bwd' [K,2,H,W] and 'sources' [K] (frame indices, -1 absent).  `pred_bwd_flow`, `visualize`,
    `concat_frame` and `visualize_bwd` are refused."""

    task = "flow"

    def __init__(self, model, frame_size, batch, device, gaps=MULTI_FLOW_GAPS, anchor=True, padding_factor=32,
                 inference_size=None, use_graph=True, return_flow=False, **model_kwargs):
        name = type(self).__name__
        _track_flags(model_kwargs, name, "the tracks run forward from the first frame")
        self.kw = _task_kwargs(model_kwargs, "flow", name)
        self.gaps, self.anchor = _multi_flow_gaps(gaps, anchor, name)
        self.k = len(self.gaps) + self.anchor
        self._init_sequence(model, frame_size, batch, device, use_graph, padding_factor, inference_size)
        self.return_flow = bool(return_flow)
        self.slots = max(self.gaps, default=0) + self.batch + 1
        with torch.cuda.device(self.dev):
            probe = self._encode(torch.zeros((1, self.h, self.w, 3), dtype=torch.uint8, device=self.dev))
        self.ring = [torch.empty((self.slots,) + tuple(f.shape[1:]), device=self.dev, dtype=f.dtype) for f in probe]
        self.carry = [r[:1] for r in self.ring]            # _prime encodes the first frame into slot 0
        self.pos, self.sig, self.vis = _multi_flow_state(self.slots, self.h, self.w, self.dev)
        # per new frame: K feature slots to gather, K state slots (-1 absent), K source frames (-1 absent), the feature
        # slot it is written to and its state slot (-1: a repeat, no state)
        cols = 3 * self.k + 2
        self.tab_pin = [torch.empty((self.batch, cols), dtype=torch.int64).pin_memory() for _ in range(2)]
        self.tab_dev = [torch.empty((self.batch, cols), dtype=torch.int64, device=self.dev) for _ in range(2)]
        self._next = 1

    def _begin(self, first):
        self._next = 1

    def _prime(self, frame):
        super()._prime(frame)
        self.pos[0], _ = _track_start(self.h, self.w, self.dev)
        self.sig[0] = 0
        self.vis[0] = 1

    def _step(self, slot):
        b, k, h, w = self.batch, self.k, self.h, self.w
        tab = self.tab_dev[slot]
        new = self._encode(self.dev_in[slot])
        for r, f in zip(self.ring, new):
            r.index_copy_(0, tab[:, 3 * k], f)
        gather = tab[:, :k].reshape(-1)
        first = [r.index_select(0, gather) for r in self.ring]
        second = [f[:, None].expand((b, k) + tuple(f.shape[1:])).reshape((b * k,) + tuple(f.shape[1:])) for f in new]
        flow = self.model.forward_encoded(first, second, pred_bidir_flow=True, **self.kw)["flow_preds"][-1]
        out = _flow_outputs(flow, self.ori, self.size, self.transposed, True, False)
        fwd, bwd = out["flow"].contiguous(), out["flow_bwd"].contiguous()
        occ, _, err = _OPS.fb_consistency_error(fwd, bwd, 0.01, 0.5)
        src = tab[:, k:2 * k].to(torch.int32).contiguous()
        dst = tab[:, 3 * k + 1].to(torch.int32).contiguous()
        tracks, visible, sigma = _OPS.multi_flow_tracks(fwd.view(b, k, 2, h, w), occ.view(b, k, h, w),
                                                        err.view(b, k, h, w), src, dst, self.pos, self.sig, self.vis)
        res = {"tracks": tracks, "visible": visible, "uncertainty": sigma}
        if self.return_flow:
            res.update(flow=fwd.view(b, k, 2, h, w), flow_bwd=bwd.view(b, k, 2, h, w), sources=tab[:, 2 * k:3 * k])
        return res

    def _reset_inputs(self, slot):
        super()._reset_inputs(slot)
        k = self.k
        t = self.tab_dev[slot]
        t[:, :k] = 0
        t[:, k:3 * k] = -1
        t[:, 3 * k] = torch.arange(1, self.batch + 1, device=self.dev)
        t[:, 3 * k + 1] = -1

    def _stage_host(self, slot, chunk):
        items = super()._stage_host(slot, chunk)
        k, m, tab = self.k, len(chunk), self.tab_pin[slot]
        for i in range(self.batch):
            t = self._next + min(i, m - 1)
            src = multi_flow_sources(t, self.gaps, self.anchor)
            fill = next(s for s in src if s >= 0)
            row = [_ring_slot(s if s >= 0 else fill, self.slots) for s in src]
            row += [_ring_slot(s, self.slots) if s >= 0 else -1 for s in src] + src
            row += [_ring_slot(t, self.slots), _ring_slot(t, self.slots) if i < m else -1]
            tab[i] = torch.tensor(row, dtype=torch.int64)
        self.tab_dev[slot].copy_(tab, non_blocking=True)
        self._next += m
        return items


class _PosedDepth:
    """What the two depth runners share: per staging slot, the step's relative poses in a pinned and a device buffer of
    views * batch [4,4] matrices, the camera operands built on them once, eagerly, before any capture (they depend on
    the intrinsics only; `UniMatch.depth_cameras` takes a float32 pose of all the step's matrices as it is, so
    `cams[slot]["pose"]` IS `pose_dev[slot]` and an upload updates the cameras), and the depth matching path on them.
    The runner sets `model`, `batch`, `dev`, `kw`, `bidir`, `from_argmax` and `inv_range` first."""

    def _init_poses(self, intrinsics, num_depth_candidates):
        npose = (2 if self.bidir else 1) * self.batch
        self.pose_pin = [torch.empty((npose, 4, 4)).pin_memory() for _ in range(2)]
        self.pose_dev = [torch.eye(4, device=self.dev).repeat(npose, 1, 1) for _ in range(2)]
        Kb = intrinsics.to(self.dev)[None].repeat(self.batch, 1, 1)
        self.cams = [self.model.depth_cameras(Kb, self.pose_dev[s], self.model.upsample_factor, *self.inv_range,
                                              num_depth_candidates, self.bidir) for s in range(2)]

    def _reset_poses(self, slot):
        self.pose_dev[slot].copy_(torch.eye(4, device=self.dev).expand_as(self.pose_dev[slot]))

    def _stage_poses(self, slot, rel):
        """the step's relative poses, float32 [views * batch, 4, 4], into pinned memory, then their H2D copy"""
        self.pose_pin[slot].copy_(torch.from_numpy(rel))
        self.pose_dev[slot].copy_(self.pose_pin[slot], non_blocking=True)

    def _depth(self, slot, first, second):
        """the model's depths [views * batch, H, W] at the inference size, from the pairs' encoded features"""
        return self.model.forward_encoded(first, second, task="depth", cameras=self.cams[slot], min_depth=self.inv_range[0],
                                          max_depth=self.inv_range[1], depth_from_argmax=self.from_argmax,
                                          pred_bidir_depth=self.bidir, **self.kw)["flow_preds"][-1]


class DepthSequenceRunner(_PosedDepth, _SequenceRunner):
    """Streaming depth over a posed frame sequence: consecutive pairs of host (uint8 frame, absolute pose) items, every frame
    uploaded and encoded once -- the depth counterpart of `VideoFlowRunner`.

    * upload: each step copies `batch` NEW frames, uint8 [H,W,3] as decoded, and the `batch` relative poses of its pairs
      (followed by their inverses when `pred_bidir_depth`), computed on the host with the reference's numpy expression
      (0.59 MB per 384x512 frame, against 4.72 MB for the two float32 images of a pair);
    * device work of a step: `um_frames_to_planar_normalized` (uint8 -> ImageNet-normalised planes at the inference size), the
      encoder on the new frames, the depth matching path on the `batch` pairs and the depth resized back.  The camera operands
      that depend on the intrinsics only (`UniMatch.depth_cameras`) are built once, eagerly, before any capture; the per-step
      poses are static device buffers that the upload fills.  The last frame's pose stays on the host for the next step;
    * download: 'depth' (and 'depth_bwd') [H,W] per pair and, with `visualize`, the uint8 RGB pictures 'vis' [H,W,3]
      (+ 'vis_bwd') that the reference writes for them (`depth_to_image`, painted inside the step's graph);
      `return_depth=False` with `visualize` sends back only the pictures.

    Sizes and semantics are those of `infer_depth_sequence` (and `infer_depth`): `min_depth` / `max_depth` are metric,
    the intrinsics [3,3] are not rescaled with the frames.  `run(items)` takes an iterable of (uint8 frame [H,W,3], pose [4,4])
    host items and yields one dict of CPU tensors per consecutive pair (pinned staging reused -- copy what you keep)."""

    task = "depth"

    def __init__(self, model, frame_size, batch, device, intrinsics, padding_factor=16, inference_size=None, min_depth=0.5,
                 max_depth=10.0, num_depth_candidates=64, depth_from_argmax=False, pred_bidir_depth=False, use_graph=True,
                 visualize=False, return_depth=True, **model_kwargs):
        _check_returns(return_depth, visualize, "return_depth", "DepthSequenceRunner")
        self.kw = _task_kwargs(model_kwargs, "depth", "DepthSequenceRunner")
        self.visualize, self.return_depth = bool(visualize), bool(return_depth)
        K = _intrinsics33(intrinsics, "DepthSequenceRunner")
        self._init_sequence(model, frame_size, batch, device, use_graph, padding_factor, inference_size)
        self.bidir, self.from_argmax = bool(pred_bidir_depth), bool(depth_from_argmax)
        self.inv_range = (1.0 / max_depth, 1.0 / min_depth)                      # the model works on inverse depth
        self._init_poses(K, num_depth_candidates)
        self.prev_pose = None                              # last frame's absolute pose, float32 [4,4] on the host

    @staticmethod
    def _frame(item):
        return item[0]

    def _begin(self, first):
        self.prev_pose = _pose44(first[1], "DepthSequenceRunner")

    def _match(self, slot, first, second):
        out = _depth_outputs(self._depth(slot, first, second), self.ori, self.size, self.bidir)
        return _colour_outputs(out, "depth", depth_to_image, self.return_depth) if self.visualize else out

    def _reset_inputs(self, slot):
        super()._reset_inputs(slot)
        self._reset_poses(slot)

    def _stage_host(self, slot, chunk):
        """the frames, then the relative poses of the step's pairs, continuing from the carried pose"""
        poses = [self.prev_pose] + [_pose44(pose, "DepthSequenceRunner") for _, pose in super()._stage_host(slot, chunk)]
        self._stage_step_poses(slot, poses, len(chunk))
        self.prev_pose = poses[-1]

    def _stage_step_poses(self, slot, poses, n_real):
        """the step's batch + 1 absolute poses (the carried one first; `n_real` real pairs) -> its relative poses"""
        self._stage_poses(slot, _relative_poses(poses, self.bidir))


class DepthFusionRunner(DepthSequenceRunner):
    """`DepthSequenceRunner` that also fuses each pair's depth into a TSDF volume on the device (`fusion.TSDFVolume`), inside
    the step's CUDA graph: after the depth of a step, one `um_tsdf_integrate` launch over its pairs' first frames t, with
    the depth of frame t from pair (t, t+1), frame t's uint8 colours and its world-to-camera matrix.  The result is
    `fuse_depths(volume, depths, frames, intrinsics, poses)` on the runner's own depths, bit for bit.

    * frames t of a step are the carried previous frame and the new frames but the last: the runner keeps a device uint8
      copy of the last frame next to the carried pyramid;
    * the world-to-camera matrices (`_world_to_camera`, the host path of `fuse_depths`) and the number of real pairs are
      staged with the relative poses, so the padding pairs of a short last step and the warm-up runs before a graph
      capture (reset inputs: no pair) fuse nothing;
    * only 'depth' is fused, so the last frame of a `run()` is not; `pred_bidir_depth` is refused, because the backward
      depth of frame t+1 would count frame t+1 twice;
    * the volume persists across `run()` calls, so a long scene can be fed in pieces (each piece's last frame is not fused);
    * `return_depth=False` without `visualize` is allowed: the volume is the result, and `run()` then yields empty dicts
      and downloads nothing.
    The intrinsics are those of the frames' size, as for `DepthSequenceRunner`.

    With `track=True` the given poses are corrected before fusion (the network still takes the given relative poses).
    Each step takes its pairs' frames t in order, inside the step's graph: the predicted pose is C P_t, with P_t the given
    pose and C `pose_correction` (device fp64 [4,4], identity at first); frame t's depth is tracked against the volume
    from there (`TSDFVolume.track`'s ICP with its defaults) and fused at the tracked pose, or at the predicted one when it
    is not tracked; a tracked frame then sets C = T_t P_t^-1.  C persists across `run()` calls with the volume, as it
    relates the given poses' frame to the volume's: reset both to start a new scene.  Each result gains 'pose' (float32
    [4,4], the camera-to-world pose frame t was fused at) and 'tracked' (bool), which are all that is downloaded with
    `return_depth=False` and no pictures.

    With `consistency_views=k > 0` each frame t is checked against the previous k frames t before it is tracked and
    fused: `fusion.filter_depths` with `max_pixel=1.0`, `max_relative=0.01` and `min_views=consistency_min_views` on the
    network's depths, at the given poses (those the depths were computed with).  The check is causal, so streaming needs
    no delay: the runner keeps a device ring of the raw depths of the last k frames t (all zeros when empty, so an empty
    slot is never a consistent source) and the host keeps their given poses; each step stages the rows of the ring's
    frames and its own, and one `um_depth_consistency` launch on the (k + batch) stack filters its frames inside the
    step's graph.  The filtered depth is what is fused (and tracked), so the volume equals `fuse_depths(volume,
    filter_depths(D, K, poses, sequence_sources(n, k, 0), min_views=m)['depth'], frames, K, poses)` on the runner's own
    depths D.  The ring persists across `run()` calls with the volume (and `pose_correction`); `reset_scene()` empties
    all three.  'depth' stays the network's depth, and each result gains 'views' (uint8 [H,W], the number of consistent
    earlier frames), which is downloaded even with `return_depth=False`.  The first `consistency_min_views` frames of a
    scene have fewer earlier frames than the count requires, so they are not fused.  `consistency_views=0` is the runner
    without the check: no ring and no extra launch."""

    def __init__(self, model, frame_size, batch, device, intrinsics, volume, padding_factor=16, inference_size=None,
                 min_depth=0.5, max_depth=10.0, num_depth_candidates=64, depth_from_argmax=False, pred_bidir_depth=False,
                 use_graph=True, visualize=False, return_depth=True, track=False, consistency_views=0,
                 consistency_min_views=2, **model_kwargs):
        from .fusion import MAX_CONSISTENCY_SOURCES, TSDFVolume, _ICP
        k, m = consistency_views, consistency_min_views
        if isinstance(k, bool) or not isinstance(k, int) or not 0 <= k <= MAX_CONSISTENCY_SOURCES:
            raise ValueError("DepthFusionRunner: consistency_views must be an int in [0, 255]")
        if k and (isinstance(m, bool) or not isinstance(m, int) or not 1 <= m <= k):
            raise ValueError("DepthFusionRunner: consistency_min_views must be an int in [1, consistency_views]")
        if pred_bidir_depth:
            raise ValueError("DepthFusionRunner: pred_bidir_depth is refused: the backward depth of frame t+1 would fuse "
                             "frame t+1 twice")
        if not isinstance(volume, TSDFVolume):
            raise ValueError("DepthFusionRunner: volume must be a TSDFVolume")
        dev = torch.device(device)
        if dev.type != "cuda" or (dev.index if dev.index is not None else torch.cuda.current_device()) != volume.device.index:
            raise ValueError("DepthFusionRunner: the volume must be on the runner's device")
        super().__init__(model, frame_size, batch, device, intrinsics, padding_factor=padding_factor,
                         inference_size=inference_size, min_depth=min_depth, max_depth=max_depth,
                         num_depth_candidates=num_depth_candidates, depth_from_argmax=depth_from_argmax,
                         use_graph=use_graph, visualize=visualize, return_depth=True, **model_kwargs)
        self.return_depth = bool(return_depth)
        self.volume = volume
        self.K = _intrinsics33(intrinsics, "DepthFusionRunner")
        self.carry_frame = torch.zeros((1, self.h, self.w, 3), dtype=torch.uint8, device=self.dev)
        self.w2c_pin = [torch.empty((self.batch, 3, 4)).pin_memory() for _ in range(2)]
        self.w2c_dev = [torch.zeros((self.batch, 3, 4), device=self.dev) for _ in range(2)]
        self.nvalid_pin = [torch.zeros((1,), dtype=torch.int32).pin_memory() for _ in range(2)]
        self.nvalid_dev = [torch.zeros((1,), dtype=torch.int32, device=self.dev) for _ in range(2)]
        self.track = bool(track)
        if self.track:
            self._icp = _ICP(volume, self.K, 1, self.h, self.w, 3, (4, 5, 10), 0.1, 20.0, 0.3, "DepthFusionRunner")
            self.pose_correction = torch.eye(4, dtype=torch.float64, device=self.dev)
            self.given_pin = [torch.empty((self.batch, 4, 4), dtype=torch.float64).pin_memory() for _ in range(2)]
            self.given_dev = [torch.zeros((self.batch, 4, 4), dtype=torch.float64, device=self.dev) for _ in range(2)]
            self.real_pin = [torch.zeros((self.batch,), dtype=torch.int32).pin_memory() for _ in range(2)]
            self.real_dev = [torch.zeros((self.batch,), dtype=torch.int32, device=self.dev) for _ in range(2)]
        self.consistency_views, self.consistency_min_views = k, m
        if k:
            b = self.batch
            self.ring = torch.zeros((k, self.h, self.w), device=self.dev)
            self.ring_poses = []                           # the given poses of the ring's frames, oldest first
            # stack rows: the ring's k frames, oldest first, then the step's frames t; step row i is checked against
            # stack rows k + i - 1, ..., i (the k frames before it)
            self.cons_refs = torch.arange(k, k + b, dtype=torch.int32, device=self.dev)
            self.cons_sources = (torch.arange(b)[:, None] + k - torch.arange(1, k + 1)[None, :]).to(torch.int32).to(self.dev)
            self.rows_pin = [torch.empty((2, k + b, 3, 4)).pin_memory() for _ in range(2)]       # c2w, then w2c
            self.rows_dev = [torch.eye(4, device=self.dev)[:3].repeat(2, k + b, 1, 1) for _ in range(2)]
            self.ring_idx_pin = [torch.empty((k,), dtype=torch.int64).pin_memory() for _ in range(2)]
            self.ring_idx_dev = [torch.arange(k, device=self.dev) for _ in range(2)]    # the stack rows the ring keeps

    def reset_scene(self):
        """Start a new scene: empty the volume, the consistency ring and `pose_correction`"""
        self.volume.reset()
        if self.track:
            self.pose_correction.copy_(torch.eye(4, dtype=torch.float64, device=self.dev))
        if self.consistency_views:
            self.ring.zero_()
            self.ring_poses = []

    def _match(self, slot, first, second):
        out = _depth_outputs(self._depth(slot, first, second), self.ori, self.size, False)
        frames = torch.cat((self.carry_frame, self.dev_in[slot][:-1]), dim=0)        # frame t of every pair
        depth, extra = out["depth"].contiguous(), {}
        if self.consistency_views:
            depth, extra["views"] = self._filter(slot, depth)
        poses = self._track_and_fuse(slot, depth, frames) if self.track else {}
        if not self.track:
            self.volume._integrate(depth, frames, self.w2c_dev[slot], self.nvalid_dev[slot], self.K)
        self.carry_frame.copy_(self.dev_in[slot][-1:])
        extra.update(poses)
        if self.visualize:
            return dict(_colour_outputs(out, "depth", depth_to_image, self.return_depth), **extra)
        return dict(out, **extra) if self.return_depth else extra

    def _filter(self, slot, depth):
        """One um_depth_consistency launch on the ring and the step's depths, then the ring keeps the last k real rows of
        that stack; returns the filtered depths [batch,H,W] and the counts"""
        stack = torch.cat((self.ring, depth), dim=0)
        rows = self.rows_dev[slot]
        K = self.K
        views, filtered = _OPS.depth_consistency(stack, rows[0], rows[1], self.cons_refs, self.cons_sources,
                                                 float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]), 1.0,
                                                 0.01, self.consistency_min_views)
        self.ring.copy_(stack.index_select(0, self.ring_idx_dev[slot]))
        return filtered, views

    def _track_and_fuse(self, slot, depth, frames):
        """Frames t in order: track against the volume from C P_t, fuse at the result, update C; padding pairs (real
        flag 0) are untouched.  Returns the step's 'pose' [batch,4,4] and 'tracked' [batch]."""
        b = self.batch
        pose = torch.empty((b, 4, 4), dtype=torch.float32, device=self.dev)
        tracked = torch.empty((b,), dtype=torch.uint8, device=self.dev)
        inliers = torch.empty((b,), dtype=torch.int64, device=self.dev)
        rmse = torch.empty((b,), dtype=torch.float32, device=self.dev)
        pyramid, normals = self._icp.prepare(depth)
        for t in range(b):
            real = self.real_dev[slot][t:t + 1]
            self._icp.track([p[t:t + 1] for p in pyramid], [n[t:t + 1] for n in normals], self.given_dev[slot][t:t + 1],
                            real, (pose[t:t + 1], tracked[t:t + 1], inliers[t:t + 1], rmse[t:t + 1]),
                            correction=self.pose_correction)
            self.volume._integrate(depth[t:t + 1], frames[t:t + 1], self._icp.w2c_out, real, self.K)
        return {"pose": pose, "tracked": tracked.view(torch.bool)}

    def _prime(self, frame):
        super()._prime(frame)
        self.carry_frame.copy_(frame)

    def _reset_inputs(self, slot):
        super()._reset_inputs(slot)
        self.nvalid_dev[slot].zero_()
        if self.track:
            self.real_dev[slot].zero_()
        if self.consistency_views:                       # no real pair: the ring keeps its rows
            self.ring_idx_dev[slot].copy_(torch.arange(self.consistency_views, device=self.dev))

    def _stage_step_poses(self, slot, poses, n_real):
        """the relative poses, then the world-to-camera rows of the pairs' frames t and the number of real pairs (with
        `track`, also the frames' given poses in fp64 and a 0 / 1 flag per pair)"""
        super()._stage_step_poses(slot, poses, n_real)
        self.w2c_pin[slot].copy_(torch.from_numpy(_world_to_camera(poses[:-1])))
        self.nvalid_pin[slot][0] = n_real
        self.w2c_dev[slot].copy_(self.w2c_pin[slot], non_blocking=True)
        self.nvalid_dev[slot].copy_(self.nvalid_pin[slot], non_blocking=True)
        if self.track:
            self.given_pin[slot].copy_(torch.from_numpy(np.stack(poses[:-1]).astype(np.float64)))
            self.real_pin[slot].copy_(torch.arange(self.batch) < n_real)
            self.given_dev[slot].copy_(self.given_pin[slot], non_blocking=True)
            self.real_dev[slot].copy_(self.real_pin[slot], non_blocking=True)
        k = self.consistency_views
        if k:
            eye = np.eye(4, dtype=np.float32)
            stack = [eye] * (k - len(self.ring_poses)) + self.ring_poses + list(poses[:-1])
            self.rows_pin[slot][0].copy_(torch.from_numpy(_camera_to_world(stack)))
            self.rows_pin[slot][1].copy_(torch.from_numpy(_world_to_camera(stack)))
            self.ring_idx_pin[slot].copy_(torch.arange(n_real, n_real + k))
            self.rows_dev[slot].copy_(self.rows_pin[slot], non_blocking=True)
            self.ring_idx_dev[slot].copy_(self.ring_idx_pin[slot], non_blocking=True)
            self.ring_poses = (self.ring_poses + list(poses[:n_real]))[-k:]


def _depth_step_layout(sizes, batch, pred_bidir_depth):
    """Descriptor tables of one depth step of `batch` pairs, whose real pairs have the frame sizes `sizes` = [((h, w) of
    frame t, (h, w) of frame t+1)] (1 <= len <= batch).  Returns (frames, outputs, frame_bytes, used, results):
    * frames: 2*batch items over the packed uint8 frames -- the real pairs' frames t back to back, then their frames t+1,
      each at its own size; the items of a short step's filler pairs point at its last pair's frames;
    * outputs: batch items ('depth'), or 2*batch with `pred_bidir_depth` ('depth', then 'depth_bwd'), packed back to back,
      each at the size of its pair's frame t with scale 1 (depth is not rescaled with the resize); fillers are empty items,
      which the kernels skip;
    * frame_bytes / used: the used prefixes of the packed frames and depths;
    * results: per real pair, the (key, offset, h, w) of each of its outputs."""
    frames, nbytes = _frame_table(tuple(zip(*sizes)), batch)
    keys = ("depth", "depth_bwd") if pred_bidir_depth else ("depth",)
    outputs, used, results = _scalar_outputs(keys, [t for t, _ in sizes], batch)
    return frames, outputs, nbytes, used, results


class MixedSizeDepthRunner(_PosedDepth, _MixedSizeRunner):
    """Streaming depth over posed pairs of ANY size up to `max_frame_size`: `inference_depth` (evaluate_depth.py:338-417),
    which takes each pair at its own size, as a stream.  Each item is one pair (uint8 frame t [h, w, 3], uint8 frame t+1
    [h', w', 3], relative pose [4, 4]); the relative pose is the reference's host float32 `inv(pose[t+1]) @ pose[t]`, as
    `_relative_poses` computes it, and with `pred_bidir_depth` its inverse is appended on the host.

    * buckets: a pair's bucket is the size the model sees, frame t's size rounded up to a multiple of `padding_factor`, or
      `inference_size` (depth has no portrait rule); steps are formed as in `MixedSizeStereoRunner` (`_batches`, at most
      `max_buckets` open);
    * upload: the step's frames t, then its frames t+1, packed back to back as uint8 (the used bytes only), the descriptor
      table and the step's relative poses, on a side stream while the previous step computes;
    * device work of a step, one CUDA graph per bucket and staging slot: `um_frames_to_planar_normalized_ragged` (every frame
      normalised and resized from its own size to the bucket's, so frame t+1 follows frame t's inference size), the encoder
      and the depth matching path, `um_resize_bilinear_ragged` back to frame t's size with scale 1, and with `visualize`
      `um_depth_to_image_ragged`.  The intrinsics [3, 3] are not rescaled with the frames, as in the reference; the camera
      operands are built once per staging slot before any capture, on static pose buffers the upload fills, and shared by
      every bucket (they do not depend on the size);
    * download: only the used prefixes of the packed depths and pictures.

    Every pair encodes both of its frames: frame t+1 is seen at frame t's inference size and again at its own, so the
    encode-once path of `DepthSequenceRunner` does not hold in general.  A directory of one frame size is better served
    by that runner.  `run(items)` yields (index, result) as steps complete -- completion order, not input order; `index`
    is the pair's position in the input, each exactly once.  `result` holds CPU views 'depth' [h, w] (+ 'depth_bwd') at
    frame t's size and, with `visualize`, the uint8 RGB pictures 'vis' [h, w, 3] (+ 'vis_bwd') of `depth_to_image`;
    `return_depth=False` with `visualize` sends back only the pictures.  The views point into reused pinned staging -- copy
    what you keep.  `stats` counts steps, pairs, captures and the bytes copied each way."""

    value_key = "depth"

    def __init__(self, model, max_frame_size, batch, device, intrinsics, padding_factor=16, inference_size=None,
                 min_depth=0.5, max_depth=10.0, num_depth_candidates=64, depth_from_argmax=False, pred_bidir_depth=False,
                 visualize=False, return_depth=True, use_graph=True, max_buckets=4, **model_kwargs):
        name = type(self).__name__
        _check_returns(return_depth, visualize, "return_depth", name)
        self.kw = _task_kwargs(model_kwargs, "depth", name)
        K = _intrinsics33(intrinsics, name)
        self.padding_factor, self.inference_size = padding_factor, inference_size
        self.bidir, self.from_argmax = bool(pred_bidir_depth), bool(depth_from_argmax)
        self.visualize, self.return_depth = bool(visualize), bool(return_depth)
        self.inv_range = (1.0 / max_depth, 1.0 / min_depth)                      # the model works on inverse depth
        views = 2 if self.bidir else 1
        self._init_mixed(model, max_frame_size, batch, device, use_graph, max_buckets, (2 + views) * int(batch), views)
        self._init_poses(K, num_depth_candidates)

    # ---- host side
    def _pair(self, pair):
        name = type(self).__name__
        if len(pair) != 3:
            raise ValueError("%s: an item is (frame t, frame t+1, relative pose)" % name)
        return self._frame(pair[0]), self._frame(pair[1]), _pose44(pair[2], name)

    @staticmethod
    def _sizes(pairs):
        return [(tuple(p[0].shape[:2]), tuple(p[1].shape[:2])) for p in pairs]

    def _step_layout(self, sizes, size):
        return _depth_step_layout(sizes, self.batch, self.bidir)

    def _poses(self, pairs):
        """the step's relative poses, a short step's last one repeated, then with `pred_bidir_depth` their inverses
        (as `_relative_poses` forms them): float32 [views * batch, 4, 4]"""
        return _with_inverses([pairs[min(i, len(pairs) - 1)][2] for i in range(self.batch)], self.bidir)

    def _stage_host(self, slot, chunk):
        """the packed frames and the table (`_MixedSizeRunner`), then the step's relative poses"""
        super()._stage_host(slot, chunk)
        self._stage_poses(slot, self._poses([p for _, p in chunk]))
        self.stats["h2d_bytes"] += self.pose_pin[slot].nbytes

    # ---- device side
    def _reset_inputs(self, slot):
        """zero frames, a full-capacity table and identity poses: valid for any bucket"""
        cap = (self.hmax, self.wmax)
        table, _, _ = self._table([(cap, cap)] * self.batch, cap)
        self.dev_in[slot].zero_()
        self.dev_desc[slot].copy_(torch.from_numpy(table))
        self._reset_poses(slot)

    def _step(self, slot, size):
        b = self.batch
        items = self.dev_desc[slot]
        x = _OPS.frames_to_planar_normalized_ragged(self.dev_in[slot], items[:2 * b], self.hmax, self.wmax, int(size[0]),
                                                    int(size[1]), list(IMAGENET_MEAN), list(IMAGENET_STD))
        feats = self.model.encode_frames(x, task="depth")
        depth = self._depth(slot, [f[:b] for f in feats], [f[b:] for f in feats])                 # [views * b, H, W]
        return self._resize_back(depth.unsqueeze(1), items[2 * b:], _OPS.depth_to_image_ragged)


# ------------------------------------------------------------------------------------------------------ stereo scene flow
@torch.no_grad()
def warp_disparity(disp_next, flow):
    """The second disparity of scene flow from device tensors a caller holds, one `um_warp_disparity` launch.

    `disp_next`: [B,H,W], the disparity of left frame t+1; `flow`: planar [B,2,H,W], the optical flow from left frame t to
    left frame t+1, in pixels at the same size.  Returns {'disp_1': [B,H,W] fp32, 'in_frame': [B,H,W] uint8}: disp_1 at pixel
    p of frame t is the bilinear sample of disp_next at q = p + flow(p) clamped into the frame (grid_sample with
    padding_mode='border', align_corners=True), so a point that leaves the frame takes the nearest in-frame value and the
    map stays dense; in_frame is 1 where q lies inside [0, W-1] x [0, H-1].  fp32, with the order of operations of
    include/unimatch_sm100.h.  No occlusion handling."""
    if not torch.is_tensor(disp_next) or disp_next.dim() != 3:
        raise ValueError("warp_disparity expects disparities [B,H,W]")
    b, h, w = disp_next.shape
    if not torch.is_tensor(flow) or tuple(flow.shape) != (b, 2, h, w):
        raise ValueError("warp_disparity: flow must be planar [B,2,H,W] like the disparities")
    disp1, in_frame = _OPS.warp_disparity(disp_next.float().contiguous(), flow.float().contiguous())
    return {"disp_1": disp1, "in_frame": in_frame}


def _stereo_quadruples(frames, name):
    """(B, H, W) of the four device uint8 [B,H,W,3] views left0, right0, left1, right1, refused unless they agree"""
    shape = None
    for k, f in zip(("left0", "right0", "left1", "right1"), frames):
        if not torch.is_tensor(f) or f.dtype != torch.uint8 or f.dim() != 4 or f.shape[-1] != 3 or f.shape[0] < 1:
            raise ValueError("%s: %s must be uint8 frames [B,H,W,3] as decoded" % (name, k))
        if shape is None:
            shape = tuple(f.shape)
        elif tuple(f.shape) != shape:
            raise ValueError("%s: the four views must have one shape, %s is %s against %s" % (name, k, list(f.shape), list(shape)))
    return shape[:3]


def _flow_kwargs(flow_kwargs, name):
    kw = _task_kwargs(flow_kwargs or {}, "flow", name)
    for k in ("pred_bidir_flow", "fwd_bwd_consistency_check"):
        if kw.pop(k, False):
            raise ValueError("%s: %s is not supported (scene flow takes the forward flow only)" % (name, k))
    return kw


def _stereo_kwargs(stereo_kwargs, name):
    kw = _task_kwargs(stereo_kwargs or {}, "stereo", name)
    for k in ("pred_bidir_disp", "pred_right_disp"):
        if kw.pop(k, False):
            raise ValueError("%s: %s is not supported (scene flow takes the left disparity only)" % (name, k))
    return kw


@torch.no_grad()
def infer_scene_flow(stereo_model, flow_model, left0, right0, left1, right1, *, stereo_kwargs=None, flow_kwargs=None,
                     stereo_padding_factor=16, flow_padding_factor=32, stereo_inference_size=None, flow_inference_size=None):
    """Stereo scene flow of B stereo quadruples: the disparity at time t, the disparity of the same pixels at t+1, and the
    optical flow between the two left frames (what KITTI 2015's scene-flow benchmark scores).

    `left0`, `right0` (time t) and `left1`, `right1` (time t+1) are device uint8 frames [B,H,W,3] as decoded.  Geometry is
    that of `_stereo_from_frames` / `infer_stereo` for stereo and `infer_flow` for flow: each network resizes to a multiple of
    its padding factor (or to its inference size), and its output is resized back and rescaled.  One stereo forward over the
    2B pairs (left0, left1 then right0, right1), normalised on the device (`um_frames_to_planar_normalized`); one flow forward
    on (left0, left1) (`um_frames_to_planar`); one `um_warp_disparity`.  `stereo_kwargs` / `flow_kwargs` go to the models
    (attn_type, attn_splits_list, corr_radius_list, prop_radius_list, num_reg_refine).
    Returns {'disp_0': [B,H,W], 'disp_1': [B,H,W], 'flow': [B,2,H,W], 'in_frame': [B,H,W] uint8} at the frames' size;
    disp_1 and in_frame are `warp_disparity` of the disparity at t+1 and the flow."""
    b, h, w = _stereo_quadruples((left0, right0, left1, right1), "infer_scene_flow")
    skw, fkw = _stereo_kwargs(stereo_kwargs, "infer_scene_flow"), _flow_kwargs(flow_kwargs, "infer_scene_flow")
    disp = _stereo_from_frames(stereo_model, torch.cat((left0, left1, right0, right1)), padding_factor=stereo_padding_factor,
                               inference_size=stereo_inference_size, **skw)["disp"]
    transposed, ori, size = _frame_geometry(h, w, flow_padding_factor, flow_inference_size, "flow")
    planes = _frames_to_model(torch.cat((left0, left1)), "flow", transposed, size)
    flow = flow_model(planes[:b], planes[b:], **fkw)["flow_preds"][-1]
    flow = _flow_outputs(flow, ori, size, transposed, False, False)["flow"].contiguous()
    out = {"disp_0": disp[:b].contiguous(), "flow": flow}
    out["disp_1"], out["in_frame"] = _OPS.warp_disparity(disp[b:].contiguous(), flow)
    return {k: out[k] for k in ("disp_0", "disp_1", "flow", "in_frame")}


class SceneFlowRunner(_SequenceRunner):
    """Streaming stereo scene flow over a stereo video: consecutive pairs of host (left, right) uint8 frames, each frame's
    stereo computed once and each left frame encoded once for the flow.

    * upload: each step copies `batch` NEW stereo frames in one pinned uint8 [2B,H,W,3] buffer (the B left frames, then the
      B right ones, as `StereoRunner` packs them);
    * device work of a step, captured once per staging slot in a CUDA graph: the stereo network on the B new pairs
      (`_stereo_from_frames`), the flow encoder on the B new left frames and the flow matching path on the B pairs (previous
      step's last frame, new frames) with the last pyramid carried, as `VideoFlowRunner` does, and `um_warp_disparity` of each
      new frame's disparity through its pair's flow.  The last frame's disparity is carried to the next step as its first
      pair's disp_0;
    * download per consecutive pair (t, t+1): 'disp_0' [H,W] (frame t), 'disp_1' [H,W] (frame t+1's disparity in frame t's
      grid), 'flow' [2,H,W] and 'in_frame' [H,W] uint8, 17 bytes per pixel; with `visualize` also 'vis_disp_0' / 'vis_disp_1'
      (`disparity_to_image`, BGR) and 'vis_flow' (`flow_to_image`, RGB), painted inside the step's graph.

    Sizes, semantics and keywords are those of `infer_scene_flow` (`stereo_padding_factor` / `stereo_inference_size` for
    the stereo network, `flow_padding_factor` / `flow_inference_size` for the flow network); the outputs equal `infer_scene_flow` on the
    consecutive quadruples up to the encoder's fp32 summation order.  One frame size per runner; a short last step is filled
    with repeats of its last item and the extra results are dropped.  `run(items)` takes an iterable of (left, right) host
    uint8 frames [H,W,3] and yields one dict of CPU tensors per consecutive pair (pinned staging reused -- copy what you
    keep)."""

    task = "flow"

    def __init__(self, stereo_model, flow_model, frame_size, batch, device, *, stereo_kwargs=None, flow_kwargs=None,
                 stereo_padding_factor=16, flow_padding_factor=32, stereo_inference_size=None, flow_inference_size=None,
                 visualize=False, use_graph=True):
        self.kw = _flow_kwargs(flow_kwargs, "SceneFlowRunner")
        self.stereo_kw = _stereo_kwargs(stereo_kwargs, "SceneFlowRunner")
        self.stereo_model = stereo_model
        self.stereo_geometry = dict(padding_factor=stereo_padding_factor, inference_size=stereo_inference_size)
        self.visualize = bool(visualize)
        self._init_sequence(flow_model, frame_size, batch, device, use_graph, flow_padding_factor, flow_inference_size)
        shape = (2 * self.batch, self.h, self.w, 3)
        self.stereo_pin = [torch.empty(shape, dtype=torch.uint8).pin_memory() for _ in range(2)]
        self.stereo_dev = [torch.empty(shape, dtype=torch.uint8, device=self.dev) for _ in range(2)]
        self.pin = [p[:self.batch] for p in self.stereo_pin]          # the left frames, which the flow encoder reads
        self.dev_in = [d[:self.batch] for d in self.stereo_dev]
        self.carry_disp = torch.zeros((1, self.h, self.w), device=self.dev)
        self.first_right = None

    def _graph_models(self):
        return (self.model, self.stereo_model)

    def _item(self, item):
        """(left, right) host uint8 frames [H,W,3] of one stereo frame"""
        if not isinstance(item, (tuple, list)) or len(item) != 2:
            raise ValueError("SceneFlowRunner: items are (left, right) stereo frames")
        views = [torch.as_tensor(v) for v in item]
        for v in views:
            if v.dtype != torch.uint8 or tuple(v.shape) != (self.h, self.w, 3):
                raise ValueError("SceneFlowRunner: frames must be uint8 [%d, %d, 3]" % (self.h, self.w))
        return views

    def _frame(self, item):
        return self._item(item)[0]

    def _begin(self, first):
        self.first_right = self._item(first)[1]

    def _disparity(self, frames_u8):
        return _stereo_from_frames(self.stereo_model, frames_u8, **self.stereo_geometry, **self.stereo_kw)["disp"]

    def _match(self, slot, first, second):
        disp = self._disparity(self.stereo_dev[slot])
        flow = self.model.forward_encoded(first, second, **self.kw)["flow_preds"][-1]
        flow = _flow_outputs(flow, self.ori, self.size, self.transposed, False, False)["flow"].contiguous()
        out = {"disp_0": torch.cat((self.carry_disp, disp[:-1])), "flow": flow}
        out["disp_1"], out["in_frame"] = _OPS.warp_disparity(disp.contiguous(), flow)
        self.carry_disp.copy_(disp[-1:])
        if self.visualize:
            out["vis_disp_0"], out["vis_disp_1"] = disparity_to_image(out["disp_0"]), disparity_to_image(out["disp_1"])
            out["vis_flow"] = flow_to_image(flow)
        return out

    def _reset_inputs(self, slot):
        self.stereo_dev[slot].zero_()

    def _prime(self, frame):
        """the first frame's pyramid and disparity (eagerly), carried into the first step"""
        super()._prime(frame)
        right = self.first_right.to(self.dev)[None]
        self.carry_disp.copy_(self._disparity(torch.cat((frame, right))))

    def _stage_host(self, slot, chunk):
        """the step's left frames, then its right frames, into the pinned buffer; then their one H2D copy"""
        for i in range(self.batch):
            left, right = self._item(chunk[min(i, len(chunk) - 1)])
            self.stereo_pin[slot][i].copy_(left)
            self.stereo_pin[slot][self.batch + i].copy_(right)
        self.stereo_dev[slot].copy_(self.stereo_pin[slot], non_blocking=True)
