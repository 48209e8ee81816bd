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
colouring of utils/flow_viz.py on the device.  Decoding frames and writing videos (mp4) stay out of scope; the leaderboard
files (.flo, PNG, PFM) are written by `submission.py`.

Posed sequences (`inference_depth`, evaluate_depth.py:297-419): `infer_depth_sequence` runs the consecutive pairs of a frame
sequence with absolute camera poses, every frame encoded once and the relative poses computed on the host as the reference
does; `DepthSequenceRunner` streams host (uint8 frame, pose) items through the same path, replayed as a CUDA graph;
`depth_to_image` is the reference's `viz_depth_tensor(1. / depth)` (inverse depth scaled by its exact 95th percentile,
matplotlib's `plasma` map, evaluate_depth.py:403-417) on the device.  Writing files (PNG) stays out of scope.

Stereo (`inference_stereo`, evaluate_stereo.py:711-843): `StereoRunner` streams host uint8 (left, right) pairs, normalised and
resized on the device, through the same path as `infer_stereo`, replayed as a CUDA graph; `disparity_to_image` is the
reference's `vis_disparity` (min-max scaling, cv2's INFERNO map) on the device.  Writing files (PNG, PFM) stays out of scope.
"""
import math

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
    _check_flow_args(pred_bidir_flow, fwd_bwd_consistency_check, model_kwargs, "infer_flow")
    transposed = image1.size(-2) > image1.size(-1)
    if transposed:
        image1, image2 = image1.transpose(-2, -1), image2.transpose(-2, -1)
    ori = tuple(image1.shape[-2:])
    size = _inference_size(ori, padding_factor, inference_size)
    if size != ori:
        image1, image2 = _resize(image1, size), _resize(image2, size)
    flow = model(image1.contiguous(), image2.contiguous(), pred_bidir_flow=pred_bidir_flow, **model_kwargs)["flow_preds"][-1]
    return _flow_outputs(flow, ori, size, transposed, pred_bidir_flow, fwd_bwd_consistency_check)


def _check_flow_args(pred_bidir_flow, fwd_bwd_consistency_check, model_kwargs, name):
    if fwd_bwd_consistency_check and not pred_bidir_flow:
        raise ValueError("fwd_bwd_consistency_check needs pred_bidir_flow=True (evaluate_flow.py:774-792)")
    if model_kwargs.setdefault("task", "flow") != "flow":
        raise ValueError("%s drives the flow task only" % name)


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
    _check_flow_args(pred_bidir_flow, fwd_bwd_consistency_check, model_kwargs, "infer_flow_video")
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
    if pred_bidir_disp and pred_right_disp:
        raise ValueError("choose one of pred_bidir_disp / pred_right_disp")
    ori = tuple(left.shape[-2:])
    size = _inference_size(ori, padding_factor, inference_size)
    if size != ori:
        left, right = _resize(left, size), _resize(right, size)
    return _stereo_outputs(model, left, right, ori, size, pred_bidir_disp, pred_right_disp, model_kwargs)


def _stereo_outputs(model, left, right, ori, size, pred_bidir_disp, pred_right_disp, model_kwargs):
    """Normalised pairs at the inference size -> the stereo driver's outputs at the original size: the hflip batching, the
    forward, and the resize back with the width rescale and the flip back (evaluate_stereo.py:789-836)."""
    resized = size != ori
    b = left.shape[0]
    if pred_bidir_disp:
        left, right = torch.cat((left, _hflip(right)), dim=0), torch.cat((right, _hflip(left)), dim=0)
    elif pred_right_disp:
        left, right = _hflip(right), _hflip(left)
    model_kwargs["task"] = "stereo"
    disp = model(left.float().contiguous(), right.float().contiguous(), **model_kwargs)["flow_preds"][-1]     # [B or 2B, H, W]
    disp = disp.unsqueeze(1)
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
    if not torch.is_tensor(disp) or disp.dim() not in (2, 3) or not disp.dtype.is_floating_point or 0 in disp.shape:
        raise ValueError("disparity_to_image expects float disparities [N,H,W] or [H,W]")
    shape = tuple(disp.shape) + (3,)
    if out is None:
        out = torch.empty(shape, device=disp.device, dtype=torch.uint8)
    elif not torch.is_tensor(out) or tuple(out.shape) != shape or out.dtype != torch.uint8:
        raise ValueError("disparity_to_image: out must be uint8 %s" % (list(shape),))
    if disp.dim() == 2:
        _OPS.disparity_to_image(disp[None].float().contiguous(), out[None])
    else:
        _OPS.disparity_to_image(disp.float().contiguous(), out)
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
    if not torch.is_tensor(depth) or depth.dim() not in (2, 3) or not depth.dtype.is_floating_point or 0 in depth.shape:
        raise ValueError("depth_to_image expects float depths [N,H,W] or [H,W]")
    shape = tuple(depth.shape) + (3,)
    if out is None:
        out = torch.empty(shape, device=depth.device, dtype=torch.uint8)
    elif not torch.is_tensor(out) or tuple(out.shape) != shape or out.dtype != torch.uint8:
        raise ValueError("depth_to_image: out must be uint8 %s" % (list(shape),))
    if depth.dim() == 2:
        _OPS.depth_to_image(depth[None].float().contiguous(), out[None])
    else:
        _OPS.depth_to_image(depth.float().contiguous(), out)
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
def _depth_task_kwargs(model_kwargs, name):
    if model_kwargs.pop("task", "depth") != "depth":
        raise ValueError("%s drives the depth task only" % name)
    return model_kwargs


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
    rel = [np.linalg.inv(poses[t + 1]) @ poses[t] for t in range(len(poses) - 1)]
    if bidir:
        rel += [np.linalg.inv(r) for r in rel]
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
    model_kwargs = _depth_task_kwargs(model_kwargs, "infer_depth_sequence")
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
    copies of a step's outputs into pinned buffers) and `_results(slot, n)` (one dict of host tensors per item) apply."""

    def _init_pipeline(self, device, use_graph):
        self.dev = torch.device(device)
        self.copy_stream = torch.cuda.Stream(device=self.dev)
        self.graphs = [None, None]
        self.static_out = [None, None]
        self.use_graph = use_graph
        self.out_pin = [None, None]
        self._held_buffers = []

    def _download(self, slot, out):
        if self.out_pin[slot] is None:
            self.out_pin[slot] = {k: torch.empty(v.shape, dtype=v.dtype).pin_memory() for k, v in out.items()}
        for k, v in out.items():
            self.out_pin[slot][k].copy_(v, non_blocking=True)

    def _results(self, slot, n):
        for i in range(n):
            yield {k: v[i] for k, v in self.out_pin[slot].items()}

    def _capture(self):
        with torch.cuda.device(self.dev):
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(2):            # eager warm-up: builds the module's cached operand planes outside the capture
                    for slot in range(2):
                        self._reset_inputs(slot)
                        self._step(slot)
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            for slot in range(2):
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    self.static_out[slot] = self._step(slot)
                self.graphs[slot] = g
            # the graphs hold the raw addresses of the module's cached planes; calls at other shapes may evict them from
            # the module's caches, so the runner keeps them alive for as long as it may replay
            self._held_buffers = self.model.cached_buffers()
            torch.cuda.synchronize()

    def _stage(self, slot, chunk):
        """host side of one batch, then the H2D copies on the side stream; returns their completion event"""
        with torch.cuda.stream(self.copy_stream):
            self._stage_host(slot, chunk)
            ev = torch.cuda.Event()
            ev.record(self.copy_stream)
        return ev

    def _pipeline(self, items, start=None):
        """Yields the results of `items` taken `self.batch` at a time.  `start()` runs (eagerly, on the main stream) before
        the first step, after the graphs exist."""
        if self.use_graph and self.graphs[0] is None:
            self._capture()
        it = iter(items)

        def next_chunk():
            chunk = []
            for p in it:
                chunk.append(p)
                if len(chunk) == self.batch:
                    break
            return chunk

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
            if self.use_graph:
                self.graphs[slot].replay()
                out = self.static_out[slot]
            else:
                out = self._step(slot)
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

    @torch.no_grad()
    def run(self, pairs):
        with torch.cuda.device(self.dev):
            yield from self._pipeline(pairs)


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
        if pred_bidir_disp and pred_right_disp:
            raise ValueError("choose one of pred_bidir_disp / pred_right_disp")
        if not return_disp and not visualize:
            raise ValueError("nothing to return: return_disp=False needs visualize=True")
        self.kw = dict(model_kwargs)
        if self.kw.pop("task", "stereo") != "stereo":
            raise ValueError("StereoRunner drives the stereo task only")
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
        if self.visualize:
            for k in [k for k in ("disp", "disp_right") if k in out]:
                out[k.replace("disp", "vis")] = disparity_to_image(out[k])
                if not self.return_disp:
                    del out[k]
        return out

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

    @torch.no_grad()
    def run(self, pairs):
        with torch.cuda.device(self.dev):
            yield from self._pipeline(pairs)


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

    Sizes, transpose and rescale semantics are those of `infer_flow_video` (and `infer_flow`); the flows equal
    `infer_flow_video` on the whole sequence up to fp32 summation order.  `run(frames)` takes an iterable of host uint8 frames
    [H,W,3] (numpy arrays or tensors) and yields one dict of CPU tensors per consecutive pair (pinned staging reused -- copy
    what you keep)."""

    task = "flow"

    def __init__(self, model, frame_size, batch, device, padding_factor=32, inference_size=None, use_graph=True,
                 visualize=False, concat_frame=False, pred_bidir_flow=False, fwd_bwd_consistency_check=False,
                 return_flow=True, **model_kwargs):
        self.kw = dict(model_kwargs)
        _check_flow_args(pred_bidir_flow, fwd_bwd_consistency_check, self.kw, "VideoFlowRunner")
        if concat_frame and not visualize:
            raise ValueError("concat_frame needs visualize=True")
        if not return_flow and not visualize:
            raise ValueError("nothing to return: return_flow=False needs visualize=True")
        self._init_sequence(model, frame_size, batch, device, use_graph, padding_factor, inference_size)
        self.bidir, self.check = bool(pred_bidir_flow), bool(fwd_bwd_consistency_check)
        self.visualize, self.concat, self.return_flow = bool(visualize), bool(concat_frame), bool(return_flow)
        self.concat_axis = 0 if self.h < self.w else 1                                  # evaluate_flow.py:822
        self.carry_frame = torch.zeros((1, self.h, self.w, 3), dtype=torch.uint8, device=self.dev)

    def _match(self, slot, first, second):
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
            if not self.return_flow:
                del out["flow"]
        self.carry_frame.copy_(self.dev_in[slot][-1:])
        return out

    def _prime(self, frame):
        super()._prime(frame)
        self.carry_frame.copy_(frame)


class DepthSequenceRunner(_SequenceRunner):
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
        if not return_depth and not visualize:
            raise ValueError("nothing to return: return_depth=False needs visualize=True")
        self.kw = _depth_task_kwargs(dict(model_kwargs), "DepthSequenceRunner")
        self.visualize, self.return_depth = bool(visualize), bool(return_depth)
        K = _intrinsics33(intrinsics, "DepthSequenceRunner")
        self._init_sequence(model, frame_size, batch, device, use_graph, padding_factor, inference_size)
        self.bidir, self.from_argmax = bool(pred_bidir_depth), bool(depth_from_argmax)
        self.inv_range = (1.0 / max_depth, 1.0 / min_depth)                      # the model works on inverse depth
        npose = (2 if self.bidir else 1) * self.batch
        self.pose_pin = [torch.empty((npose, 4, 4)).pin_memory() for _ in range(2)]
        self.pose_dev = [torch.eye(4, device=self.dev).repeat(npose, 1, 1) for _ in range(2)]
        Kb = K.to(self.dev)[None].repeat(self.batch, 1, 1)
        # cams[slot]["pose"] IS pose_dev[slot] (a float32 pose of 2B matrices is taken as it is), so the upload updates it
        self.cams = [model.depth_cameras(Kb, self.pose_dev[s], model.upsample_factor, *self.inv_range, num_depth_candidates,
                                         self.bidir) for s in range(2)]
        self.prev_pose = None                              # last frame's absolute pose, float32 [4,4] on the host

    @staticmethod
    def _frame(item):
        return item[0]

    def _begin(self, first):
        self.prev_pose = _pose44(first[1], "DepthSequenceRunner")

    def _match(self, slot, first, second):
        depth = self.model.forward_encoded(first, second, task="depth", cameras=self.cams[slot], min_depth=self.inv_range[0],
                                           max_depth=self.inv_range[1], depth_from_argmax=self.from_argmax,
                                           pred_bidir_depth=self.bidir, **self.kw)["flow_preds"][-1]
        out = _depth_outputs(depth, self.ori, self.size, self.bidir)
        if self.visualize:
            for k in [k for k in ("depth", "depth_bwd") if k in out]:
                out[k.replace("depth", "vis")] = depth_to_image(out[k])
                if not self.return_depth:
                    del out[k]
        return out

    def _reset_inputs(self, slot):
        super()._reset_inputs(slot)
        self.pose_dev[slot].copy_(torch.eye(4, device=self.dev).expand_as(self.pose_dev[slot]))

    def _stage_host(self, slot, chunk):
        """the frames, then the relative poses of the step's pairs, continuing from the carried pose"""
        poses = [self.prev_pose] + [_pose44(pose, "DepthSequenceRunner") for _, pose in super()._stage_host(slot, chunk)]
        self.pose_pin[slot].copy_(torch.from_numpy(_relative_poses(poses, self.bidir)))
        self.prev_pose = poses[-1]
        self.pose_dev[slot].copy_(self.pose_pin[slot], non_blocking=True)
