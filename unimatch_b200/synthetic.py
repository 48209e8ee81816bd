"""Deterministic synthetic weights and image pairs (there is no network for checkpoints/datasets).

Weights: every tensor of `spec.param_spec` is drawn from a CPU `torch.Generator` in table order,
with the magnitudes the reference's initialisers produce (kaiming-normal fan_out for convs,
`backbone.py:88-90`; xavier-uniform for the transformer / propagation matrices,
`transformer.py:222-224`, `attention.py:180-182`; torch defaults for biases), so logits have the same
statistics as a random-init reference model (SURVEY.md §7.2 #1).  The same state_dict is loaded into
the reference (golden generation), the oracle and the CUDA module.

Inputs follow SURVEY.md §8d: a box-blurred noise texture and a translated copy, so a true match exists.
"""
import math

import torch
import torch.nn.functional as F

from .spec import WORKLOADS, param_spec

IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)


# The weight set bench.py and the full-size parity tests load.  Random-init statistics make the network numerically chaotic at
# 480x832 (the reference's OWN output moves by 0.78 px mean / 34 px max when its inputs are scaled by 1 + 1e-7, almost all of it
# in the convex-upsampling softmax of the random mask head; tools/self_noise.py), which would make "EPE vs reference"
# unmeasurable.  These gains keep every layer's shape, arithmetic and cost and bring the reference's self-noise down to
# 2e-5 px mean / 1.3e-4 px max (measured, same tool): smaller encoder output and LayerNorm gains -> matching logits of a
# trained-network size; small flow-head / mask-head gains -> sub-pixel residual updates and a soft 9-tap upsampling mask.
BENCH_WEIGHTS = dict(damp=0.5, refine_gain=0.02, backbone_gain=0.25, norm_gain=0.25, mask_gain=0.05)


def synthetic_state_dict(seed=326, damp=1.0, refine_gain=0.02, backbone_gain=1.0, norm_gain=1.0, mask_gain=1.0,
                         **model_kwargs):
    """Flat state_dict for `UniMatch(**model_kwargs)`.

    `damp` scales the transformer matrices (damp=0.5 is the 'damped' set of SURVEY.md §8d that tames
    the chaotic random-init logits).  `refine_gain` scales the last conv of the refinement flow head
    (`refine.flow_head.conv2`): with kaiming-init weights the RAFT-style update block is an EXPANDING map
    (measured: the reference's own 1-thread vs 8-thread outputs drift apart x2-x7 per refinement
    iteration, 27 px mean EPE after six), whereas a trained block is contractive with sub-pixel residuals;
    0.02 gives residuals of a few tenths of a pixel per iteration so end-to-end parity is measurable."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for key, shape in param_spec(**model_kwargs).items():
        if len(shape) == 4:
            cout, cin, kh, kw = shape
            t = torch.randn(shape, generator=g) * math.sqrt(2.0 / (cout * kh * kw))
        elif len(shape) == 2:
            a = math.sqrt(6.0 / (shape[0] + shape[1]))
            t = (torch.rand(shape, generator=g) * 2 - 1) * a
            if key.startswith("transformer."):
                t = t * damp
        elif ".norm" in key:
            t = torch.randn(shape, generator=g) * 0.1 + (1.0 if key.endswith("weight") else 0.0)
        else:  # conv / linear bias: U(-1/sqrt(fan_in), 1/sqrt(fan_in)) with a nominal fan_in
            t = (torch.rand(shape, generator=g) * 2 - 1) * 0.05
        if key.startswith("refine.flow_head.conv2."):
            t = t * refine_gain
        if key.startswith(("backbone.conv2.", "backbone.trident_conv.")):
            t = t * backbone_gain       # output scale of the encoder (InstanceNorm makes every earlier layer scale-free)
        if key.startswith("transformer.") and ".norm" in key:
            t = t * norm_gain           # size of the messages added to the residual stream -> size of the matching logits
        if key.startswith(("refine.mask.2.", "upsampler.2.")):
            t = t * mask_gain           # logits of the convex-upsampling softmax (9 taps)
        sd[key] = t.float().contiguous()
    return sd


def synthetic_model(workload, device="cuda"):
    """`UniMatch` of `WORKLOADS[workload]` in eval mode with the BENCH_WEIGHTS state_dict (seed 326) loaded strictly, on
    `device`: the model bench.py, the workload tests and the tools run."""
    from .unimatch import UniMatch          # here, so that importing this module does not load the CUDA library
    cfg = WORKLOADS[workload]["model"]
    m = UniMatch(**cfg).eval()
    m.load_state_dict(synthetic_state_dict(seed=326, **BENCH_WEIGHTS, **cfg), strict=True)
    return m.to(device)


def workload_call(workload, drop=()):
    """A copy of the forward keywords of `WORKLOADS[workload]` without the keys named in `drop`."""
    return {k: v for k, v in WORKLOADS[workload]["call"].items() if k not in drop}


def _texture(g, h, w):
    x = torch.rand((1, 3, h, w), generator=g) * 255.0
    k = torch.ones((3, 1, 5, 5)) / 25.0
    return F.conv2d(F.pad(x, (2, 2, 2, 2), mode="replicate"), k, groups=3)


def synthetic_pair(task, h, w, index=0, seed=1234):
    """One image pair [1,3,H,W] x2 (+ intrinsics/pose for depth), generator seed = seed + index."""
    g = torch.Generator().manual_seed(seed + index)
    m = 40
    canvas = _texture(g, h + 2 * m, w + 2 * m)
    if task == "flow":
        dx = int(torch.randint(-8, 9, (1,), generator=g))
        dy = int(torch.randint(-8, 9, (1,), generator=g))
        img0 = canvas[:, :, m:m + h, m:m + w]
        img1 = canvas[:, :, m + dy:m + dy + h, m + dx:m + dx + w]
        return dict(img0=img0.contiguous(), img1=img1.contiguous())
    mean = torch.tensor(IMAGENET_MEAN).view(1, 3, 1, 1)
    std = torch.tensor(IMAGENET_STD).view(1, 3, 1, 1)
    d = int(torch.randint(0, 33, (1,), generator=g))
    left = canvas[:, :, m:m + h, m:m + w]
    right = canvas[:, :, m:m + h, m - d:m - d + w]       # right view = left shifted by +d px
    left = ((left / 255.0 - mean) / std).contiguous()
    right = ((right / 255.0 - mean) / std).contiguous()
    if task == "stereo":
        return dict(img0=left, img1=right)
    K = torch.tensor([[0.9 * w, 0.0, w / 2.0], [0.0, 0.9 * w, h / 2.0], [0.0, 0.0, 1.0]]).view(1, 3, 3)
    pose = torch.eye(4).view(1, 4, 4).clone()
    pose[0, 0, 3] = 0.1
    return dict(img0=left, img1=right, intrinsics=K, pose=pose)


def synthetic_batch(task, batch, h, w, first_index=0, seed=1234):
    items = [synthetic_pair(task, h, w, first_index + i, seed) for i in range(batch)]
    return {k: torch.cat([it[k] for it in items], dim=0) for k in items[0]}


def synthetic_video(T, h, w, seed=1234, step=3):
    """T frames uint8 [T,H,W,3] (channel-last, as a decoder returns them) cropped from one box-blurred noise canvas along a
    seeded path that moves up to `step` px per frame and axis, so consecutive frames have a true match."""
    g = torch.Generator().manual_seed(seed)
    m = step * max(T - 1, 0) + 1
    canvas = _texture(g, h + 2 * m, w + 2 * m)[0].round().clamp(0, 255).to(torch.uint8).permute(1, 2, 0)
    moves = torch.randint(-step, step + 1, (max(T - 1, 0), 2), generator=g)
    y = x = m
    frames = [canvas[y:y + h, x:x + w]]
    for dy, dx in moves.tolist():
        y, x = y + dy, x + dx
        frames.append(canvas[y:y + h, x:x + w])
    return torch.stack(frames, 0).contiguous()


def synthetic_stereo_frames(n, h, w, seed=1234):
    """n rectified stereo pairs as decoded: left and right uint8 frames [n,H,W,3] (channel-last), pair i cropped from band i
    of one box-blurred noise canvas, the right view being the left shifted by a seeded whole-pixel disparity in [0, 32] --
    the uint8 counterpart of `synthetic_pair("stereo")`."""
    g = torch.Generator().manual_seed(seed)
    m = 32
    canvas = _texture(g, n * h, w + m)[0].round().clamp(0, 255).to(torch.uint8).permute(1, 2, 0)
    disps = torch.randint(0, m + 1, (n,), generator=g).tolist()
    lefts = [canvas[i * h:(i + 1) * h, m:m + w] for i in range(n)]
    rights = [canvas[i * h:(i + 1) * h, m - d:m - d + w] for i, d in enumerate(disps)]      # right view = left shifted by +d px
    return torch.stack(lefts, 0).contiguous(), torch.stack(rights, 0).contiguous()


def synthetic_stereo_video(T, h, w, seed=1234, step=3):
    """A rectified stereo clip as decoded: left and right uint8 frames [T,H,W,3] (channel-last).  The left view is
    `synthetic_video`'s moving crops of one box-blurred noise canvas; the right view is each left crop shifted by a seeded
    whole-pixel disparity in [0, 32] of the whole clip (a fronto-parallel scene: disparity d everywhere, in every frame)."""
    g = torch.Generator().manual_seed(seed)
    m, d_max = step * max(T - 1, 0) + 1, 32
    canvas = _texture(g, h + 2 * m, w + 2 * m + d_max)[0].round().clamp(0, 255).to(torch.uint8).permute(1, 2, 0)
    moves = torch.randint(-step, step + 1, (max(T - 1, 0), 2), generator=g)
    d = int(torch.randint(0, d_max + 1, (1,), generator=g))
    y, x = m, m + d_max
    lefts, rights = [], []
    for dy, dx in [(0, 0)] + moves.tolist():
        y, x = y + dy, x + dx
        lefts.append(canvas[y:y + h, x:x + w])
        rights.append(canvas[y:y + h, x - d:x - d + w])         # right view = left shifted by +d px
    return torch.stack(lefts, 0).contiguous(), torch.stack(rights, 0).contiguous()


def synthetic_posed_sequence(T, h, w, seed=1234, step=3, plane_depth=2.0):
    """A posed frame sequence for depth inference: T frames uint8 [T,H,W,3] of a fronto-parallel textured plane at depth
    `plane_depth`, the intrinsics K [3,3] (focal 0.9 W, centred principal point) and the absolute camera-to-world poses
    [T,4,4] (float32, as the reference loads pose files).  The camera moves along x only, by seeded whole-pixel amounts of up
    to `step` px per frame: the frames are crops of one box-blurred noise canvas at matching integer x-shifts, so every
    consecutive pair has a true match with depth `plane_depth` everywhere."""
    g = torch.Generator().manual_seed(seed)
    m = step * max(T - 1, 0) + 1
    canvas = _texture(g, h, w + 2 * m)[0].round().clamp(0, 255).to(torch.uint8).permute(1, 2, 0)
    shifts = torch.randint(-step, step + 1, (max(T - 1, 0),), generator=g).tolist()
    focal = 0.9 * w
    K = torch.tensor([[focal, 0.0, w / 2.0], [0.0, focal, h / 2.0], [0.0, 0.0, 1.0]])
    frames, poses, x = [], [], 0
    for t in range(T):
        if t > 0:
            x += shifts[t - 1]
        frames.append(canvas[:, m + x:m + x + w])          # camera moved right by x px -> the crop moves right by x px
        pose = torch.eye(4, dtype=torch.float64)
        pose[0, 3] = x * plane_depth / focal
        poses.append(pose)
    return torch.stack(frames, 0).contiguous(), K, torch.stack(poses, 0).float()


def noise_batch(task, batch, h, w, seed=99):
    """Cheap pure-noise batch for throughput runs (no match structure; same arithmetic)."""
    g = torch.Generator().manual_seed(seed)
    out = dict(img0=torch.rand((batch, 3, h, w), generator=g) * 255.0,
               img1=torch.rand((batch, 3, h, w), generator=g) * 255.0)
    if task != "flow":
        mean = torch.tensor(IMAGENET_MEAN).view(1, 3, 1, 1)
        std = torch.tensor(IMAGENET_STD).view(1, 3, 1, 1)
        out = {k: (v / 255.0 - mean) / std for k, v in out.items()}
    if task == "depth":
        K = torch.tensor([[0.9 * w, 0.0, w / 2.0], [0.0, 0.9 * w, h / 2.0], [0.0, 0.0, 1.0]])
        pose = torch.eye(4)
        pose[0, 3] = 0.1
        out["intrinsics"] = K.view(1, 3, 3).repeat(batch, 1, 1)
        out["pose"] = pose.view(1, 4, 4).repeat(batch, 1, 1)
    return out
