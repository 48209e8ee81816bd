#!/usr/bin/env python
"""Video inference against pairwise inference on the same consecutive pairs, on one GPU.

    python tools/video_bench.py [--workload config4|config2|config5] [--steps K] [--warmup W] [--pairs-per-step B]
                                [--visualize]

Flow workloads (config4, config2): the timed video step is what `unimatch_b200.VideoFlowRunner` does per step: B new synthetic
uint8 frames are copied from pinned memory, converted on the device (`um_frames_to_planar`), encoded, paired with the previous
step's last frame (its feature pyramid is carried, not re-encoded) and run as B pairs; the flow goes back to pinned memory.
The pairwise step is `UniMatch.forward` on the same B pairs, uploaded as two float32 images per pair and downloaded the same way.
Depth workload (config5): the timed sequence step is what `unimatch_b200.DepthSequenceRunner` does per step: B new uint8 frames
of a synthetic posed sequence and their B relative poses are copied from pinned memory, normalised and converted on the device
(`um_frames_to_planar_normalized`), encoded and run as B pairs with the carried frame; the pairwise step is `UniMatch.forward`
on the same B pairs as ImageNet-normalised float32 images, with their intrinsics and relative poses.
The two steps alternate in one process, eager on both sides, and the workloads, sizes and weights are those of bench.py.
With --visualize (config5 only) a third step alternates with the two: the same sequence step with `visualize=True,
return_depth=False`, which paints the pictures the reference's depth driver writes (`depth_to_image`) and downloads them
instead of the depths; the line then also holds `depth_to_image` alone on the step's depths (CUDA events, bytes moved), its
agreement with oracle/depth_viz.py, and that oracle's host time per picture as a numpy stand-in for matplotlib.
Prints ONE JSON line: pairs/s of each path, the encoder ("backbone") section time of each, H2D / D2H bytes per step, and how
far the two outputs are apart (they are not bit-identical: see `UniMatch.encode_frames`).  Exits non-zero beyond 1e-4 of the
largest output value.  Writes nothing to the tree.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import BENCH_WORKLOADS  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="config4", choices=["config4", "config2", "config5"])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--pairs-per-step", type=int, default=0, help="B (default: the workload's pairs per GPU in bench.py)")
    ap.add_argument("--visualize", action="store_true", help="config5: also time the step that downloads depth pictures")
    args = ap.parse_args()
    if args.visualize and args.workload != "config5":
        ap.error("--visualize applies to the depth workload (config5)")
    run(args)


def run(args):
    """One runner step (B new synthetic uint8 frames uploaded from pinned memory, the previous step's last frame carried, B
    pairs, output back to pinned memory) against `UniMatch.forward` on the same B pairs as float32 images (uploaded and
    downloaded the same way), alternating step by step in one process, eager on both sides."""
    from unimatch_b200 import ops
    from unimatch_b200.spec import WORKLOADS
    from unimatch_b200.synthetic import synthetic_model
    wl_name, H, W, ppg, cfg_idx, _, _ = BENCH_WORKLOADS[args.workload]
    cfg = WORKLOADS[wl_name]
    B = args.pairs_per_step or ppg
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    model = synthetic_model(wl_name, dev)
    setup = _flow_steps if cfg["model"]["task"] == "flow" else _depth_steps
    video_step, pair_step, out_v, out_p, io, notes = setup(model, cfg, H, W, B, dev)
    vis_step, out_vis = _depth_picture_step(model, cfg, H, W, B, dev) if args.visualize else (None, None)
    steps = [video_step, pair_step] + ([vis_step] if vis_step else [])

    for _ in range(max(args.warmup, 2)):
        for fn in steps:
            fn()
    torch.cuda.synchronize()
    identical = bool(torch.equal(out_v, out_p))
    rel_diff = (out_v - out_p).abs().max().item() / max(1.0, out_p.abs().max().item())

    def timed(fns, steps, timer=None):
        model.kernel_timer = timer
        ev = [[torch.cuda.Event(enable_timing=True) for _ in range(2)] for _ in fns]
        tot = [0.0] * len(fns)
        for _ in range(steps):
            for j, fn in enumerate(fns):
                ev[j][0].record(); fn(); ev[j][1].record()
            torch.cuda.synchronize()
            for j in range(len(fns)):
                tot[j] += ev[j][0].elapsed_time(ev[j][1])
        model.kernel_timer = None
        return [t / steps for t in tot]

    ms = timed(steps, args.steps)
    ms_v, ms_p = ms[:2]
    sections = {}
    for name, fn in (("video", video_step), ("pairwise", pair_step)):
        timer = {}
        timed([fn], args.steps, timer)
        acc = {}
        for tag, a, b, _ in timer.pop("_events", []):
            if tag.startswith("sec:"):
                acc[tag[4:]] = acc.get(tag[4:], 0.0) + a.elapsed_time(b)
        sections[name] = {k: round(v / args.steps, 3) for k, v in acc.items()}
    props = torch.cuda.get_device_properties(dev)
    res = {"metric": "pairs/s of consecutive %s pairs @%dx%d %s, %s path vs pairwise forward" % (notes["kind"], H, W, wl_name,
                                                                                                  notes["kind"]),
           "device": props.name, "workload": "%s %dx%d, %d pairs per step (BASELINE configs[%d])" % (wl_name, H, W, B, cfg_idx),
           "steps": args.steps, "warmup": max(args.warmup, 2), "data": notes["data"], "cuda_graph": False,
           "video": {"pairs_per_s": B / (ms_v / 1e3), "ms_per_step": round(ms_v, 3),
                     "sections_ms_per_step": {"backbone": sections["video"].get("backbone")},
                     "h2d_bytes_per_step": io[0], "d2h_bytes_per_step": int(out_v.numel() * 4),
                     "note": "B new frames encoded, the carried frame's pyramid reused (restored to frame 0's by a device copy "
                             "inside the step so that every step runs the same pairs)"},
           "pairwise": {"pairs_per_s": B / (ms_p / 1e3), "ms_per_step": round(ms_p, 3),
                        "sections_ms_per_step": {"backbone": sections["pairwise"].get("backbone")},
                        "h2d_bytes_per_step": io[1], "d2h_bytes_per_step": int(out_p.numel() * 4)},
           "speedup": ms_p / ms_v, "outputs_bit_identical": identical, "max_abs_diff_rel_to_max_" + notes["value"]: rel_diff,
           "identity_note": "um_conv2d_tc sums a tile's K chunks in an order rotated by the CTA owning the tile; encoding B frames "
                            "instead of 2B changes the tile-to-CTA map, hence the last bits (tolerance 1e-4 of the largest %s)"
                            % notes["value"],
           "launches_per_process": ops.launch_count()}
    if vis_step:
        res["pictures"] = _picture_report(ms[2], out_v, out_vis, B, dev)
    print(json.dumps(res))
    if rel_diff > 1e-4:
        sys.exit(1)


def _video_step(runner, frames, out, key, pin_pose=None):
    """(runner step on frames 1..B paired with frame 0, H2D bytes per step): B new uint8 frames (and, for depth, their
    relative poses) copied from pinned memory, the step's `key` output copied back to `out`."""
    runner.carry = [f.clone() for f in runner._encode(frames[:1].to(runner.dev))]
    saved = [c.clone() for c in runner.carry]                                # frame 0's pyramid
    pin_new = frames[1:].contiguous().pin_memory()

    def step():
        for c, f in zip(runner.carry, saved):                                # same pairs every step: (0,1), (1,2), ...
            c.copy_(f)
        runner.dev_in[0].copy_(pin_new, non_blocking=True)
        if pin_pose is not None:
            runner.pose_dev[0].copy_(pin_pose, non_blocking=True)
        out.copy_(runner._step(0)[key], non_blocking=True)
    return step, int(pin_new.numel() + (0 if pin_pose is None else pin_pose.numel() * 4))


def _flow_steps(model, cfg, H, W, B, dev):
    """VideoFlowRunner step and pairwise forward on the same B pairs of a synthetic video"""
    from unimatch_b200.inference import VideoFlowRunner
    from unimatch_b200.synthetic import synthetic_video
    call = {k: v for k, v in cfg["call"].items() if k != "task"}
    frames = synthetic_video(B + 1, H, W, seed=77)                          # frame 0 = carried, frames 1..B = new
    runner = VideoFlowRunner(model, (H, W), B, dev, padding_factor=cfg["pad"], use_graph=False, **call)
    planar = frames.permute(0, 3, 1, 2).float()
    pin0, pin1 = planar[:-1].contiguous().pin_memory(), planar[1:].contiguous().pin_memory()
    out_v, out_p = torch.empty((B, 2, H, W)).pin_memory(), torch.empty((B, 2, H, W)).pin_memory()
    video_step, io_v = _video_step(runner, frames, out_v, "flow")

    def pair_step():
        a, b = pin0.to(dev, non_blocking=True), pin1.to(dev, non_blocking=True)
        out_p.copy_(model(a, b, **cfg["call"])["flow_preds"][-1], non_blocking=True)

    io = (io_v, int((pin0.numel() + pin1.numel()) * 4))
    return video_step, pair_step, out_v, out_p, io, dict(kind="video", data="synthetic_video seed 77", value="flow")


def _depth_runner(model, cfg, H, W, B, dev, **extra):
    """(DepthSequenceRunner, frames, K, pinned relative poses) of a synthetic posed sequence of B + 1 frames.  bench.py's
    call gives the model's inverse-depth range; the runner takes the metric one."""
    from unimatch_b200.inference import DepthSequenceRunner, _relative_poses
    from unimatch_b200.synthetic import synthetic_posed_sequence
    call = cfg["call"]
    kw = {k: v for k, v in call.items() if k not in ("task", "min_depth", "max_depth", "num_depth_candidates")}
    frames, K, poses = synthetic_posed_sequence(B + 1, H, W, seed=77)     # frame 0 = carried, frames 1..B = new
    runner = DepthSequenceRunner(model, (H, W), B, dev, K, padding_factor=cfg["pad"], use_graph=False,
                                 min_depth=1.0 / call["max_depth"], max_depth=1.0 / call["min_depth"],
                                 num_depth_candidates=call["num_depth_candidates"], **kw, **extra)
    rel = torch.from_numpy(_relative_poses([p for p in poses.numpy()], False))
    return runner, frames, K, rel.contiguous().pin_memory()


def _depth_steps(model, cfg, H, W, B, dev):
    """DepthSequenceRunner step and pairwise forward on the same B pairs of a synthetic posed sequence."""
    from unimatch_b200.synthetic import IMAGENET_MEAN, IMAGENET_STD
    call = cfg["call"]
    runner, frames, K, pin_pose = _depth_runner(model, cfg, H, W, B, dev)
    mean, std = torch.tensor(IMAGENET_MEAN).view(1, 3, 1, 1), torch.tensor(IMAGENET_STD).view(1, 3, 1, 1)
    planar = (frames.permute(0, 3, 1, 2).float() / 255. - mean) / std
    pin0, pin1 = planar[:-1].contiguous().pin_memory(), planar[1:].contiguous().pin_memory()
    pin_k = K[None].repeat(B, 1, 1).contiguous().pin_memory()
    out_v, out_p = torch.empty((B, H, W)).pin_memory(), torch.empty((B, H, W)).pin_memory()
    video_step, io_v = _video_step(runner, frames, out_v, "depth", pin_pose)

    def pair_step():
        a, b = pin0.to(dev, non_blocking=True), pin1.to(dev, non_blocking=True)
        k, p = pin_k.to(dev, non_blocking=True), pin_pose.to(dev, non_blocking=True)
        out_p.copy_(model(a, b, intrinsics=k, pose=p, **call)["flow_preds"][-1], non_blocking=True)

    io = (io_v, int((pin0.numel() + pin1.numel() + pin_k.numel() + pin_pose.numel()) * 4))
    return video_step, pair_step, out_v, out_p, io, dict(kind="depth-sequence", data="synthetic_posed_sequence seed 77",
                                                        value="depth")


def _depth_picture_step(model, cfg, H, W, B, dev):
    """the sequence step of `_depth_steps` with visualize=True, return_depth=False: the pictures come back instead of the
    depths"""
    runner, frames, _, pin_pose = _depth_runner(model, cfg, H, W, B, dev, visualize=True, return_depth=False)
    out = torch.empty((B, H, W, 3), dtype=torch.uint8).pin_memory()
    return _video_step(runner, frames, out, "vis", pin_pose)[0], out


def _picture_report(ms_step, depth, pictures, B, dev):
    """The picture step's rate and D2H bytes, `depth_to_image` alone on the step's depths (CUDA events over 50 calls; bytes:
    the depths read by the four radix-select passes and the colouring pass, the pictures written once), whether it equals
    the oracle, and the oracle's host time per picture."""
    import time

    import numpy as np

    from oracle import depth_viz
    from unimatch_b200.inference import depth_to_image
    dd = depth.to(dev)
    out = depth_to_image(dd)
    for _ in range(3):
        depth_to_image(dd, out)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(50):
        depth_to_image(dd, out)
    e1.record()
    torch.cuda.synchronize()
    kernel_ms = e0.elapsed_time(e1) / 50
    nbytes = dd.numel() * (5 * 4 + 3)
    host = depth.numpy()
    t0 = time.perf_counter()
    ref = depth_viz.viz_inverse_depth_batch(host)
    host_ms = (time.perf_counter() - t0) * 1e3 / B
    return {"ms_per_step": round(ms_step, 3), "pairs_per_s": B / (ms_step / 1e3),
            "d2h_bytes_per_step": int(pictures.numel()),
            "note": "the sequence step with visualize=True, return_depth=False: depth_to_image inside the step, uint8 RGB "
                    "pictures downloaded instead of fp32 depths",
            "depth_to_image": {"ms": round(kernel_ms, 4), "bytes": int(nbytes), "GB_per_s": round(nbytes / kernel_ms / 1e6, 1),
                               "pictures": B, "equals_oracle": bool(np.array_equal(out.cpu().numpy(), ref))},
            "host_oracle_ms_per_picture": round(host_ms, 2),
            "host_note": "oracle/depth_viz.py on one CPU thread, a numpy stand-in for matplotlib's viz_depth_tensor (exact "
                         "percentile by a full sort, float64 plasma lookup)"}


if __name__ == "__main__":
    main()
