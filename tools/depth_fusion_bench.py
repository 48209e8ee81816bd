#!/usr/bin/env python
"""TSDF fusion of a posed depth sequence, three ways, on one GPU.

    python tools/depth_fusion_bench.py [--batch 8] [--frames 65] [--height 480] [--width 640] [--voxel 0.01] [--repeats 3]

Synthetic gmdepth-scale1-regrefine1 (its workload's keywords) on a seeded `synthetic_posed_sequence` clip at ScanNet's
480x640, 65 frames (64 pairs), into the volume `TSDFVolume.covering` builds over the clip's frusta up to `--max-depth` at
1 cm voxels.  Arms, each from host uint8 frames and poses to a fused volume on the device:
  (a) `DepthFusionRunner`: the depths fused inside each step's CUDA graph, nothing downloaded;
  (b) `DepthSequenceRunner` returning the depths, then `fuse_depths` on the re-uploaded depths and frames;
  (c) what a user writes today: `DepthSequenceRunner` returning the depths, then a plain torch-ops TSDF integration on the
      GPU, frame by frame over every voxel (same projection, nearest pixel, truncation and running mean).
After one warm-up pass of every arm the arms alternate for `--repeats` rounds (the volume reset before each); each arm's
frames/s is the median round (a fused frame per pair).  Also reported: CUDA-event times of `um_tsdf_integrate` at the
step's shape (batch depth maps into the volume) over `--kernel-iters` launches, with the bytes it must move computed from
shapes -- the inputs, plus the voxel state (20 bytes read and 20 written) both for every voxel (dense bound) and for the
voxels the step actually updates -- and the share of the H100 SXM data-sheet 3.35 TB/s; the extraction's time and point
count; each arm's peak device memory in its warm-up pass; the largest TSDF difference of (b) and (c) from (a); the card's
name, power limit and SM clocks, read in the same run.  The synthetic weights' depths are not meaningful: this measures
speed, not reconstruction quality.  Prints ONE JSON line.  Writes nothing to the tree.
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.common import card, timed  # noqa: E402

HBM_DATASHEET_GBS = 3350.0
MODEL = "gmdepth-scale1-regrefine1"
_DEPTH_RANGE = ("min_depth", "max_depth", "num_depth_candidates")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--frames", type=int, default=65)
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--width", type=int, default=640)
    ap.add_argument("--voxel", type=float, default=0.01)
    ap.add_argument("--max-depth", type=float, default=2.5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--kernel-iters", type=int, default=50)
    run(ap.parse_args())


def _event_ms(fn, iters):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def torch_integrate(vol, depths, frames, poses, K):
    """The TSDF update in plain torch ops, one frame at a time over every voxel (what a user writes without the kernel)"""
    Z, Y, X = vol.tsdf.shape
    dev = vol.tsdf.device
    axes = [torch.arange(n, device=dev, dtype=torch.float32).add_(0.5).mul_(vol.voxel_size).add_(o)
            for n, o in zip((X, Y, Z), vol.origin)]
    pz, py, px = torch.meshgrid(axes[2], axes[1], axes[0], indexing="ij")
    p = torch.stack((px.reshape(-1), py.reshape(-1), pz.reshape(-1)), 0)                   # [3, N]
    F, Wt, C = vol.tsdf.view(-1), vol.weight.view(-1), vol.color.view(3, -1)
    h, w = depths.shape[1:]
    fx, fy, cx, cy = float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])
    for t in range(depths.shape[0]):
        M = torch.linalg.inv(torch.as_tensor(poses[t], dtype=torch.float32)).to(dev)
        c = M[:3, :3] @ p + M[:3, 3:]
        z = c[2]
        u = torch.floor(fx * c[0] / z + cx + 0.5)
        v = torch.floor(fy * c[1] / z + cy + 0.5)
        ok = (z > 0) & (u >= 0) & (u < w) & (v >= 0) & (v < h)
        pix = (v.clamp(0, h - 1) * w + u.clamp(0, w - 1)).long()
        d = depths[t].reshape(-1)[pix]
        sdf = d - z
        ok &= torch.isfinite(d) & (d > 0) & (sdf >= -vol.trunc)
        f = torch.clamp(sdf / vol.trunc, max=1.0)
        w1 = Wt + 1
        F.copy_(torch.where(ok, (F * Wt + f) / w1, F))
        rgb = frames[t].reshape(-1, 3)[pix].T.float()
        C.copy_(torch.where(ok, (C * Wt + rgb) / w1, C))
        Wt.copy_(torch.where(ok, w1, Wt))


@torch.no_grad()
def run(args):
    from unimatch_b200.fusion import TSDFVolume, fuse_depths
    from unimatch_b200.inference import DepthFusionRunner, DepthSequenceRunner, _world_to_camera
    from unimatch_b200.synthetic import synthetic_model, synthetic_posed_sequence, workload_call
    if not torch.cuda.is_available():
        raise SystemExit("depth_fusion_bench: needs a CUDA device")
    dev = torch.device("cuda", 0)
    B, T, H, W = args.batch, args.frames, args.height, args.width
    m, call = synthetic_model(MODEL), workload_call(MODEL)
    kw = {k: v for k, v in call.items() if k not in _DEPTH_RANGE + ("task",)}
    frames, K, poses = synthetic_posed_sequence(T, H, W, seed=2017)
    items = list(zip(frames.numpy(), poses.numpy()))
    host_poses = poses.numpy()
    pairs = T - 1

    def volume():
        return TSDFVolume.covering(K, host_poses, (H, W), args.max_depth, args.voxel, device=dev)

    vols = {k: volume() for k in ("runner", "fuse_depths", "today")}
    fusion_runner = DepthFusionRunner(m, (H, W), B, dev, K, vols["runner"], return_depth=False, **kw)
    depth_runner = DepthSequenceRunner(m, (H, W), B, dev, K, **kw)

    def arm_runner():
        vols["runner"].reset()
        for _ in fusion_runner.run(items):
            pass

    def depths_on_host():
        return torch.stack([r["depth"].clone() for r in depth_runner.run(items)])

    def arm_fuse_depths():
        vols["fuse_depths"].reset()
        d = depths_on_host()
        fuse_depths(vols["fuse_depths"], d.pin_memory().to(dev, non_blocking=True),
                    frames[:-1].pin_memory().to(dev, non_blocking=True), K, host_poses[:-1])

    def arm_today():
        vols["today"].reset()
        d = depths_on_host().to(dev)
        torch_integrate(vols["today"], d, frames[:-1].to(dev), host_poses[:-1], K)

    arms = {"runner": arm_runner, "fuse_depths": arm_fuse_depths, "today": arm_today}
    peaks, times = {}, {k: [] for k in arms}
    for name, fn in arms.items():                       # warm-up pass: graph captures, module caches, allocator
        torch.cuda.reset_peak_memory_stats(dev)
        timed(fn)
        peaks[name] = torch.cuda.max_memory_allocated(dev)
    for _ in range(args.repeats):
        for name, fn in arms.items():
            times[name].append(timed(fn)[0])

    ref = vols["runner"]
    agreement = {k: (vols[k].tsdf - ref.tsdf).abs().max().item() for k in ("fuse_depths", "today")}
    agreement["weights_differ_fraction"] = {k: torch.ne(vols[k].weight, ref.weight).float().mean().item()
                                            for k in ("fuse_depths", "today")}

    # um_tsdf_integrate at the step's shape: B depth maps of H x W into the volume
    vol = volume()
    d = depths_on_host()[:B].to(dev).contiguous()
    f = frames[:B].to(dev).contiguous()
    w2c = torch.from_numpy(_world_to_camera(host_poses[:B])).to(dev)
    nv = torch.tensor([B], dtype=torch.int32, device=dev)
    before = vol.weight.clone()
    vol._integrate(d, f, w2c, nv, K)
    touched = torch.ne(vol.weight, before).sum().item()
    voxels = vol.tsdf.numel()
    inputs = B * H * W * (4 + 3) + B * 48
    ms = _event_ms(lambda: vol._integrate(d, f, w2c, nv, K), args.kernel_iters)

    def rate(nbytes):
        return {"bytes": nbytes, "GB_s": round(nbytes / ms / 1e6, 1),
                "share_of_3350_GB_s": round(nbytes / ms / 1e6 / HBM_DATASHEET_GBS, 4)}
    integrate = {"ms": round(ms, 4), "voxels": voxels, "touched_voxels": touched, "frames": B,
                 "dense_state": rate(inputs + 40 * voxels), "touched_state": rate(inputs + 40 * touched)}

    vol = vols["runner"]
    ext = []
    for _ in range(5):
        sec, (pts, _) = timed(vol.extract_points)
        ext.append(sec)

    fps = {k: round(pairs / statistics.median(v), 2) for k, v in times.items()}
    X, Y, Z = vols["runner"].dims
    print(json.dumps({
        "card": card(), "model": MODEL, "frame_size": [H, W], "frames": T, "fused_frames": pairs, "batch": B,
        "volume": {"dims": [X, Y, Z], "voxel_size": args.voxel, "max_depth": args.max_depth,
                   "GiB": round(20 * X * Y * Z / 2 ** 30, 3)},
        "repeats": args.repeats, "frames_per_s": fps,
        "runner_speedup_vs_fuse_depths": round(fps["runner"] / fps["fuse_depths"], 3),
        "runner_speedup_vs_today": round(fps["runner"] / fps["today"], 3),
        "seconds": {k: [round(x, 4) for x in v] for k, v in times.items()},
        "peak_device_memory_GiB": {k: round(v / 2 ** 30, 3) for k, v in peaks.items()},
        "um_tsdf_integrate": integrate,
        "extract_points": {"ms_median": round(1000 * statistics.median(ext), 3), "points": int(pts.shape[0])},
        "agreement_max_abs_tsdf_vs_runner": agreement, "time": time.strftime("%Y-%m-%d %H:%M:%S")}))


if __name__ == "__main__":
    main()
