#!/usr/bin/env python
"""The multi-view consistency filter of depth maps on one GPU.

    python tools/consistency_bench.py [--batch 8] [--frames 65] [--height 480] [--width 640] [--views 4] [--repeats 3]

Synthetic gmdepth-scale1-regrefine1 (its workload's keywords) on `depth_fusion_bench`'s seeded `synthetic_posed_sequence`
clip at 480x640, 65 frames (64 pairs), fused at 1 cm voxels into `TSDFVolume.covering` up to 2.5 m.  Reported:
  * `DepthFusionRunner` frames/s with `consistency_views` 0 and `--views` (min_views 2), after one warm-up pass of each,
    alternated for `--repeats` rounds (volume and ring reset before each), the median round per arm;
  * CUDA-event times of `um_depth_consistency` over `--kernel-iters` launches at the runner step's shape (`--views` +
    batch maps, batch references, `--views` sources) and at 64 frames x 8 sources (`sequence_sources(64, 4, 4)`), on the
    runner's own depths, with the bytes it must move computed from shapes (every map read once, views and depth written
    once) and their share of the H100 SXM data-sheet 3.35 TB/s;
  * the same check restated in torch ops with `grid_sample` (bilinear, align_corners=True, the four taps' validity
    sampled as a mask) on the same inputs: its time and the number of pixels whose kept / dropped decision differs;
  * `depth_points` of the 64 filtered frames: its time and point count P;
  * the card's name, power limit and SM clocks, read in the same run.
The synthetic weights' depths are not meaningful: this measures speed, not reconstruction quality.  Prints ONE JSON line.
Writes nothing to the tree.
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

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
    ap.add_argument("--views", type=int, default=4)
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


def torch_filter(depth, c2w, w2c, K, sources, min_views, max_pixel=1.0, max_relative=0.01):
    """The check in torch ops, pair by pair with grid_sample (what a user writes without the kernel): counts [N,H,W]"""
    n, h, w = depth.shape
    dev = depth.device
    fx, fy, cx, cy = float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])
    ys, xs = torch.meshgrid(torch.arange(h, device=dev, dtype=torch.float32),
                            torch.arange(w, device=dev, dtype=torch.float32), indexing="ij")
    valid = torch.isfinite(depth) & (depth > 0)
    clean = torch.where(valid, depth, torch.zeros_like(depth))
    counts = torch.zeros((n, h, w), dtype=torch.int32, device=dev)
    for r in range(n):
        d = clean[r]
        p = torch.stack(((xs - cx) / fx * d, (ys - cy) / fy * d, d), 0).reshape(3, -1)
        world = c2w[r, :, :3] @ p + c2w[r, :, 3:]
        for s in sources[r].tolist():
            if s < 0:
                continue
            c = w2c[s, :, :3] @ world + w2c[s, :, 3:]
            u, v = fx * c[0] / c[2] + cx, fy * c[1] / c[2] + cy
            grid = torch.stack((2 * u / (w - 1) - 1, 2 * v / (h - 1) - 1), -1).view(1, h, w, 2)
            ds = F.grid_sample(clean[s][None, None], grid, mode="bilinear", align_corners=True).view(-1)
            vs = F.grid_sample(valid[s][None, None].float(), grid, mode="bilinear", align_corners=True).view(-1)
            q = torch.stack(((u - cx) / fx * ds, (v - cy) / fy * ds, ds), 0)
            back = w2c[r, :, :3] @ (c2w[s, :, :3] @ q + c2w[s, :, 3:]) + w2c[r, :, 3:]
            u2, v2 = fx * back[0] / back[2] + cx, fy * back[1] / back[2] + cy
            err = torch.sqrt((u2 - xs.reshape(-1)) ** 2 + (v2 - ys.reshape(-1)) ** 2)
            rel = (back[2] - d.view(-1)).abs() / d.view(-1)
            ok = valid[r].view(-1) & (c[2] > 0) & (u >= 0) & (u <= w - 1) & (v >= 0) & (v <= h - 1) & (vs >= 1 - 1e-6) \
                & (back[2] > 0) & (err < max_pixel) & (rel < max_relative)
            counts[r] += ok.view(h, w).int()
    return counts


@torch.no_grad()
def run(args):
    from unimatch_b200.fusion import TSDFVolume, depth_points, filter_depths, sequence_sources
    from unimatch_b200.inference import DepthFusionRunner, DepthSequenceRunner, _camera_to_world, _world_to_camera
    from unimatch_b200.synthetic import synthetic_model, synthetic_posed_sequence, workload_call
    if not torch.cuda.is_available():
        raise SystemExit("consistency_bench: needs a CUDA device")
    dev = torch.device("cuda", 0)
    B, T, H, W, k = args.batch, args.frames, args.height, args.width, args.views
    m, call = synthetic_model(MODEL), workload_call(MODEL)
    kw = {key: v for key, v in call.items() if key not in _DEPTH_RANGE + ("task",)}
    frames, K, poses = synthetic_posed_sequence(T, H, W, seed=2017)
    items = list(zip(frames.numpy(), poses.numpy()))
    host_poses = poses.numpy()
    pairs = T - 1

    def volume():
        return TSDFVolume.covering(K, host_poses, (H, W), args.max_depth, args.voxel, device=dev)

    runners = {"consistency_views_0": DepthFusionRunner(m, (H, W), B, dev, K, volume(), return_depth=False, **kw),
               "consistency_views_%d" % k: DepthFusionRunner(m, (H, W), B, dev, K, volume(), return_depth=False,
                                                             consistency_views=k, consistency_min_views=2, **kw)}

    def arm(runner):
        def go():
            runner.reset_scene()
            for _ in runner.run(items):
                pass
        return go

    arms = {name: arm(r) for name, r in runners.items()}
    times = {name: [] for name in arms}
    for fn in arms.values():                                # warm-up pass: graph captures, module caches, allocator
        timed(fn)
    for _ in range(args.repeats):
        for name, fn in arms.items():
            times[name].append(timed(fn)[0])
    fps = {name: round(pairs / statistics.median(v), 2) for name, v in times.items()}

    depths = torch.stack([r["depth"].clone() for r in DepthSequenceRunner(m, (H, W), B, dev, K, **kw).run(items)]).to(dev)
    ps = list(host_poses[:-1])
    c2w = torch.from_numpy(_camera_to_world(ps)).to(dev)
    w2c = torch.from_numpy(_world_to_camera(ps)).to(dev)
    fx, fy, cx, cy = float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])
    ops = torch.ops.unimatch_sm100

    def kernel(n_maps, refs, table):
        d = depths[:n_maps].contiguous()
        refs_d = torch.tensor(refs, dtype=torch.int32, device=dev)
        table_d = torch.from_numpy(np.ascontiguousarray(table, np.int32)).to(dev)
        ms = _event_ms(lambda: ops.depth_consistency(d, c2w[:n_maps].contiguous(), w2c[:n_maps].contiguous(), refs_d,
                                                     table_d, fx, fy, cx, cy, 1.0, 0.01, 2), args.kernel_iters)
        nbytes = n_maps * H * W * 4 + len(refs) * H * W * 5 + n_maps * 96 + 4 * table.size + 4 * len(refs)
        return {"maps": n_maps, "references": len(refs), "sources": int(table.shape[1]), "ms": round(ms, 4),
                "bytes": nbytes, "GB_s": round(nbytes / ms / 1e6, 1),
                "share_of_3350_GB_s": round(nbytes / ms / 1e6 / HBM_DATASHEET_GBS, 4)}

    step_table = (np.arange(B)[:, None] + k - np.arange(1, k + 1)[None, :]).astype(np.int32)
    step = kernel(k + B, list(range(k, k + B)), step_table)
    n64 = min(64, depths.shape[0])
    src64 = sequence_sources(n64, 4, 4)
    clip = kernel(n64, list(range(n64)), src64)

    out = filter_depths(depths[:n64], K, ps[:n64], src64, min_views=2)
    sec_torch = []
    for _ in range(3):
        sec, counts = timed(lambda: torch_filter(depths[:n64], c2w[:n64], w2c[:n64], K, src64, 2))
        sec_torch.append(sec)
    differ = torch.ne(counts >= 2, out["views"] >= 2).sum().item()
    restated = {"ms_median": round(1000 * statistics.median(sec_torch), 2), "decision_differs_pixels": int(differ),
                "pixels": n64 * H * W, "kept_by_kernel": int((out["views"] >= 2).sum().item()),
                "count_differs_pixels": int(torch.ne(counts, out["views"].int()).sum().item())}

    pts_t = []
    f64 = frames[:n64].to(dev)
    for _ in range(5):
        sec, (pts, _) = timed(lambda: depth_points(out["depth"], f64, K, ps[:n64]))
        pts_t.append(sec)

    print(json.dumps({
        "card": card(), "model": MODEL, "frame_size": [H, W], "frames": T, "fused_frames": pairs, "batch": B,
        "repeats": args.repeats, "frames_per_s": fps, "seconds": {key: [round(x, 4) for x in v] for key, v in times.items()},
        "um_depth_consistency": {"step": step, "clip_64x8": clip}, "torch_grid_sample_restatement_64x8": restated,
        "depth_points_64": {"ms_median": round(1000 * statistics.median(pts_t), 3), "points": int(pts.shape[0])},
        "time": time.strftime("%Y-%m-%d %H:%M:%S")}))


if __name__ == "__main__":
    main()
