#!/usr/bin/env python
"""Stereo scene flow over a stereo clip, three ways, on one GPU.

    python tools/scene_flow_bench.py [--batch 4] [--frames 21] [--height 375] [--width 1242] [--repeats 3]

Synthetic gmstereo-scale2-regrefine3 and gmflow-scale2-regrefine6 (their workloads' keywords) on a seeded stereo clip at
KITTI's 375x1242 with padding factor 32 for both networks (384x1248), 21 frames (the length of a KITTI multiview clip), so
20 consecutive pairs.  Arms, each from host uint8 frames to host outputs:
  (a) `SceneFlowRunner`: each frame's stereo once, each left frame encoded once, one CUDA graph per step;
  (b) `infer_scene_flow` per quadruple, `--batch` quadruples per call, uploaded from host uint8 and downloaded;
  (c) what a user writes without it: `StereoRunner` over every frame, `VideoFlowRunner` over the left frames, and the second
      disparity warped on the CPU with grid_sample(padding_mode='border', align_corners=True).
After one warm-up pass of every arm (graph captures included) the arms alternate for `--repeats` rounds; each arm's
pairs/s is the median round (a pair per frame after the first, so it is also frames/s).  Also reported: CUDA-event times of
`um_warp_disparity` and `um_scene_flow_stats` (noc set and obj_map on) at [batch, 375, 1242] with the bytes they must move,
computed from shapes, and the share of the H100 SXM data-sheet 3.35 TB/s; each arm's peak device memory in its warm-up pass (the runner goes first, so its figure is the two networks and
its graphs alone; the later arms' figures include the memory the earlier runners still hold); the largest
difference of the runner's outputs from (b)'s; the card's name, power limit and SM clocks, read in the same run.
Prints ONE JSON line.  Writes nothing to the tree.
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
STEREO, FLOW = "gmstereo-scale2-regrefine3", "gmflow-scale2-regrefine6"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--frames", type=int, default=21)
    ap.add_argument("--height", type=int, default=375)
    ap.add_argument("--width", type=int, default=1242)
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


@torch.no_grad()
def run(args):
    import torch.nn.functional as F
    from unimatch_b200.inference import SceneFlowRunner, StereoRunner, VideoFlowRunner, infer_scene_flow
    from unimatch_b200.synthetic import synthetic_model, synthetic_stereo_video, workload_call
    if not torch.cuda.is_available():
        raise SystemExit("scene_flow_bench: needs a CUDA device")
    dev = torch.device("cuda", 0)
    B, T, H, W = args.batch, args.frames, args.height, args.width
    sm, fm = synthetic_model(STEREO), synthetic_model(FLOW)
    skw, fkw = workload_call(STEREO), workload_call(FLOW)
    left, right = synthetic_stereo_video(T, H, W, seed=2015)
    items = [(left[t].numpy(), right[t].numpy()) for t in range(T)]
    pairs = T - 1
    geometry = dict(stereo_padding_factor=32, flow_padding_factor=32, stereo_kwargs=skw, flow_kwargs=fkw)

    runner = SceneFlowRunner(sm, fm, (H, W), B, dev, **geometry)
    stereo_runner = StereoRunner(sm, (H, W), B, dev, padding_factor=32, **skw)
    flow_runner = VideoFlowRunner(fm, (H, W), B, dev, padding_factor=32, **fkw)

    def arm_runner():
        return [{k: v.clone() for k, v in r.items()} for r in runner.run(items)]

    def arm_quadruples():
        out = []
        for t0 in range(0, pairs, B):
            t1 = min(t0 + B, pairs)
            views = [x.pin_memory().to(dev, non_blocking=True) for x in (left[t0:t1], right[t0:t1], left[t0 + 1:t1 + 1],
                                                                          right[t0 + 1:t1 + 1])]
            r = infer_scene_flow(sm, fm, *views, **geometry)
            host = {k: v.cpu() for k, v in r.items()}
            out.extend({k: v[i] for k, v in host.items()} for i in range(t1 - t0))
        return out

    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")

    def arm_today():
        disps = [r["disp"].clone() for r in stereo_runner.run(items)]
        flows = [r["flow"].clone() for r in flow_runner.run([f for f, _ in items])]
        out = []
        for t, flow in enumerate(flows):
            gx = (xs + flow[0]) / (W - 1) * 2 - 1
            gy = (ys + flow[1]) / (H - 1) * 2 - 1
            d1 = F.grid_sample(disps[t + 1][None, None], torch.stack((gx, gy), -1)[None], mode="bilinear",
                               padding_mode="border", align_corners=True)[0, 0]
            out.append({"disp_0": disps[t], "disp_1": d1, "flow": flow})
        return out

    arms = {"runner": arm_runner, "per_quadruple": arm_quadruples, "today": arm_today}
    results, peaks, times = {}, {}, {k: [] for k in arms}
    for name, fn in arms.items():                       # warm-up pass: graph captures, module caches, allocator
        torch.cuda.reset_peak_memory_stats(dev)
        results[name] = timed(fn)[1]
        peaks[name] = torch.cuda.max_memory_allocated(dev)
    for _ in range(args.repeats):
        for name, fn in arms.items():
            times[name].append(timed(fn)[0])

    def worst(a, b, key):
        return max((x[key].float() - y[key].float()).abs().max().item() / max(y[key].abs().max().item(), 1e-30)
                   for x, y in zip(results[a], results[b]))
    agreement = {"runner_vs_per_quadruple_rel": {k: worst("runner", "per_quadruple", k) for k in ("disp_0", "disp_1", "flow")},
                 "today_vs_per_quadruple_rel": {k: worst("today", "per_quadruple", k) for k in ("disp_0", "disp_1", "flow")}}

    # the two new kernels at [B, H, W]
    ops = torch.ops.unimatch_sm100
    g = torch.Generator(device=dev).manual_seed(7)
    disp = torch.rand((B, H, W), device=dev, generator=g) * 90
    flow = torch.randn((B, 2, H, W), device=dev, generator=g) * 20
    gt = [torch.rand((B, H, W), device=dev, generator=g) * 90, torch.rand((B, H, W), device=dev, generator=g) * 90,
          torch.randn((B, 2, H, W), device=dev, generator=g) * 20, (torch.rand((B, H, W), device=dev, generator=g) < 0.9).float()]
    obj = (torch.rand((B, H, W), device=dev, generator=g) < 0.2).float()
    px = B * H * W
    kernels = {}
    for name, fn, nbytes in (
            ("um_warp_disparity", lambda: ops.warp_disparity(disp, flow), px * (4 + 8 + 4 + 1)),
            ("um_scene_flow_stats", lambda: ops.scene_flow_stats(disp, disp, flow, *gt, *gt, obj), px * (16 + 2 * 20 + 4))):
        ms = _event_ms(fn, args.kernel_iters)
        kernels[name] = {"ms": round(ms, 4), "bytes": nbytes, "GB_s": round(nbytes / ms / 1e6, 1),
                         "share_of_3350_GB_s": round(nbytes / ms / 1e6 / HBM_DATASHEET_GBS, 3)}

    fps = {k: round(pairs / statistics.median(v), 2) for k, v in times.items()}
    print(json.dumps({
        "card": card(), "models": [STEREO, FLOW], "frame_size": [H, W], "inference_size": [-(-H // 32) * 32, -(-W // 32) * 32],
        "frames": T, "pairs": pairs, "batch": B, "repeats": args.repeats,
        "pairs_per_s": fps, "ms_per_pair": {k: round(1000.0 / v, 2) for k, v in fps.items()},
        "runner_speedup_vs_per_quadruple": round(fps["runner"] / fps["per_quadruple"], 3),
        "runner_speedup_vs_today": round(fps["runner"] / fps["today"], 3),
        "seconds": {k: [round(x, 4) for x in v] for k, v in times.items()},
        "peak_device_memory_GiB": {k: round(v / 2 ** 30, 3) for k, v in peaks.items()},
        "kernels": kernels, "agreement": agreement, "time": time.strftime("%Y-%m-%d %H:%M:%S")}))


if __name__ == "__main__":
    main()
