#!/usr/bin/env python
"""Dense point tracks over a video on one GPU: the tracks chained on the device against the flows downloaded and chained on
the host.

    python tools/track_bench.py [--workload config4|config2] [--steps K] [--warmup W] [--pairs-per-step B]

Three paths run the same synthetic clip of 1 + K * B uint8 frames (bench.py's workload, size and weights), alternating
clip by clip, each a CUDA-graph runner over the whole clip:
  * tracks:    `VideoTrackRunner`: forward / backward flow, occlusion masks and `um_chain_tracks` inside the step; only
               'tracks' and 'visible' are downloaded;
  * flow:      `VideoFlowRunner(pred_bidir_flow=True, fwd_bwd_consistency_check=True)`, the same step without the chain,
               downloading the flows and masks;
  * host loop: the flow path, then what a user writes today on the host: each frame's forward flow and mask composed with
               `torch.nn.functional.grid_sample` (align_corners=True, zero padding) on the CPU, one frame at a time.
Pairs/s are pairs over the wall time of the whole clip (every result handed out).  `um_chain_tracks` alone is timed with
CUDA events around each of many launches on B seeded random flows and masks of the step's shape (state reset between
launches, outside the events); its bytes are computed from shapes: the flows, the masks, the state read and written and the outputs written once.
The card's name, power limit and maximum SM clock are read in the same run.  Prints ONE JSON line; writes nothing.
"""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import BENCH_WORKLOADS  # noqa: E402
from tools.common import card as read_card, timed  # noqa: E402


def host_tracks(h, w):
    """The host loop's state and step: p [1,H,W,2] in pixels, vis [H,W] bool; step(flow [2,H,W], occ [H,W]) on the CPU"""
    ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32), indexing="ij")
    state = {"p": torch.stack((xs, ys), -1)[None], "vis": torch.ones((h, w), dtype=torch.bool)}
    scale = torch.tensor([2.0 / (w - 1), 2.0 / (h - 1)])

    def step(flow, occ):
        p = state["p"]
        grid = p * scale - 1
        d = F.grid_sample(flow[None], grid, mode="bilinear", padding_mode="zeros", align_corners=True)[0]
        o = F.grid_sample(occ[None, None], grid, mode="bilinear", padding_mode="zeros", align_corners=True)[0, 0]
        p = p + d.permute(1, 2, 0)[None]
        x, y = p[0, ..., 0], p[0, ..., 1]
        state["vis"] = state["vis"] & (o < 0.5) & (x >= 0) & (x <= w - 1) & (y >= 0) & (y <= h - 1)
        state["p"] = p
        return p[0], state["vis"]
    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="config4", choices=["config4", "config2"])
    ap.add_argument("--steps", type=int, default=5, help="K: steps per clip")
    ap.add_argument("--warmup", type=int, default=1, help="clips per path before timing")
    ap.add_argument("--repeats", type=int, default=3, help="timed clips per path")
    ap.add_argument("--pairs-per-step", type=int, default=0, help="B (default: the workload's pairs per GPU in bench.py)")
    ap.add_argument("--kernel-launches", type=int, default=200)
    args = ap.parse_args()
    from unimatch_b200.inference import VideoFlowRunner, VideoTrackRunner, chain_tracks
    from unimatch_b200.spec import WORKLOADS
    from unimatch_b200.synthetic import synthetic_model, synthetic_video, workload_call
    wl_name, H, W, ppg, cfg_idx, _, _ = BENCH_WORKLOADS[args.workload]
    cfg = WORKLOADS[wl_name]
    B = args.pairs_per_step or ppg
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    card = read_card()
    model = synthetic_model(wl_name, dev)
    call = workload_call(wl_name, drop=("task",))
    frames = list(synthetic_video(1 + args.steps * B, H, W, seed=77).numpy())
    pairs = len(frames) - 1
    tr = VideoTrackRunner(model, (H, W), B, dev, padding_factor=cfg["pad"], **call)
    fr = VideoFlowRunner(model, (H, W), B, dev, padding_factor=cfg["pad"], pred_bidir_flow=True,
                         fwd_bwd_consistency_check=True, **call)
    last = {}

    def run_tracks():
        for r in tr.run(frames):
            last["tracks"] = (r["tracks"].clone(), r["visible"].clone())

    def run_flow():
        for r in fr.run(frames):
            pass

    def run_host():
        step = host_tracks(H, W)
        for r in fr.run(frames):
            p, v = step(r["flow"], r["fwd_occ"])
        last["host"] = (p, v)

    paths = [("tracks", run_tracks), ("flow", run_flow), ("host_loop", run_host)]
    for _ in range(max(args.warmup, 1)):
        for _, fn in paths:
            fn()
    secs = {k: 0.0 for k, _ in paths}
    for _ in range(args.repeats):
        for k, fn in paths:
            secs[k] += timed(fn)[0]

    # parity of the device chain with the host loop on the last frame
    (tp, tv), (hp, hv) = last["tracks"], last["host"]
    both = tv.bool() & hv
    diff = (tp - hp).abs().max(-1).values
    parity = {"max_px_diff": float(diff[diff.isfinite()].max()),
              "max_px_diff_where_both_visible": float(diff[both].max()) if both.any() else None,
              "visibility_differs_fraction": float((tv.bool() != hv).float().mean()),
              "visible_fraction": float(tv.float().mean())}

    # um_chain_tracks alone on B flows and masks of the step's shape
    g = torch.Generator(device=dev).manual_seed(5)
    fl = torch.randn((B, 2, H, W), device=dev, generator=g) * 2
    occ = (torch.rand((B, H, W), device=dev, generator=g) < 0.1).float()
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32, device=dev), torch.arange(W, dtype=torch.float32,
                                                                                            device=dev), indexing="ij")
    start = torch.stack((xs, ys), -1)
    pos, vis = start.clone(), torch.ones((H, W), dtype=torch.uint8, device=dev)
    for _ in range(5):
        chain_tracks(fl, occ, (pos, vis))
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.kernel_launches)]
    for a, b in ev:
        pos.copy_(start)
        vis.fill_(1)
        a.record()
        chain_tracks(fl, occ, (pos, vis))
        b.record()
    torch.cuda.synchronize()
    k_ms = sum(a.elapsed_time(b) for a, b in ev) / len(ev)
    k_bytes = B * H * W * (8 + 4) + H * W * (8 + 1) * 2 + B * H * W * (8 + 1)
    step_ms = secs["tracks"] / args.repeats / args.steps * 1e3

    res = {"metric": "pairs/s of dense point tracks over consecutive video pairs @%dx%d %s, device chain vs host loop"
                     % (H, W, wl_name),
           "card": card, "device": torch.cuda.get_device_name(dev),
           "workload": "%s %dx%d, %d pairs per step, %d steps per clip (BASELINE configs[%d])" % (wl_name, H, W, B,
                                                                                                  args.steps, cfg_idx),
           "repeats": args.repeats, "cuda_graph": True, "data": "synthetic_video seed 77",
           "paths": {k: {"pairs_per_s": round(pairs * args.repeats / secs[k], 3),
                         "ms_per_step": round(secs[k] / args.repeats / args.steps * 1e3, 3)} for k, _ in paths},
           "d2h_bytes_per_frame": {"tracks": 9 * H * W, "flow": 24 * H * W, "host_loop": 24 * H * W,
                                   "host_loop_needed": 12 * H * W},
           "um_chain_tracks": {"ms": round(k_ms, 4), "bytes": int(k_bytes), "GB_per_s": round(k_bytes / k_ms / 1e6, 1),
                               "flows": B, "share_of_track_step": round(k_ms / step_ms, 5),
                               "note": "CUDA events around each launch, mean of %d; bytes from shapes (flows and masks read "
                                       "once, state read and written, outputs written)" % args.kernel_launches},
           "parity_last_frame": parity}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
