#!/usr/bin/env python
"""Video optical flow against pairwise inference on the same consecutive pairs, on one GPU.

    python tools/video_bench.py [--workload config4|config2] [--steps K] [--warmup W] [--pairs-per-step B]

The timed video step is what `unimatch_b200.VideoFlowRunner` does per step: B new synthetic uint8 frames are copied from pinned
memory, converted on the device (`um_frames_to_planar`), encoded, paired with the previous step's last frame (its feature
pyramid is carried, not re-encoded) and run as B pairs; the flow goes back to pinned memory.  The pairwise step is
`UniMatch.forward` on the same B pairs, uploaded as two float32 images per pair and downloaded the same way.  The two steps
alternate in one process, eager on both sides, and the workloads, sizes and weights are those of bench.py.  Prints ONE JSON
line: pairs/s of each path, the encoder ("backbone") section time of each, H2D / D2H bytes per step, and how far the two
outputs are apart (they are not bit-identical: see `UniMatch.encode_frames`).  Exits non-zero beyond 1e-4 of the largest flow.
Writes nothing to the tree.
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
    ap.add_argument("--workload", default="config4", choices=["config4", "config2"])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--pairs-per-step", type=int, default=0, help="B (default: the workload's pairs per GPU in bench.py)")
    args = ap.parse_args()
    run(args)


def run(args):
    """One VideoFlowRunner step (B new synthetic uint8 frames uploaded from pinned memory, the previous step's last
    frame carried, B pairs, flow back to pinned memory) against `UniMatch.forward` on the same B pairs as float32 images
    (uploaded and downloaded the same way), alternating step by step in one process, eager on both sides."""
    from unimatch_b200 import UniMatch, ops
    from unimatch_b200.inference import VideoFlowRunner
    from unimatch_b200.spec import WORKLOADS
    from unimatch_b200.synthetic import BENCH_WEIGHTS, synthetic_state_dict, synthetic_video
    wl_name, H, W, ppg, cfg_idx, _, _ = BENCH_WORKLOADS[args.workload]
    cfg = WORKLOADS[wl_name]
    if cfg["model"]["task"] != "flow":
        raise SystemExit("video inference runs the flow workloads only (config4, config2)")
    B = args.pairs_per_step or ppg
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    model = UniMatch(**cfg["model"]).eval()
    model.load_state_dict(synthetic_state_dict(seed=326, **BENCH_WEIGHTS, **cfg["model"]), strict=True)
    model = model.to(dev)
    call = {k: v for k, v in cfg["call"].items() if k != "task"}
    frames = synthetic_video(B + 1, H, W, seed=77)                          # frame 0 = carried, frames 1..B = new
    runner = VideoFlowRunner(model, (H, W), B, dev, padding_factor=cfg["pad"], use_graph=False, **call)
    runner.carry = [f.clone() for f in runner._encode(frames[:1].to(dev))]
    saved = [c.clone() for c in runner.carry]                                # frame 0's pyramid
    pin_new = frames[1:].contiguous().pin_memory()
    planar = frames.permute(0, 3, 1, 2).float()
    pin0, pin1 = planar[:-1].contiguous().pin_memory(), planar[1:].contiguous().pin_memory()
    out_v, out_p = torch.empty((B, 2, H, W)).pin_memory(), torch.empty((B, 2, H, W)).pin_memory()

    def video_step():
        for c, f in zip(runner.carry, saved):                                # same pairs every step: (0,1), (1,2), ...
            c.copy_(f)
        runner.dev_in[0].copy_(pin_new, non_blocking=True)
        out_v.copy_(runner._step(0)["flow"], non_blocking=True)

    def pair_step():
        a, b = pin0.to(dev, non_blocking=True), pin1.to(dev, non_blocking=True)
        out_p.copy_(model(a, b, **cfg["call"])["flow_preds"][-1], non_blocking=True)

    for _ in range(max(args.warmup, 2)):
        video_step(); pair_step()
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

    ms_v, ms_p = timed([video_step, pair_step], args.steps)
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
    res = {"metric": "pairs/s of consecutive video pairs @%dx%d %s, video path vs pairwise forward" % (H, W, wl_name),
           "device": props.name, "workload": "%s %dx%d, %d pairs per step (BASELINE configs[%d])" % (wl_name, H, W, B, cfg_idx),
           "steps": args.steps, "warmup": max(args.warmup, 2), "data": "synthetic_video seed 77", "cuda_graph": False,
           "video": {"pairs_per_s": B / (ms_v / 1e3), "ms_per_step": round(ms_v, 3),
                     "sections_ms_per_step": {"backbone": sections["video"].get("backbone")},
                     "h2d_bytes_per_step": int(pin_new.numel()), "d2h_bytes_per_step": int(out_v.numel() * 4),
                     "note": "B new frames encoded, the carried frame's pyramid reused (restored to frame 0's by a device copy "
                             "inside the step so that every step runs the same pairs)"},
           "pairwise": {"pairs_per_s": B / (ms_p / 1e3), "ms_per_step": round(ms_p, 3),
                        "sections_ms_per_step": {"backbone": sections["pairwise"].get("backbone")},
                        "h2d_bytes_per_step": int((pin0.numel() + pin1.numel()) * 4), "d2h_bytes_per_step": int(out_p.numel() * 4)},
           "speedup": ms_p / ms_v, "outputs_bit_identical": identical, "max_abs_diff_rel_to_max_flow": rel_diff,
           "identity_note": "um_conv2d_tc sums a tile's K chunks in an order rotated by the CTA owning the tile; encoding B frames "
                            "instead of 2B changes the tile-to-CTA map, hence the last bits (tolerance 1e-4 of the largest flow)",
           "launches_per_process": ops.launch_count()}
    print(json.dumps(res))
    if rel_diff > 1e-4:
        sys.exit(1)


if __name__ == "__main__":
    main()
