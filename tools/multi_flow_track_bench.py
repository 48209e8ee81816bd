#!/usr/bin/env python
"""Multi-flow dense point tracks over a video on one GPU: the encode-once runner against the pairwise forward, and what the
extra pairs cost next to the consecutive-pair tracks.

    python tools/multi_flow_track_bench.py [--workload config4|config2] [--steps K] [--batch B] [--repeats R]

Three paths run the same synthetic clip of 1 + K * B uint8 frames (bench.py's workload, size and weights), alternating
clip by clip:
  * runner:    `MultiFlowTrackRunner` with the default gaps (1, 2, 4, 8, 16, 32) and the anchor, B new frames per step,
               CUDA graph: every frame encoded once, 7 pairs per new frame gathered from the feature ring;
  * pairwise:  the same pairs through `infer_flow(..., pred_bidir_flow=True)`, B frames' pairs per call (every pair encodes
               both of its frames), then one `multi_flow_tracks` over the clip; the frames are on the device beforehand;
  * chain:     `VideoTrackRunner` (consecutive pairs only, `um_chain_tracks`), B pairs per step, CUDA graph.
Frames/s are new frames over the wall time of the whole clip; pairs/s count the pairs each path computes: the runner
computes K pairs for every frame, filling the absent sources of the first max(gaps) frames, the pairwise path only the
present ones.  `um_fb_consistency_error` and `um_multi_flow_tracks` alone
are timed with CUDA events around each of many launches at the runner's step shape on seeded random inputs; their bytes
are computed from shapes (each buffer read or written once).  The card's name, power limit and maximum SM clock are read
in the same run.  Prints ONE JSON line; writes nothing.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import BENCH_WORKLOADS  # noqa: E402
from tools.common import card as read_card, timed  # noqa: E402

HBM_BYTES_PER_S = 3.35e12          # H100 SXM HBM3, NVIDIA data sheet


def event_ms(fn, launches, before=None):
    """mean ms of fn() between CUDA events, `before()` (outside the events) ahead of each launch"""
    for _ in range(5):
        fn()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(launches)]
    for a, b in ev:
        if before is not None:
            before()
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return sum(a.elapsed_time(b) for a, b in ev) / launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="config4", choices=["config4", "config2"])
    ap.add_argument("--steps", type=int, default=32, help="K: steps per clip (the default reaches past max(gaps) = 32)")
    ap.add_argument("--batch", type=int, default=2, help="B: new frames per step")
    ap.add_argument("--warmup", type=int, default=1, help="clips per path before timing")
    ap.add_argument("--repeats", type=int, default=3, help="timed clips per path")
    ap.add_argument("--kernel-launches", type=int, default=200)
    args = ap.parse_args()
    from unimatch_b200.inference import (MULTI_FLOW_GAPS, MultiFlowTrackRunner, VideoTrackRunner, infer_flow,
                                         multi_flow_sources, multi_flow_tracks)
    from unimatch_b200.spec import WORKLOADS
    from unimatch_b200.synthetic import synthetic_model, synthetic_video, workload_call
    wl_name, H, W, _, cfg_idx, _, _ = BENCH_WORKLOADS[args.workload]
    cfg = WORKLOADS[wl_name]
    B, gaps = args.batch, MULTI_FLOW_GAPS
    K = len(gaps) + 1
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    card = read_card()
    model = synthetic_model(wl_name, dev)
    call = workload_call(wl_name, drop=("task",))
    video = synthetic_video(1 + args.steps * B, H, W, seed=77)
    frames = list(video.numpy())
    T = len(frames)
    mf = MultiFlowTrackRunner(model, (H, W), B, dev, gaps=gaps, padding_factor=cfg["pad"], **call)
    ch = VideoTrackRunner(model, (H, W), B, dev, padding_factor=cfg["pad"], **call)
    images = video.permute(0, 3, 1, 2).float().to(dev)
    srcs = [multi_flow_sources(t, gaps, True) for t in range(1, T)]
    present = sum(s >= 0 for row in srcs for s in row)
    last = {}

    def run_runner():
        for r in mf.run(frames):
            last["runner"] = r["visible"].float().mean().item()

    def run_pairwise():
        fwd = torch.zeros((T - 1, K, 2, H, W), device=dev)
        bwd = torch.zeros_like(fwd)
        for t0 in range(1, T, B):
            ts = range(t0, min(t0 + B, T))
            first = [s for t in ts for s in srcs[t - 1] if s >= 0]
            second = [t for t in ts for s in srcs[t - 1] if s >= 0]
            out = infer_flow(model, images[first], images[second], padding_factor=cfg["pad"], pred_bidir_flow=True, **call)
            i = 0
            for t in ts:
                idx = [j for j, s in enumerate(srcs[t - 1]) if s >= 0]
                fwd[t - 1, idx], bwd[t - 1, idx] = out["flow"][i:i + len(idx)], out["flow_bwd"][i:i + len(idx)]
                i += len(idx)
        res = multi_flow_tracks(fwd, bwd, gaps, True)
        last["pairwise"] = res["visible"][-1].float().mean().item()

    def run_chain():
        for _ in ch.run(frames):
            pass

    paths = [("runner", run_runner, (T - 1) * K), ("pairwise", run_pairwise, present), ("chain", run_chain, T - 1)]
    for _ in range(max(args.warmup, 1)):
        for _, fn, _ in paths:
            fn()
    secs = {k: 0.0 for k, _, _ in paths}
    for _ in range(args.repeats):
        for k, fn, _ in paths:
            secs[k] += timed(fn)[0]

    # the two kernels alone at the runner's step shape
    ops = torch.ops.unimatch_sm100
    g = torch.Generator(device=dev).manual_seed(5)
    n = B * K
    fl = torch.randn((n, 2, H, W), device=dev, generator=g) * 2
    fb = -fl + 0.3 * torch.randn((n, 2, H, W), device=dev, generator=g)
    fb_ms = event_ms(lambda: ops.fb_consistency_error(fl, fb, 0.01, 0.5), args.kernel_launches)
    occ, _, err = ops.fb_consistency_error(fl, fb, 0.01, 0.5)
    slots = max(gaps) + B + 1
    pos = torch.empty((slots, H, W, 2), device=dev)
    sig = torch.rand((slots, H, W), device=dev, generator=g)
    vis = torch.ones((slots, H, W), device=dev, dtype=torch.uint8)
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32, device=dev), torch.arange(W, dtype=torch.float32,
                                                                                            device=dev), indexing="ij")
    start = torch.stack((xs, ys), -1)
    t_mid = 40                                      # a frame past max(gaps): all K sources present
    ring = lambda f: 0 if f == 0 else 1 + (f - 1) % (slots - 1)
    src = torch.tensor([[ring(s) for s in multi_flow_sources(t, gaps, True)] for t in range(t_mid, t_mid + B)],
                       dtype=torch.int32, device=dev)
    dst = torch.tensor([ring(t) for t in range(t_mid, t_mid + B)], dtype=torch.int32, device=dev)

    def reset():
        pos.copy_(start.expand_as(pos))
        vis.fill_(1)
    reset()
    mf_ms = event_ms(lambda: ops.multi_flow_tracks(fl.view(B, K, 2, H, W), occ.view(B, K, H, W), err.view(B, K, H, W),
                                                   src, dst, pos, sig, vis), args.kernel_launches, reset)
    hw = H * W
    fb_bytes = n * hw * (8 + 8 + 4 + 4 + 4)                      # both flows read, two masks and the residual written
    mf_bytes = B * hw * (K * (8 + 4 + 4 + 13) + 13 + 13)          # per candidate flow, mask, residual, source state;
    kernel = {}                                                   # per frame its state and outputs written
    for name, ms, nbytes in (("um_fb_consistency_error", fb_ms, fb_bytes), ("um_multi_flow_tracks", mf_ms, mf_bytes)):
        kernel[name] = {"ms": round(ms, 4), "bytes": int(nbytes), "GB_per_s": round(nbytes / ms / 1e6, 1),
                        "share_of_hbm_peak": round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 3)}
    step_ms = secs["runner"] / args.repeats / args.steps * 1e3
    for v in kernel.values():
        v["share_of_runner_step"] = round(v["ms"] / step_ms, 5)

    res = {"metric": "frames/s of multi-flow dense point tracks @%dx%d %s: encode-once runner vs pairwise forward vs "
                     "consecutive-pair chain" % (H, W, wl_name),
           "card": card, "device": torch.cuda.get_device_name(dev),
           "workload": "%s %dx%d, gaps %s + anchor (%d pairs per new frame), %d new frames per step, %d steps per clip "
                       "(BASELINE configs[%d])" % (wl_name, H, W, list(gaps), K, B, args.steps, cfg_idx),
           "repeats": args.repeats, "data": "synthetic_video seed 77",
           "paths": {k: {"frames_per_s": round((T - 1) * args.repeats / secs[k], 3),
                         "pairs_per_s": round(p * args.repeats / secs[k], 3),
                         "ms_per_step": round(secs[k] / args.repeats / args.steps * 1e3, 3)} for k, _, p in paths},
           "kernels_at_step_shape": kernel,
           "kernel_note": "CUDA events around each launch, mean of %d; bytes from shapes; share of the 3.35 TB/s HBM3 "
                          "data-sheet figure" % args.kernel_launches,
           "visible_fraction_last_frame": {k: round(v, 4) for k, v in last.items()}}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
