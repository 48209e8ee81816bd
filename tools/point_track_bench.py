#!/usr/bin/env python
"""Query point tracks over a video on one GPU: the tracks chained on the device against the flows downloaded and chained
on the host.

    python tools/point_track_bench.py [--workload config4|config2] [--steps K] [--queries N] [--repeats R]

One synthetic clip of 1 + K * B uint8 frames (bench.py's workload, size and weights) and two query sets of N seeded points:
all at frame 0, and spread over every 5th frame but the last.  Two paths run each query set, alternating clip by clip, each
a CUDA-graph runner over the whole clip:
  * device:    `PointTrackRunner.track`: flows, masks and `um_track_points_forward` after each step, the backward history
               on the device, one `um_track_points_backward` launch and one N x T x 9-byte download at the end;
  * host loop: `VideoFlowRunner(pred_bidir_flow=True, fwd_bwd_consistency_check=True)` downloading all four outputs,
               then what a user writes today: `torch.nn.functional.grid_sample` (align_corners=True, zero padding) on the
               points on the CPU, forward from each query's frame as the pairs arrive, backward over the backward flows
               and masks kept on the host.
Pairs/s are pairs over the wall time of the whole clip.  The two launches are timed alone with CUDA events around each of
many launches of the step's shape (B seeded flows and masks, N queries at frame 0) and of the backward launch over the
spread set's history (max(t_q) pairs).  Bytes downloaded and history bytes are computed from shapes.  The card's name,
power limit and maximum SM clock are read in the same run.  Prints ONE JSON line; writes nothing.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import BENCH_WORKLOADS  # noqa: E402
from tools.common import card as read_card, timed  # noqa: E402


def query_sets(n, nframes, h, w, seed=3):
    """{'frame0': N queries at frame 0, 'every5': N queries over frames 0, 5, ... < nframes - 1}, float32 [N,3] (t, y, x)"""
    rng = np.random.default_rng(seed)
    yx = np.stack((rng.random(n) * (h - 1), rng.random(n) * (w - 1)), -1)
    frames = np.arange(0, nframes - 1, 5)
    return {"frame0": np.concatenate((np.zeros((n, 1)), yx), -1).astype(np.float32),
            "every5": np.concatenate((frames[np.arange(n) % len(frames)][:, None], yx), -1).astype(np.float32)}


def host_point_tracks(runner, frames, queries, h, w):
    """The host loop: flows from the runner, points chained with grid_sample on the CPU.  Returns (tracks [N,T,2],
    visible [N,T] bool, bytes downloaded)."""
    q = torch.from_numpy(queries)
    tq = q[:, 0].long()
    nq, nt = q.shape[0], len(frames)
    scale = torch.tensor([2.0 / (w - 1), 2.0 / (h - 1)])
    tracks = torch.empty((nq, nt, 2))
    visible = torch.zeros((nq, nt), dtype=torch.bool)
    start = q[:, [2, 1]]
    tracks[torch.arange(nq), tq] = start
    visible[torch.arange(nq), tq] = True

    def step(p, v, flow, occ):
        grid = (p * scale - 1)[None, None]
        d = F.grid_sample(flow[None], grid, mode="bilinear", padding_mode="zeros", align_corners=True)[0, :, 0].t()
        o = F.grid_sample(occ[None, None], grid, mode="bilinear", padding_mode="zeros", align_corners=True)[0, 0, 0]
        p = p + d
        v = v & (o < 0.5) & (p[:, 0] >= 0) & (p[:, 0] <= w - 1) & (p[:, 1] >= 0) & (p[:, 1] <= h - 1)
        return p, v

    p, v = start.clone(), torch.ones(nq, dtype=torch.bool)
    history, nbytes, tmax = [], 0, int(tq.max())
    for j, r in enumerate(runner.run(frames)):
        nbytes += sum(t.numel() * t.element_size() for t in r.values())
        on = tq <= j
        np_, nv = step(p, v, r["flow"], r["fwd_occ"])
        p, v = torch.where(on[:, None], np_, start), torch.where(on, nv, torch.ones_like(nv))
        tracks[on, j + 1], visible[on, j + 1] = p[on], v[on]
        if j < tmax:
            history.append((r["flow_bwd"].clone(), r["bwd_occ"].clone()))
    p, v = start.clone(), torch.ones(nq, dtype=torch.bool)
    for j in range(tmax - 1, -1, -1):
        on = tq > j
        np_, nv = step(p, v, *history[j])
        p, v = torch.where(on[:, None], np_, start), torch.where(on, nv, torch.ones_like(nv))
        tracks[on, j], visible[on, j] = p[on], v[on]
    return tracks, visible, nbytes


def event_ms(fn, launches, reset=None):
    """mean CUDA-event time of `fn` over `launches` launches (reset, outside the events, before each); common.timed is the
    host-clock time of a whole path"""
    for _ in range(5):
        fn()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(launches)]
    for a, b in ev:
        if reset is not None:
            reset()
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return sum(a.elapsed_time(b) for a, b in ev) / launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="config4", choices=["config4", "config2"])
    ap.add_argument("--steps", type=int, default=5, help="K: steps per clip")
    ap.add_argument("--queries", type=int, default=1024, help="N: queries per set")
    ap.add_argument("--warmup", type=int, default=1, help="clips per path and set before timing")
    ap.add_argument("--repeats", type=int, default=3, help="timed clips per path and set")
    ap.add_argument("--pairs-per-step", type=int, default=0, help="B (default: the workload's pairs per GPU in bench.py)")
    ap.add_argument("--kernel-launches", type=int, default=200)
    args = ap.parse_args()
    from unimatch_b200.inference import PointTrackRunner, VideoFlowRunner
    from unimatch_b200.spec import WORKLOADS
    from unimatch_b200.synthetic import synthetic_model, synthetic_video, workload_call
    ops = torch.ops.unimatch_sm100
    wl_name, H, W, ppg, cfg_idx, _, _ = BENCH_WORKLOADS[args.workload]
    cfg = WORKLOADS[wl_name]
    B = args.pairs_per_step or ppg
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    card = read_card()
    model = synthetic_model(wl_name, dev)
    call = workload_call(wl_name, drop=("task",))
    frames = list(synthetic_video(1 + args.steps * B, H, W, seed=77).numpy())
    T, pairs = len(frames), len(frames) - 1
    sets = query_sets(args.queries, T, H, W)
    pr = PointTrackRunner(model, (H, W), B, dev, padding_factor=cfg["pad"], **call)
    fr = VideoFlowRunner(model, (H, W), B, dev, padding_factor=cfg["pad"], pred_bidir_flow=True,
                         fwd_bwd_consistency_check=True, **call)
    last = {}

    def device_path(name):
        def run():
            last[name, "device"] = pr.track(frames, sets[name])
        return run

    def host_path(name):
        def run():
            last[name, "host"] = host_point_tracks(fr, frames, sets[name], H, W)
        return run

    paths = [((s, p), fn(s)) for s in sets for p, fn in (("device", device_path), ("host_loop", host_path))]
    for _ in range(max(args.warmup, 1)):
        for _, fn in paths:
            fn()
    secs = {k: 0.0 for k, _ in paths}
    for _ in range(args.repeats):
        for k, fn in paths:
            secs[k] += timed(fn)[0]

    results = {}
    for s, q in sets.items():
        tmax = int(q[:, 0].max())
        d, (ht, hv, host_bytes) = last[s, "device"], last[s, "host"]
        tq = q[:, 0].astype(int)
        dt = (d["tracks"] - ht).abs().amax(-1).numpy()
        one_step = np.abs(np.arange(T)[None] - tq[:, None]) == 1
        results[s] = {
            "max_query_frame": tmax,
            "device": {"pairs_per_s": round(pairs * args.repeats / secs[s, "device"], 3),
                       "ms_per_step": round(secs[s, "device"] / args.repeats / args.steps * 1e3, 3),
                       "d2h_bytes": int(q.shape[0] * T * 9), "history_bytes": int(tmax * 12 * H * W)},
            "host_loop": {"pairs_per_s": round(pairs * args.repeats / secs[s, "host_loop"], 3),
                          "ms_per_step": round(secs[s, "host_loop"] / args.repeats / args.steps * 1e3, 3),
                          "d2h_bytes": int(host_bytes), "host_history_bytes": int(tmax * 12 * H * W)},
            "vs_host_loop": {"max_px_diff_one_step_from_query": float(dt[one_step].max()),
                             "max_px_diff": float(dt[np.isfinite(dt)].max()),
                             "visibility_differs_fraction": float((d["visible"].bool() != hv).float().mean()),
                             "visible_fraction": float(d["visible"].float().mean())}}

    # the two launches alone: the forward launch of one step (B pairs, N queries at frame 0) and the backward launch over
    # the spread set's history
    g = torch.Generator(device=dev).manual_seed(5)
    q0 = torch.from_numpy(sets["frame0"]).to(dev)
    qs = torch.from_numpy(sets["every5"]).to(dev)
    nq = q0.shape[0]
    hist = int(sets["every5"][:, 0].max())
    fl = torch.randn((max(B, hist), 2, H, W), device=dev, generator=g) * 2
    occ = (torch.rand((max(B, hist), H, W), device=dev, generator=g) < 0.1).float()
    tracks = torch.empty((nq, T, 2), device=dev)
    visible = torch.empty((nq, T), device=dev, dtype=torch.uint8)
    pos, vis = torch.empty((nq, 2), device=dev), torch.empty((nq,), device=dev, dtype=torch.uint8)
    fwd_ms = event_ms(lambda: ops.track_points_forward(fl[:B], occ[:B], 0, q0, pos, vis, tracks, visible),
                      args.kernel_launches)
    bwd_ms = event_ms(lambda: ops.track_points_backward(fl[:hist], occ[:hist], qs, tracks, visible), args.kernel_launches)

    res = {"metric": "pairs/s of query point tracks over consecutive video pairs @%dx%d %s, device chain vs host loop"
                     % (H, W, wl_name),
           "card": card, "device": torch.cuda.get_device_name(dev),
           "workload": "%s %dx%d, %d pairs per step, %d steps per clip (%d frames), %d queries per set (BASELINE "
                       "configs[%d])" % (wl_name, H, W, B, args.steps, T, args.queries, cfg_idx),
           "repeats": args.repeats, "cuda_graph": True, "data": "synthetic_video seed 77",
           "query_sets": results,
           "um_track_points_forward": {"ms": round(fwd_ms, 4), "pairs": B, "queries": nq,
                                       "share_of_device_step": round(fwd_ms / results["frame0"]["device"]["ms_per_step"],
                                                                     6)},
           "um_track_points_backward": {"ms": round(bwd_ms, 4), "pairs": hist, "queries": nq},
           "note": "launch times: CUDA events around each launch, mean of %d; bytes from shapes" % args.kernel_launches}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
