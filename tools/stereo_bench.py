#!/usr/bin/env python
"""Streaming stereo (StereoRunner) against today's host-side path on the same pairs, on one GPU.

    python tools/stereo_bench.py [--workload config3] [--model gmstereo-scale2|gmstereo-scale2-regrefine3] [--steps K]
                                 [--warmup W] [--pairs-per-step B]

The workload is bench.py's config3 (544x960, 16 pairs per step, bench weights); `--model` swaps the network.  Two steps
alternate in one process on the same B pairs:
  * runner step: what `unimatch_b200.StereoRunner` does per step with `visualize=True` -- the B uint8 pairs are copied from
    pinned memory, normalised and converted on the device, run forward and coloured (`disparity_to_image`), all replayed as
    one CUDA graph, and the disparity and the picture go back to pinned memory;
  * today's path: the pairs normalised on the host CPU (the stereo data pipeline's float32 ToTensor + Normalize) are
    uploaded as float32, run through `infer_stereo`, the disparity is copied back and coloured on the CPU by the oracle's
    `vis_disparity`.
Prints ONE JSON line: the device and its power limit, device ms per step and pairs/s of each path, the host CPU ms per step
that the runner removes (normalisation and colouring), H2D / D2H bytes per step, and the `disparity_to_image` kernel time with
its achieved bandwidth as a share of the H100 SXM data-sheet 3.35 TB/s.  Exits non-zero unless the two disparities are bit
for bit identical.  Writes nothing to the tree.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench import BENCH_WORKLOADS  # noqa: E402

HBM_DATASHEET_GBS = 3350.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="config3", choices=["config3"])
    ap.add_argument("--model", default=None, choices=["gmstereo-scale2", "gmstereo-scale2-regrefine3"],
                    help="network (default: the workload's)")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--pairs-per-step", type=int, default=0, help="B (default: the workload's pairs per GPU in bench.py)")
    run(ap.parse_args())


def _power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


@torch.no_grad()
def run(args):
    import refops_depth
    from oracle import disp_viz as OD
    from unimatch_b200 import UniMatch
    from unimatch_b200.inference import StereoRunner, disparity_to_image, infer_stereo
    from unimatch_b200.spec import WORKLOADS
    from unimatch_b200.synthetic import BENCH_WEIGHTS, IMAGENET_MEAN, IMAGENET_STD, synthetic_state_dict, synthetic_stereo_frames
    wl_name, H, W, ppg, cfg_idx, _, _ = BENCH_WORKLOADS[args.workload]
    name = args.model or wl_name
    cfg = WORKLOADS[name]
    B = args.pairs_per_step or ppg
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    model = UniMatch(**cfg["model"]).eval()
    model.load_state_dict(synthetic_state_dict(seed=326, **BENCH_WEIGHTS, **cfg["model"]), strict=True)
    model = model.to(dev)
    call = {k: v for k, v in cfg["call"].items() if k != "task"}
    pad = cfg["pad"]
    lefts, rights = synthetic_stereo_frames(B, H, W, seed=77)

    # runner step: the runner's own staging buffer, graph and pinned outputs, slot 0
    runner = StereoRunner(model, (H, W), B, dev, padding_factor=pad, visualize=True, **call)
    runner.pin[0][:B].copy_(lefts)
    runner.pin[0][B:].copy_(rights)
    runner._capture()
    static = runner.static_out[0]
    out_r = {k: torch.empty(v.shape, dtype=v.dtype).pin_memory() for k, v in static.items()}

    def runner_step():
        runner.dev_in[0].copy_(runner.pin[0], non_blocking=True)
        runner.graphs[0].replay()
        for k, v in static.items():
            out_r[k].copy_(v, non_blocking=True)

    # today's path: host normalisation, float32 upload, infer_stereo, disparity back, colouring on the CPU
    def host_normalise():
        return [refops_depth.normalize_frames(f, IMAGENET_MEAN, IMAGENET_STD).contiguous() for f in (lefts, rights)]

    pin_l, pin_r = (t.pin_memory() for t in host_normalise())
    out_t = torch.empty((B, H, W)).pin_memory()

    def today_step():
        a, b = pin_l.to(dev, non_blocking=True), pin_r.to(dev, non_blocking=True)
        out_t.copy_(infer_stereo(model, a, b, padding_factor=pad, **call)["disp"], non_blocking=True)

    for _ in range(max(args.warmup, 1)):
        runner_step(); today_step()
    torch.cuda.synchronize()
    identical = bool(torch.equal(out_r["disp"], out_t))
    max_diff = (out_r["disp"] - out_t).abs().max().item()
    vis_ok = bool(torch.equal(out_r["vis"], torch.from_numpy(OD.vis_disparity_batch(out_t.numpy()))))

    ev = [[torch.cuda.Event(enable_timing=True) for _ in range(2)] for _ in range(2)]
    tot = [0.0, 0.0]
    host = {"normalise": 0.0, "colour": 0.0}
    for _ in range(args.steps):
        for j, fn in enumerate((runner_step, today_step)):
            ev[j][0].record(); fn(); ev[j][1].record()
        torch.cuda.synchronize()
        for j in range(2):
            tot[j] += ev[j][0].elapsed_time(ev[j][1])
        t0 = time.perf_counter()
        host_normalise()
        t1 = time.perf_counter()
        OD.vis_disparity_batch(out_t.numpy())
        t2 = time.perf_counter()
        host["normalise"] += (t1 - t0) * 1e3
        host["colour"] += (t2 - t1) * 1e3
    ms_r, ms_t = tot[0] / args.steps, tot[1] / args.steps

    disp, pic = static["disp"], torch.empty((B, H, W, 3), dtype=torch.uint8, device=dev)
    for _ in range(5):
        disparity_to_image(disp, pic)
    k0, k1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 100
    k0.record()
    for _ in range(reps):
        disparity_to_image(disp, pic)
    k1.record()
    torch.cuda.synchronize()
    kms = k0.elapsed_time(k1) / reps
    kbytes = B * H * W * (4 + 4 + 3)
    hw = B * H * W
    res = {"metric": "pairs/s of %d stereo pairs @%dx%d %s per step: StereoRunner step (uint8 in, graph, disparity + picture "
                     "back) vs today's path (host-normalised float32 in, infer_stereo, disparity back, coloured on the CPU)"
                     % (B, H, W, name),
           "device": torch.cuda.get_device_name(dev), "power_limit": _power_limit(),
           "workload": "%s %dx%d, %d pairs per step (bench.py %s weights, BASELINE configs[%d])" % (name, H, W, B, args.workload,
                                                                                                    cfg_idx),
           "steps": args.steps, "warmup": max(args.warmup, 1), "data": "synthetic_stereo_frames seed 77",
           "runner": {"device_ms_per_step": round(ms_r, 3), "pairs_per_s": round(B / (ms_r / 1e3), 2), "cuda_graph": True,
                      "h2d_bytes_per_step": 2 * hw * 3, "d2h_bytes_per_step": hw * 4 + hw * 3},
           "today": {"device_ms_per_step": round(ms_t, 3), "pairs_per_s": round(B / (ms_t / 1e3), 2), "cuda_graph": False,
                     "h2d_bytes_per_step": 2 * hw * 3 * 4, "d2h_bytes_per_step": hw * 4,
                     "host_cpu_ms_per_step": {k: round(v / args.steps, 1) for k, v in host.items()},
                     "host_cores": os.cpu_count(), "torch_threads": torch.get_num_threads()},
           "host_cpu_ms_removed_per_step": round((host["normalise"] + host["colour"]) / args.steps, 1),
           "disparity_to_image": {"shape": [B, H, W], "ms": round(kms, 4), "bytes": kbytes,
                                  "achieved_GBps": round(kbytes / kms / 1e6, 1),
                                  "share_of_datasheet_3.35TBps": round(kbytes / kms / 1e6 / HBM_DATASHEET_GBS, 3)},
           "disp_bit_identical": identical, "max_abs_disp_diff": max_diff, "vis_equals_oracle": vis_ok}
    print(json.dumps(res))
    if not (identical and vis_ok):
        sys.exit(1)


if __name__ == "__main__":
    main()
