#!/usr/bin/env python
"""Mixed-size flow streaming (MixedSizeFlowRunner) against today's options on an interleaved stream, on one GPU.

    python tools/flow_mixed_bench.py [--models gmflow-scale2-regrefine6,gmflow-scale1] [--pairs N] [--batch B] [--reps R]
                                     [--kernel-launches L]

The seeded stream interleaves uint8 pairs at KITTI's four frame sizes (375x1242, 370x1226, 374x1238, 376x1241), Sintel's
436x1024 and a portrait 832x480 (synthetic content, bench weights, padding 32: three inference sizes, 384x1248, 448x1024
and 480x832).  Per model and with pictures on and off, three arms alternate, `--reps` times each, in one process:
  1. mixed: one `MixedSizeFlowRunner` over the whole stream;
  2. per_pair: the host loop of `inference_flow` around the same module -- one pair per call, converted to float32 on the
     host, uploaded, `infer_flow` at batch 1, the flow copied back and coloured on the CPU by the oracle's `flow_to_image`;
  3. per_size: one `BatchedFlowRunner` per exact frame size, fed float32 tensors, each over its own pairs.  It pads where
     the others resize and does not transpose portrait pairs, so its flows are another computation: a throughput arm only.
     It cannot paint; with pictures on its flows are coloured on the CPU like arm 2's.
Every repetition builds an arm, runs the stream once (all buckets captured and warm; that first pass is reported as
`cold_s`), times a second pass (`wall_s`) and frees the arm: at batch 8 the CUDA graphs of the mixed runner and of the
per-size pool do not fit one 80 GB card together.  A timing is a host clock around the whole stream, ending in a device
synchronise; all repetitions are printed.
Then the four ragged kernels are timed alone with CUDA events over `--kernel-launches` launches on a full KITTI step, with
the bytes they must move (from shapes) over that time: they are bandwidth-bound, so GB/s is the figure to read.
Prints ONE JSON line with the device name and power limit.  Fails without a CUDA device.  Writes nothing to the tree.
"""
import argparse
import gc
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from tools.common import card, timed  # noqa: E402

KITTI_SIZES = [(375, 1242), (370, 1226), (374, 1238), (376, 1241)]
SIZES = KITTI_SIZES + [(436, 1024), (832, 480)]
CAP = (832, 1242)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="gmflow-scale2-regrefine6,gmflow-scale1")
    ap.add_argument("--pairs", type=int, default=48)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--kernel-launches", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("flow_mixed_bench needs a CUDA device: nothing is measured without one")
    run(args)


def _stream(n, seed=17):
    """n pairs at seeded sizes from SIZES, distinct content per pair (one synthetic clip per size, rolled by the index)"""
    from unimatch_b200.synthetic import synthetic_video
    rng = np.random.default_rng(seed)
    sizes = [SIZES[int(k)] for k in rng.integers(0, len(SIZES), size=n)]
    clips = {s: synthetic_video(2, s[0], s[1], seed=90 + k) for k, s in enumerate(SIZES)}
    return sizes, [tuple(torch.roll(f, 7 * i, 1).numpy() for f in clips[s]) for i, s in enumerate(sizes)]


def _kernel_times(batch, launches, dev):
    """ms per launch of the four ragged kernels on a full step of KITTI pairs at 384x1248, and the bytes each must move"""
    from unimatch_b200 import ops
    from unimatch_b200.inference import _flow_step_layout
    _OPS = torch.ops.unimatch_sm100
    size = (384, 1248)
    sizes = [KITTI_SIZES[i % 4] for i in range(batch)]
    frames, planes, flows, pictures, masks, nbytes, used, _ = _flow_step_layout(sizes, batch, size, True, True)

    def table(t):
        return torch.from_numpy(t.view(np.uint8).reshape(-1, ops.RAGGED_ITEM_BYTES)).to(dev)

    frames, planes, flows, pictures, masks = (table(t) for t in (frames, planes, flows, pictures, masks))
    g = torch.Generator().manual_seed(1)
    packed_frames = torch.randint(0, 256, (nbytes,), generator=g, dtype=torch.uint8).to(dev)
    model_flow = (torch.randn((4 * batch, 1) + size, generator=g) * 20).to(dev)
    cap = CAP[0] * CAP[1]
    packed = _OPS.resize_bilinear_ragged(model_flow, planes, CAP[0], CAP[1], 4 * batch * cap)
    occ = torch.empty((2 * batch * cap,), device=dev)
    pics = torch.empty((6 * batch * cap,), dtype=torch.uint8, device=dev)
    pix = sum(h * w for h, w in sizes)
    calls = {
        "um_frames_to_planar_ragged": (lambda: _OPS.frames_to_planar_ragged(packed_frames, frames, CAP[0], CAP[1], *size),
                                       nbytes + 2 * batch * 3 * size[0] * size[1] * 4),
        "um_resize_bilinear_ragged": (lambda: _OPS.resize_bilinear_ragged(model_flow, planes, CAP[0], CAP[1], 4 * batch * cap),
                                      model_flow.numel() * 4 + 4 * pix * 4),
        "um_fb_consistency_ragged": (lambda: _OPS.fb_consistency_ragged(packed, flows, occ, masks, CAP[0], CAP[1], 0.01, 0.5),
                                     4 * pix * 4 + 2 * pix * 4),
        "um_flow_to_image_ragged": (lambda: _OPS.flow_to_image_ragged(packed, flows, pics, pictures, CAP[0], CAP[1]),
                                    2 * 4 * pix * 4 + 2 * pix * 3),          # the flows are read twice: maximum, then colours
    }
    out = {}
    for name, (fn, nbytes_moved) in calls.items():
        for _ in range(10):
            fn()
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        start.record()
        for _ in range(launches):
            fn()
        end.record()
        torch.cuda.synchronize()
        ms = start.elapsed_time(end) / launches
        out[name] = {"ms_per_call": round(ms, 4), "bytes_per_call": nbytes_moved, "GB_per_s": round(nbytes_moved / ms / 1e6, 1),
                     "launches": launches}
    return out


@torch.no_grad()
def run(args):
    from oracle import flow_viz as OV
    from unimatch_b200 import BatchedFlowRunner, MixedSizeFlowRunner, infer_flow
    from unimatch_b200.synthetic import synthetic_model, workload_call

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B, N = args.batch, args.pairs
    sizes, pairs = _stream(N)
    floats = [tuple(torch.from_numpy(f).permute(2, 0, 1).float() for f in p) for p in pairs]     # arm 3's input format
    res = {"metric": "pairs/s of an interleaved mixed-size flow stream (%d pairs of %d sizes, batch %d, padding 32): "
                     "MixedSizeFlowRunner vs the per-pair host loop vs one BatchedFlowRunner per size" % (N, len(SIZES), B),
           "device": torch.cuda.get_device_name(dev), "power_limit": card()["power_limit"], "pairs": N, "batch": B,
           "sizes": [list(s) for s in SIZES], "runs": {}}

    for name in args.models.split(","):
        model = synthetic_model(name, dev)
        call = workload_call(name, drop=("task",))
        groups = {s: [i for i in range(N) if sizes[i] == s] for s in SIZES if s in sizes}
        for pictures in (True, False):
            stats = {}

            def make_mixed():
                mixed = MixedSizeFlowRunner(model, CAP, B, dev, padding_factor=32, visualize=pictures, **call)
                stats["mixed"] = mixed
                return lambda: sum(1 for _ in mixed.run(pairs))

            def make_loop():
                def loop_pass():
                    for a, b in pairs:
                        a, b = (torch.from_numpy(f).permute(2, 0, 1)[None].float().to(dev) for f in (a, b))
                        flow = infer_flow(model, a, b, padding_factor=32, **call)["flow"][0].cpu()
                        if pictures:
                            OV.flow_to_image(flow.permute(1, 2, 0).numpy())
                return loop_pass

            def make_pool():
                pool = {s: BatchedFlowRunner(model, s, B, dev, padding_factor=32, **call) for s in groups}

                def pool_pass():
                    for s, runner in pool.items():
                        for flow in runner.run([floats[i] for i in groups[s]]):
                            if pictures:
                                OV.flow_to_image(flow.permute(1, 2, 0).numpy())
                return pool_pass

            # the graphs of one arm (two per inference size, or two per frame size) take tens of GB at batch 8, and those of
            # the mixed runner and the per-size pool do not fit one 80 GB card together: every repetition builds an arm,
            # runs its first pass (captures included, `cold_s`), times its second pass (`wall_s`) and frees it
            arms = {"mixed": make_mixed, "per_pair": make_loop, "per_size": make_pool}
            cold, walls = {k: [] for k in arms}, {k: [] for k in arms}
            for _ in range(args.reps):
                for k, make in arms.items():
                    fn = make()
                    cold[k].append(timed(fn)[0])
                    if k == "mixed":
                        s0 = dict(stats["mixed"].stats)
                    walls[k].append(timed(fn)[0])
                    if k == "mixed":
                        mixed = stats.pop("mixed")
                        st = {key: mixed.stats[key] - s0[key] for key in mixed.stats}
                        buckets, captures = sorted([list(b) for b in mixed.buckets]), mixed.stats["captures"]
                        del mixed
                    del fn
                    gc.collect()
                    torch.cuda.empty_cache()
            pool_steps = sum(-(-len(idx) // B) for idx in groups.values())

            def arm(k, steps, per_step, h2d, d2h):
                return {"wall_s": [round(t, 4) for t in walls[k]], "cold_s": [round(t, 4) for t in cold[k]],
                        "pairs_per_s_best": round(N / min(walls[k]), 2), "pairs_per_s_worst": round(N / max(walls[k]), 2),
                        "steps": steps, "mean_step_fill": round(N / (steps * per_step), 3), "h2d_bytes": h2d, "d2h_bytes": d2h}

            pix = sum(h * w for h, w in sizes)
            pad = {s: (-(-s[0] // 32) * 32) * (-(-s[1] // 32) * 32) for s in groups}
            pool_px = sum(-(-len(groups[s]) // B) * B * pad[s] for s in groups)
            res["runs"]["%s/%s" % (name, "pictures" if pictures else "flow_only")] = {
                "buckets": buckets, "captures": captures,
                "mixed": arm("mixed", st["steps"], B, st["h2d_bytes"], st["d2h_bytes"]),
                "per_pair": arm("per_pair", N, 1, 2 * 3 * 4 * pix, 2 * 4 * pix),
                "per_size": arm("per_size", pool_steps, B, 2 * 3 * 4 * pool_px, 2 * 4 * pool_px),
            }
        del model
    res["kernels"] = _kernel_times(B, args.kernel_launches, dev)
    res["kernels_note"] = ("full step of %d KITTI pairs at 384x1248, bidirectional; bytes are what the kernel must read and "
                           "write, computed from shapes; these kernels are bandwidth-bound" % B)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
