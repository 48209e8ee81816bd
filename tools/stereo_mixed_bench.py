#!/usr/bin/env python
"""Mixed-size stereo streaming (MixedSizeStereoRunner) against today's options on a KITTI-like stream, on one GPU.

    python tools/stereo_mixed_bench.py [--model gmstereo-scale2|gmstereo-scale2-regrefine3] [--pairs N] [--batch B]
                                       [--check K]

The stream interleaves 375x1242, 370x1226, 374x1238 and 376x1241 uint8 pairs (KITTI's four frame sizes, synthetic
content, bench weights).  It runs in two modes: `inference_size=(352, 1216)` (the reference's KITTI submission setting) and
padding 32 without it (the stereo workloads' padding: every size rounds up to 384x1248).  Both give one model shape for
these four sizes; padding 16 would send the 1226-wide frames to 384x1232, whose 1/4-resolution width (308) the 8-way swin
split of these networks does not divide, so no stereo workload here can run at that shape.  Three paths, in one process:
  1. mixed: one `MixedSizeStereoRunner` (`visualize=True`) over the whole stream;
  2. per_size: one `StereoRunner` per exact frame size (`visualize=True`), each over its own pairs -- the best the
     streaming API offered before;
  3. per_pair: the reference's loop -- one pair per call, normalised on the host, uploaded as float32, `infer_stereo` at
     batch 1, the disparity coloured on the CPU by the oracle's `vis_disparity`.
Each path runs the stream twice; the first pass includes the CUDA-graph captures (`cold_s`), the second is `wall_s`:
host clock around the whole stream, ending in a device synchronise.  Prints ONE JSON line per call: the device and its
power limit, per mode and path the wall time and pairs/s, steps and mean step fill, H2D / D2H bytes, the mixed runner's
first-step latency per bucket (capture included), and the largest disparity difference between paths 1 and 2 relative to
the largest disparity.  Exits non-zero unless path 1 equals, bit for bit, the composed reference of the GPU tests
(tests/refops_ragged.py) on `--check` sampled pairs of each mode.  Writes nothing to the tree.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from tools.common import card, timed  # noqa: E402

KITTI_SIZES = [(375, 1242), (370, 1226), (374, 1238), (376, 1241)]
MODES = {"inference_size": dict(padding_factor=32, inference_size=(352, 1216)),
         "padding32": dict(padding_factor=32, inference_size=None)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="gmstereo-scale2", choices=["gmstereo-scale2", "gmstereo-scale2-regrefine3"])
    ap.add_argument("--pairs", type=int, default=48)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--check", type=int, default=4, help="sampled pairs per mode compared with the composed reference")
    run(ap.parse_args())


@torch.no_grad()
def run(args):
    import refops_depth
    import refops_ragged
    from oracle import disp_viz as OD
    from unimatch_b200 import MixedSizeStereoRunner, StereoRunner
    from unimatch_b200.inference import infer_stereo
    from unimatch_b200.synthetic import IMAGENET_MEAN, IMAGENET_STD, synthetic_model, synthetic_stereo_frames, workload_call

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    model = synthetic_model(args.model, dev)
    call = workload_call(args.model, drop=("task",))
    B, N = args.batch, args.pairs
    sizes = [KITTI_SIZES[i % len(KITTI_SIZES)] for i in range(N)]
    frames = {s: synthetic_stereo_frames(1, s[0], s[1], seed=90 + k) for k, s in enumerate(KITTI_SIZES)}
    pairs = []
    for i, s in enumerate(sizes):                      # distinct content per pair: roll the size's frames by the index
        left, right = frames[s]
        pairs.append((torch.roll(left[0], 7 * i, 1).numpy(), torch.roll(right[0], 7 * i, 1).numpy()))
    cap = (max(h for h, _ in KITTI_SIZES), max(w for _, w in KITTI_SIZES))
    rng = np.random.default_rng(5)
    checked_ok = True
    res = {"metric": "pairs/s of a KITTI-like mixed-size stereo stream (%d pairs of 4 sizes, %s, batch %d): "
                     "MixedSizeStereoRunner vs one StereoRunner per size vs the per-pair host loop" % (N, args.model, B),
           "device": torch.cuda.get_device_name(dev), "power_limit": card()["power_limit"], "pairs": N, "batch": B,
           "sizes": [list(s) for s in KITTI_SIZES], "model": args.model, "modes": {}}

    for mode, geo in MODES.items():
        first_step = {}

        class Timed(MixedSizeStereoRunner):
            def _device_step(self, slot, chunk):
                size = self.meta[slot]["size"]
                if not self.use_graph or size in self.buckets or size in first_step:
                    return super()._device_step(slot, chunk)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                out = super()._device_step(slot, chunk)
                torch.cuda.synchronize()
                first_step[size] = time.perf_counter() - t0
                return out

        mixed = Timed(model, cap, B, dev, visualize=True, **geo, **call)

        def mixed_pass():
            return {i: {k: v.clone() for k, v in r.items()} for i, r in mixed.run(pairs)}

        cold_m, _ = timed(mixed_pass)
        s0 = dict(mixed.stats)
        wall_m, got_m = timed(mixed_pass)
        st = {k: mixed.stats[k] - s0[k] for k in mixed.stats}

        groups = {s: [i for i in range(N) if sizes[i] == s] for s in KITTI_SIZES}
        pool = {s: StereoRunner(model, s, B, dev, visualize=True, **geo, **call) for s in KITTI_SIZES}

        def pool_pass():
            out = {}
            for s, idx in groups.items():
                for i, r in zip(idx, pool[s].run([pairs[i] for i in idx])):
                    out[i] = {k: v.clone() for k, v in r.items()}
            return out

        cold_p, _ = timed(pool_pass)
        wall_p, got_p = timed(pool_pass)
        pool_steps = sum(-(-len(idx) // B) for idx in groups.values())
        pool_h2d = sum(-(-len(groups[s]) // B) * 2 * B * s[0] * s[1] * 3 for s in KITTI_SIZES)
        pool_d2h = sum(-(-len(groups[s]) // B) * B * s[0] * s[1] * 7 for s in KITTI_SIZES)

        def loop_pass():
            out = {}
            for i, (left, right) in enumerate(pairs):
                nl, nr = (refops_depth.normalize_frames(torch.from_numpy(f)[None], IMAGENET_MEAN, IMAGENET_STD).to(dev)
                          for f in (left, right))
                d = infer_stereo(model, nl, nr, **geo, **call)["disp"][0].cpu()
                out[i] = {"disp": d, "vis": torch.from_numpy(OD.vis_disparity(d.numpy()))}
            return out

        cold_l, _ = timed(loop_pass)
        wall_l, _ = timed(loop_pass)
        loop_h2d = sum(2 * 3 * h * w * 4 for h, w in sizes)
        loop_d2h = sum(4 * h * w for h, w in sizes)

        dmax = max(got_p[i]["disp"].abs().max().item() for i in range(N))
        ddiff = max((got_m[i]["disp"] - got_p[i]["disp"]).abs().max().item() for i in range(N))
        sample = set(int(i) for i in rng.choice(N, size=min(args.check, N), replace=False))
        ref = refops_ragged.composed_stereo_reference(model, call, pairs, B, mixed.max_buckets, only=sample, **geo)
        identical = all(torch.equal(got_m[i][k], ref[i][k]) for i in sample for k in ("disp", "vis"))
        checked_ok &= identical

        def path(wall, cold, steps, h2d, d2h, graphs):
            return {"wall_s": round(wall, 4), "cold_s": round(cold, 4), "pairs_per_s": round(N / wall, 2), "steps": steps,
                    "mean_step_fill": round(N / (steps * (B if graphs else 1)), 3), "h2d_bytes": h2d, "d2h_bytes": d2h,
                    "cuda_graph": graphs}

        res["modes"][mode] = {
            "geometry": {k: (list(v) if isinstance(v, tuple) else v) for k, v in geo.items()},
            "buckets": sorted([list(b) for b in mixed.buckets]),
            "mixed": dict(path(wall_m, cold_m, st["steps"], st["h2d_bytes"], st["d2h_bytes"], True),
                          first_step_s_per_bucket={"%dx%d" % b: round(t, 4) for b, t in first_step.items()},
                          captures=mixed.stats["captures"]),
            "per_size": path(wall_p, cold_p, pool_steps, pool_h2d, pool_d2h, True),
            "per_pair": path(wall_l, cold_l, N, loop_h2d, loop_d2h, False),
            "max_disp_diff_mixed_vs_per_size_rel": ddiff / dmax if dmax else 0.0,
            "checked_pairs": sorted(sample), "equals_composed_reference": identical,
        }
        del mixed, pool
        torch.cuda.empty_cache()
    print(json.dumps(res))
    if not checked_ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
