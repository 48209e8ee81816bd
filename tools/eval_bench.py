#!/usr/bin/env python
"""Validation throughput: the reference's per-sample `--eval` loop against the batched drivers, on one GPU.

    python tools/eval_bench.py --protocol sintel|kitti|kitti15|scannet [--samples N] [--batch B]

Workload: a seeded synthetic dataset at the protocol's real size (Sintel 436x1024; KITTI and KITTI15 375x1242 plus one sample
in three at 370x1226, so that the shape grouping has two open batches; ScanNet 480x640) run by the bench configurations
gmflow-scale2-regrefine6, gmstereo-scale2 and gmdepth-scale1-regrefine1 with `synthetic_state_dict(**BENCH_WEIGHTS)`.
Timed, after one untimed pass of each (module caches, allocator):
  * per-sample: the reference loop restated around this module (tests/refloop_eval.py) -- one sample per `model(...)` call,
    the metrics in torch / numpy as the reference computes them, the prediction copied to the host where the reference does;
  * batched: `validate_flow` / `validate_stereo` / `validate_depth` at batch B.
Prints the card, its power limit and SM clocks (query-only nvidia-smi) and ONE JSON line with samples/s of both and the largest
difference between their results; exits non-zero beyond 1e-4 relative on sums or 1e-3 absolute on ratios (batch composition
changes the convolutions' summation order).  Writes nothing to the tree.
"""
import argparse
import json
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True

from tools.common import card, timed  # noqa: E402
from unimatch_b200 import evaluation  # noqa: E402
from unimatch_b200.spec import WORKLOADS  # noqa: E402
from unimatch_b200.synthetic import IMAGENET_MEAN, IMAGENET_STD, synthetic_model, workload_call  # noqa: E402

PROTOCOLS = {  # protocol -> (task, workload, shapes, padding factor, driver options)
    "sintel": ("flow", "gmflow-scale2-regrefine6", [(436, 1024)], 32, dict(protocol="sintel", with_speed_metric=True)),
    "kitti": ("flow", "gmflow-scale2-regrefine6", [(375, 1242), (375, 1242), (370, 1226)], 32, dict(protocol="kitti")),
    "kitti15": ("stereo", "gmstereo-scale2", [(375, 1242), (375, 1242), (370, 1226)], 32, dict(protocol="kitti15")),
    "scannet": ("depth", "gmdepth-scale1-regrefine1", [(480, 640)], 16, dict(protocol="scannet")),
}


def dataset(task, shapes, n, seed=0):
    g = torch.Generator().manual_seed(seed)
    mean, std = torch.tensor(IMAGENET_MEAN).view(3, 1, 1), torch.tensor(IMAGENET_STD).view(3, 1, 1)
    out = []
    for i in range(n):
        h, w = shapes[i % len(shapes)]
        a, b = (torch.rand((3, h, w), generator=g) * 255 for _ in range(2))
        valid = (torch.rand((h, w), generator=g) < 0.5).float()
        if task == "flow":
            out.append((a, b, torch.randn((2, h, w), generator=g) * 10, valid))
        elif task == "stereo":
            out.append({"left": (a / 255 - mean) / std, "right": (b / 255 - mean) / std,
                        "disp": torch.rand((h, w), generator=g) * 64 * (valid > 0)})
        else:
            K = torch.tensor([[0.9 * w, 0.0, w / 2.0], [0.0, 0.9 * w, h / 2.0], [0.0, 0.0, 1.0]])
            pose = torch.eye(4)
            pose[0, 3] = 0.1
            out.append({"img_ref": (a / 255 - mean) / std, "img_tgt": (b / 255 - mean) / std, "intrinsics": K, "pose": pose,
                        "depth": 0.3 + torch.rand((h, w), generator=g) * 10, "valid": valid})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--protocol", required=True, choices=sorted(PROTOCOLS))
    ap.add_argument("--samples", type=int, default=24)
    ap.add_argument("--batch", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("eval_bench needs a CUDA device")
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import refloop_eval
    task, workload, shapes, pad, opts = PROTOCOLS[args.protocol]
    model = synthetic_model(workload)
    kw = workload_call(workload, drop=("min_depth", "max_depth"))
    driver = {"flow": evaluation.validate_flow, "stereo": evaluation.validate_stereo, "depth": evaluation.validate_depth}[task]
    data = dataset(task, shapes, args.samples)
    warm = data[:len(shapes)]

    def loop(d):
        return refloop_eval.LOOPS[task](model, d, padding_factor=pad, **opts, **kw)

    def batched(d):
        return driver(model, d, batch=args.batch, padding_factor=pad, **opts, **kw)

    gpu = ", ".join(card().values())
    print("card:", gpu, flush=True)
    times, results = {}, {}
    for name, fn in (("per_sample", loop), ("batched", batched)):
        fn(warm)
        times[name], results[name] = timed(lambda: fn(data))
    want, got = results["per_sample"], results["batched"]
    worst_sum = worst_ratio = 0.0
    for k, v in want.items():
        d = abs(got[k] - v)
        if k.endswith(("_1px", "_2px", "_3px", "_5px", "_d1", "_f1", "a1", "a2", "a3")):
            worst_ratio = max(worst_ratio, d)
        else:
            worst_sum = max(worst_sum, d / max(abs(v), 1e-30))
    res = dict(protocol=args.protocol, workload=workload, samples=args.samples, batch=args.batch,
               per_sample_samples_per_s=args.samples / times["per_sample"], batched_samples_per_s=args.samples / times["batched"],
               speedup=times["per_sample"] / times["batched"], max_rel_diff_sums=worst_sum, max_abs_diff_ratios=worst_ratio,
               results=got, card=gpu)
    print(json.dumps(res))
    if not (worst_sum <= 1e-4 and worst_ratio <= 1e-3) or any(math.isnan(v) for v in got.values()):
        sys.exit("batched results disagree with the per-sample loop")


if __name__ == "__main__":
    main()
