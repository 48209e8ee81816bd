#!/usr/bin/env python
"""Scoring a fused reconstruction against a denser reference surface, on one GPU.

    python tools/recon_eval_bench.py [--dims 294 217 258] [--voxel 0.01] [--repeats 5] [--kernel-iters 10]
                                     [--cdist-queries 20000]

The prediction is `mesh_bench`'s analytic room, `extract_points()` of its volume at `--voxel` (431,386 points at 1 cm),
plus 1 % floaters 5-50 cm off the surface along random directions.  The reference (GT) is the same room's
`extract_points()` at half the voxel size (a denser sampling of the same surface).  Arms, alternated for `--repeats`
rounds after a warm-up, each the median round:
  * `reconstruction_metrics` end to end (host clock around the call, which ends in its download), with
    `down_sample` 0.02 and None;
  * scipy `cKDTree(gt).query(pred, workers=-1)` and the reverse on the host after a download (no down-sampling);
  * a chunked exact `torch.cdist` (`compute_mode="donot_use_mm_for_euclid_dist"`) on the device, on the first
    `--cdist-queries` predicted points against the whole GT, reported per query and scaled to all queries.
Per kernel (CUDA events over `--kernel-iters` calls, down_sample None, pred queries against the GT table): keys, the
stable sort (torch), the table, the nearest search with partials, and the stats; with bytes and queries from shapes.
Checks that the GPU metrics (down_sample None) agree with the ones from cKDTree's float64 distances.  Reports the card,
power limit and clocks.  Prints ONE JSON line.  Writes nothing to the tree.
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from tools.common import card, timed  # noqa: E402
from tools.mesh_bench import build_volume  # noqa: E402


def _kernel_ms(fn, iters):
    fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def _host_metrics(d_pred, d_gt, t):
    import refops_recon as RR
    return RR.from_distances(d_pred, d_gt, np.float32(t))


@torch.no_grad()
def run(args):
    if not torch.cuda.is_available():
        raise SystemExit("recon_eval_bench: needs a CUDA device")
    from scipy.spatial import cKDTree
    from unimatch_b200.evaluation import reconstruction_metrics
    from unimatch_b200.fusion import _Table, _boxes
    dev = torch.device("cuda", 0)
    dims = tuple(args.dims)
    surface = build_volume(dims, args.voxel, dev).extract_points()[0]
    g = torch.Generator(device="cpu").manual_seed(0)
    nf = surface.shape[0] // 100
    pick = torch.randint(0, surface.shape[0], (nf,), generator=g)
    direction = torch.nn.functional.normalize(torch.randn(nf, 3, generator=g), dim=1)
    offset = 0.05 + 0.45 * torch.rand(nf, 1, generator=g)
    pred = torch.cat([surface, surface[pick] + (direction * offset).to(dev)]).contiguous()
    gt = build_volume(tuple(2 * d for d in dims), args.voxel / 2, dev).extract_points()[0]
    torch.cuda.empty_cache()
    torch.cuda.synchronize()

    arms = {"metrics_down_0.02": lambda: reconstruction_metrics(pred, gt, down_sample=0.02),
            "metrics_down_none": lambda: reconstruction_metrics(pred, gt, down_sample=None)}
    results = {k: f() for k, f in arms.items()}                        # warm-up
    pred_h, gt_h = pred.cpu().numpy(), gt.cpu().numpy()

    def kdtree():
        d_pred = cKDTree(gt_h.astype(np.float64)).query(pred_h.astype(np.float64), workers=-1)[0]
        d_gt = cKDTree(pred_h.astype(np.float64)).query(gt_h.astype(np.float64), workers=-1)[0]
        return d_pred, d_gt

    nq = min(args.cdist_queries, pred.shape[0])

    def cdist():
        best = []
        for a in range(0, nq, 1000):
            dmin = torch.full((min(1000, nq - a),), float("inf"), device=dev)
            for b in range(0, gt.shape[0], 200_000):
                d = torch.cdist(pred[a:a + 1000], gt[b:b + 200_000], compute_mode="donot_use_mm_for_euclid_dist")
                dmin = torch.minimum(dmin, d.min(1).values)
            best.append(dmin)
        out = torch.cat(best)
        torch.cuda.synchronize()
        return out

    kd = kdtree()
    cd = cdist()
    times = {k: [] for k in list(arms) + ["download_and_cKDTree", "cdist_subsample"]}
    for _ in range(args.repeats):
        for k, f in arms.items():
            torch.cuda.synchronize()
            times[k].append(1000 * timed(f)[0])
        times["download_and_cKDTree"].append(1000 * timed(lambda: (pred.cpu(), gt.cpu(), kdtree()))[0])
        times["cdist_subsample"].append(1000 * timed(cdist)[0])

    box_pred, box_gt = _boxes([pred, gt], "bench")
    table = _Table(gt, box_gt)
    ops = torch.ops.unimatch_sm100
    keys = ops.cloud_keys(gt, table.origin, table.cell, table.dims)
    skeys, order = torch.sort(keys, stable=True)
    psum, pcount = table.partials(pred, 0.05)
    out = torch.empty(2, dtype=torch.float64, device=dev)
    N, Q, C = gt.shape[0], pred.shape[0], int(np.prod(table.dims))
    k_ms = {"keys": _kernel_ms(lambda: ops.cloud_keys(gt, table.origin, table.cell, table.dims), args.kernel_iters),
            "stable_sort_torch": _kernel_ms(lambda: torch.sort(keys, stable=True), args.kernel_iters),
            "ranges": _kernel_ms(lambda: ops.cloud_ranges(skeys, order, gt, table.dims), args.kernel_iters),
            "nearest_partials": _kernel_ms(lambda: table.partials(pred, 0.05), args.kernel_iters),
            "stats": _kernel_ms(lambda: ops.cloud_stats(psum, pcount, out), args.kernel_iters)}
    nb = psum.shape[0]
    nbytes = {"keys": 12 * N + 8 * N, "stable_sort_torch": 32 * N, "ranges": 8 * N + 8 * N + 12 * N + 16 * N + 8 * C,
              "nearest_partials": 12 * Q + 16 * nb, "stats": 16 * nb}
    kernels = {k: {"ms": round(ms, 4), "bytes_from_shapes": nbytes[k]} for k, ms in k_ms.items()}
    kernels["nearest_partials"]["queries_per_s"] = round(Q / k_ms["nearest_partials"] * 1e3)

    host = _host_metrics(kd[0].astype(np.float32), kd[1].astype(np.float32), 0.05)
    gpu = results["metrics_down_none"]
    agree = {k: abs(gpu[k] - host[k]) / max(abs(host[k]), 1e-30) for k in ("acc", "comp", "chamfer", "prec", "recall")}
    gpu_d = table.nearest(pred[:nq])[0]
    cdist_rel = float(((gpu_d - cd).abs() / cd.clamp(min=1e-30)).max())
    med = {k: round(statistics.median(v), 3) for k, v in times.items()}
    print(json.dumps({
        "card": card(), "pred_points": Q, "gt_points": N, "floaters": nf, "gt_table_cells": C,
        "gt_table_dims": list(table.dims), "cell_m": table.cell, "repeats": args.repeats,
        "ms_median": med, "ms": {k: [round(x, 3) for x in v] for k, v in times.items()},
        "cdist_ms_per_query": round(med["cdist_subsample"] / nq, 6),
        "cdist_ms_scaled_to_all_queries_both_ways": round(med["cdist_subsample"] / nq * (Q + N), 1),
        "kernels_ms_per_call": kernels,
        "metrics_down_0.02": results["metrics_down_0.02"], "metrics_down_none": gpu,
        "max_rel_diff_vs_cKDTree_float64": max(agree.values()), "max_rel_diff_nearest_vs_cdist": cdist_rel,
        "time": time.strftime("%Y-%m-%d %H:%M:%S")}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dims", type=int, nargs=3, default=[294, 217, 258])
    ap.add_argument("--voxel", type=float, default=0.01)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--kernel-iters", type=int, default=10)
    ap.add_argument("--cdist-queries", type=int, default=20000)
    run(ap.parse_args())


if __name__ == "__main__":
    main()
