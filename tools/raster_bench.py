#!/usr/bin/env python
"""Rasterising a reconstructed mesh at the fusion bench's shape, on one GPU.

    python tools/raster_bench.py [--dims 294 217 258] [--voxel 0.01] [--views 8] [--size 480 640] [--repeats 5]
                                 [--kernel-iters 20] [--crop 24] [--bench-steps 5] [--bench-warmup 3]

The mesh is `tools/mesh_bench.build_volume`'s analytic room with five objects, meshed with `extract_mesh`; the cameras
are `tools/render_bench.cameras` (inside the room, facing outwards, fx = fy = 0.78 W).  Arms, alternated for `--repeats`
rounds after a warm-up, each the median round (CUDA events):
  * `render_mesh()` end to end (mesh already on the device; the pose upload and the host read of the entry count
    included), with vertex colours;
  * what a user writes today in torch ops: each face's projected pixel box (vertices in front of the camera only),
    enumerated in chunks of faces, a ray-plane depth per covered pixel and a barycentric inside test, and a z-buffer by
    `scatter_reduce('amin')` on packed (depth bits << 32 | face) keys; depth and face only;
  * the numpy statement (tests/refops_raster.py, float32 kernel order) on a `--crop` x `--crop` crop of the first view,
    over the faces whose rectangles reach the crop, reported as host time per pixel.
Also: per-kernel times from CUDA events over `--kernel-iters` back-to-back launches (bin count + scan, bin, the torch
stable sort, ranges, raster) and the tile entries per face; `TSDFVolume.render` on the source volume and the quantiles
of |depth difference| between the two renderings where both hit; `visible_points` of the mesh's vertices and
`depth_metrics` of the mesh depths against the ray-cast depths on the same 8 frames; the peak device memory above the
mesh; whether the kernel equals the statement bit for bit on the crop; registers and spills of every new kernel (from
`cuobjdump --dump-resource-usage` of the built library, when the tool is on the PATH); the card's name, power limit and
SM clocks, read in the same run; and the JSON line of `bench.py --gpus 1 --steps K --warmup W`, run in the same
session.  Prints ONE JSON line.  Writes nothing to the tree.
"""
import argparse
import json
import os
import re
import shutil
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from tools.common import card, timed  # noqa: E402
from tools.mesh_bench import _event_ms, _kernel_ms, build_volume  # noqa: E402
from tools.render_bench import cameras  # noqa: E402

NEW_KERNELS = ("mesh_bin_count_kernel", "offsets_scan_kernel", "mesh_bin_kernel", "mesh_ranges_kernel", "mesh_raster_kernel",
               "visible_points_kernel", "depth_metrics_kernel", "depth_metrics_sum_kernel")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dims", type=int, nargs=3, default=[294, 217, 258])
    ap.add_argument("--voxel", type=float, default=0.01)
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--size", type=int, nargs=2, default=[480, 640])
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--kernel-iters", type=int, default=20)
    ap.add_argument("--crop", type=int, default=24)
    ap.add_argument("--bench-steps", type=int, default=5)
    ap.add_argument("--bench-warmup", type=int, default=3)
    run(ap.parse_args())


def torch_zbuffer(points, faces, K, poses, h, w, near=0.01, chunk=1 << 16):
    """The torch-ops z-buffer a user writes today: depth [n, h, w] (0: miss) and face [n, h, w] (-1: miss)"""
    dev = points.device
    fx, fy, cx, cy = (float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]))
    f64 = faces.long()
    depth, face = [], []
    for P in poses:
        M = torch.from_numpy(np.linalg.inv(P.astype(np.float64))[:3].astype(np.float32)).to(dev)
        V = points @ M[:, :3].T + M[:, 3]
        key = torch.full((h * w,), torch.iinfo(torch.int64).max, dtype=torch.int64, device=dev)
        for f0 in range(0, faces.shape[0], chunk):
            tri = V[f64[f0:f0 + chunk]]                                            # [m, 3, 3]
            front = (tri[..., 2] > near).all(1)
            tri, ids = tri[front], torch.arange(f0, f0 + min(chunk, faces.shape[0] - f0), device=dev)[front]
            u = fx * tri[..., 0] / tri[..., 2] + cx
            v = fy * tri[..., 1] / tri[..., 2] + cy
            x0, x1 = u.amin(1).floor().clamp(0, w - 1).long(), u.amax(1).ceil().clamp(0, w - 1).long()
            y0, y1 = v.amin(1).floor().clamp(0, h - 1).long(), v.amax(1).ceil().clamp(0, h - 1).long()
            bw, bh = x1 - x0 + 1, y1 - y0 + 1
            cnt = bw * bh
            rep = torch.repeat_interleave(torch.arange(len(cnt), device=dev), cnt)
            k = torch.arange(int(cnt.sum()), device=dev) - torch.repeat_interleave(torch.cumsum(cnt, 0) - cnt, cnt)
            px, py = x0[rep] + k % bw[rep], y0[rep] + k // bw[rep]
            d = torch.stack([(px.float() - cx) / fx, (py.float() - cy) / fy, torch.ones_like(px, dtype=torch.float32)], -1)
            A, B, C = tri[rep, 0], tri[rep, 1], tri[rep, 2]
            nrm = torch.cross(B - A, C - A, dim=-1)
            t = (A * nrm).sum(-1) / (d * nrm).sum(-1)
            X = d * t[:, None]
            e0 = (torch.cross(B - A, X - A, dim=-1) * nrm).sum(-1)
            e1 = (torch.cross(C - B, X - B, dim=-1) * nrm).sum(-1)
            e2 = (torch.cross(A - C, X - C, dim=-1) * nrm).sum(-1)
            ok = (e0 >= 0) & (e1 >= 0) & (e2 >= 0) & (t >= near) & torch.isfinite(t)
            packed = (t[ok].contiguous().view(torch.int32).long() << 32) | ids[rep[ok]]
            key.scatter_reduce_(0, (py * w + px)[ok], packed, "amin")
        hit = key != torch.iinfo(torch.int64).max
        depth.append(torch.where(hit, (key >> 32).int().view(torch.float32), torch.zeros((), device=dev)).view(h, w))
        face.append(torch.where(hit, (key & 0xffffffff).int(), torch.full((), -1, device=dev, dtype=torch.int32)).view(h, w))
    return torch.stack(depth), torch.stack(face)


def _resource_usage():
    """{kernel: {registers, stack, spills}} of the new kernels, from cuobjdump on the built library"""
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    lib = os.path.join(ROOT, "unimatch_b200", "libunimatch_sm100.so")
    try:
        txt = subprocess.run([tool, "--dump-resource-usage", lib], capture_output=True, text=True, timeout=120).stdout
    except (OSError, subprocess.SubprocessError):
        return "not available"
    out, name = {}, None
    for ln in txt.splitlines():
        m = re.search(r"Function ([\w$]+):", ln)
        if m:
            name = next((k for k in NEW_KERNELS if k in m.group(1)), None)
        elif name and "REG:" in ln:
            reg = re.search(r"REG:(\d+)", ln)
            stack = re.search(r"STACK:(\d+)", ln)
            local = re.search(r"LOCAL:(\d+)", ln)
            out[name] = {"registers": int(reg.group(1)), "stack": int(stack.group(1)) if stack else None,
                         "local_bytes": int(local.group(1)) if local else None}
            name = None
    return out or "not available"


@torch.no_grad()
def run(args):
    if not torch.cuda.is_available():
        raise SystemExit("raster_bench: needs a CUDA device")
    import refops_raster as RS
    from unimatch_b200.evaluation import depth_metrics
    from unimatch_b200.fusion import render_mesh, visible_points
    from unimatch_b200.inference import _world_to_camera
    ops = torch.ops.unimatch_sm100
    dev = torch.device("cuda", 0)
    vol = build_volume(tuple(args.dims), args.voxel, dev)
    points, colors, _, faces = vol.extract_mesh()
    torch.cuda.synchronize()
    h, w = args.size
    extent = [n * vol.voxel_size for n in vol.dims]
    K, poses = cameras(extent, args.views, h, w)
    T = int(faces.shape[0])

    def peak(fn):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated(dev)
        torch.cuda.reset_peak_memory_stats(dev)
        out = fn()
        torch.cuda.synchronize()
        return out, torch.cuda.max_memory_allocated(dev) - base

    out, peak_render = peak(lambda: render_mesh(points, faces, K, poses, (h, w), colors=colors))
    (zd, zf), peak_torch = peak(lambda: torch_zbuffer(points, faces, K, poses, h, w))
    hits = out["face"] >= 0
    both = hits & (zf >= 0)
    zb_agree = {"same_face_share": round(float((out["face"] == zf)[both].float().mean()), 4),
                "median_abs_depth_difference_m": float((out["depth"] - zd).abs()[both].median())}

    ray = vol.render(K, poses, (h, w))
    both = hits & (ray["depth"] > 0)
    diff = (out["depth"] - ray["depth"]).abs()[both]
    qs = torch.quantile(diff[torch.randperm(diff.numel(), device=dev)[:1 << 20]].double(),
                        torch.tensor([0.5, 0.9, 0.99, 1.0], device=dev, dtype=torch.float64)).tolist()

    c = args.crop
    y0, x0 = (h - c) // 2, (w - c) // 2
    Kc = K.copy()
    Kc[0, 2] -= x0
    Kc[1, 2] -= y0
    pts_h, tri_h, col_h = points.cpu().numpy(), faces.cpu().numpy(), colors.cpu().numpy()
    w2c = _world_to_camera(poses)
    rx0, rx1, ry0, ry1, ok = RS.rectangles(pts_h, tri_h, w2c[0], Kc, c, c, 0.01)
    sub = np.nonzero(ok)[0]                        # only these faces can reach the crop; the rest never win there

    def statement():
        d, f, col = RS.raster(pts_h, tri_h[sub], w2c[:1], Kc, c, c, colors=col_h)
        return d, np.where(f >= 0, sub[np.maximum(f, 0)], -1), col

    sd, sf, scol = statement()
    same = (np.array_equal(out["depth"][0, y0:y0 + c, x0:x0 + c].cpu().numpy().view(np.uint32), sd[0].view(np.uint32))
            and np.array_equal(out["face"][0, y0:y0 + c, x0:x0 + c].cpu().numpy(), sf[0])
            and np.array_equal(out["color"][0, y0:y0 + c, x0:x0 + c].cpu().numpy(), scol[0]))

    depths = out["depth"]
    vis = visible_points(points, depths, K, poses)
    dm = depth_metrics(depths, ray["depth"])

    times = {"render_mesh": [], "torch_ops_zbuffer": [], "visible_points": [], "depth_metrics": [],
             "tsdf_render": [], "numpy_statement_us_per_pixel": []}
    for r in range(args.repeats):
        times["render_mesh"].append(_event_ms(lambda: render_mesh(points, faces, K, poses, (h, w), colors=colors)))
        times["torch_ops_zbuffer"].append(_event_ms(lambda: torch_zbuffer(points, faces, K, poses, h, w)))
        times["visible_points"].append(_event_ms(lambda: visible_points(points, depths, K, poses)))
        times["depth_metrics"].append(_event_ms(lambda: depth_metrics(depths, ray["depth"])))
        times["tsdf_render"].append(_event_ms(lambda: vol.render(K, poses, (h, w))))
        if r < 2:
            times["numpy_statement_us_per_pixel"].append(1e6 * timed(statement)[0] / (c * c))

    w2c_dev = torch.from_numpy(w2c).to(dev)
    fi = faces.contiguous()
    cam = (h, w, float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]), 0.01, float("inf"))
    offsets = ops.mesh_bin_count(points, fi, w2c_dev, *cam)
    E = int(offsets[-1].item())
    keys, values = ops.mesh_bin(points, fi, w2c_dev, *cam, offsets, E)
    skeys, order = torch.sort(keys, stable=True)
    start, end = ops.mesh_ranges(skeys, len(poses), h, w)
    k_ms = {"bin_count_and_scan": _kernel_ms(lambda: ops.mesh_bin_count(points, fi, w2c_dev, *cam), args.kernel_iters),
            "bin": _kernel_ms(lambda: ops.mesh_bin(points, fi, w2c_dev, *cam, offsets, E), args.kernel_iters),
            "torch_stable_sort": _kernel_ms(lambda: torch.sort(keys, stable=True), args.kernel_iters),
            "ranges": _kernel_ms(lambda: ops.mesh_ranges(skeys, len(poses), h, w), args.kernel_iters),
            "raster": _kernel_ms(lambda: ops.mesh_raster(points, fi, colors, w2c_dev, *cam, order, values, start, end),
                                 args.kernel_iters)}
    tiles = len(poses) * (-(-h // 16)) * (-(-w // 16))
    lengths = (end - start).flatten().float()

    bench = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(args.bench_steps),
                            "--warmup", str(args.bench_warmup)], capture_output=True, text=True, cwd=ROOT)
    bench_line = next((ln for ln in reversed(bench.stdout.splitlines()) if ln.startswith("{")), None)
    X, Y, Z = vol.dims
    print(json.dumps({
        "card": card(), "volume": {"dims": [X, Y, Z], "voxel_size": args.voxel},
        "mesh": {"points": int(points.shape[0]), "faces": T}, "views": args.views, "size": [h, w],
        "repeats": args.repeats, "hit_share": round(float(hits.float().mean()), 4),
        "ms_median": {k: round(statistics.median(v), 3) for k, v in times.items()},
        "ms": {k: [round(x, 3) for x in v] for k, v in times.items()},
        "kernels_ms_per_call": {k: round(v, 4) for k, v in k_ms.items()},
        "tile_entries": E, "entries_per_face_and_view": round(E / (T * len(poses)), 4),
        "entries_per_tile": {"mean": round(float(lengths.mean()), 2), "max": int(lengths.max())}, "tiles": tiles,
        "peak_device_memory_above_mesh_MiB": {"render_mesh": round(peak_render / 2 ** 20, 1),
                                              "torch_ops_zbuffer": round(peak_torch / 2 ** 20, 1)},
        "torch_ops_zbuffer_agreement": zb_agree,
        "tsdf_render_abs_depth_difference_m_quantiles_50_90_99_100": [round(q, 6) for q in qs],
        "visible_points": {"vertices": int(points.shape[0]), "visible": int(vis.sum())},
        "depth_metrics_mesh_vs_raycast": {k: v for k, v in dm.items() if k != "per_frame"},
        "gpu_equals_numpy_statement_on_crop": bool(same), "crop_faces": int(len(sub)),
        "new_kernels_resource_usage": _resource_usage(),
        "bench_py": json.loads(bench_line) if bench_line else {"error": bench.stderr[-2000:]},
        "time": time.strftime("%Y-%m-%d %H:%M:%S")}))


if __name__ == "__main__":
    main()
