#!/usr/bin/env python
"""Mesh extraction from a TSDF volume at the fusion bench's shape, on one GPU.

    python tools/mesh_bench.py [--dims 294 217 258] [--voxel 0.01] [--repeats 5] [--cpu-repeats 3] [--kernel-iters 20]

The volume is built from an analytic signed distance field: a room (the inside of the volume's box, 5 cm in from its
faces: walls, floor and ceiling are surfaces) holding a few objects (spheres, boxes, a torus), truncated as
`um_tsdf_integrate` would truncate it -- F = min(1, sdf / trunc), weight 1 wherever sdf >= -trunc (trunc = 4 voxels), unobserved behind that -- and
coloured by position.  Arms, alternated for `--repeats` rounds after a warm-up, each the median round:
  * `TSDFVolume.extract_mesh()` end to end (CUDA events; its one host read of the totals included);
  * `TSDFVolume.extract_points()` (CUDA events);
  * what a user does today: download the three planes and run the vectorised numpy statement of the mesh
    (tests/refops_mesh.py, in float32 kernel order) on the host (host clock, `--cpu-repeats` rounds).
Also: P and T; per op, its CUDA-event time per call over `--kernel-iters` back-to-back calls and the bytes it must move, computed from the
shapes (below), with the share of the H100 SXM data-sheet 3.35 TB/s; the peak device memory of `extract_mesh` above the
volume; whether the GPU mesh equals the numpy statement's bit for bit; the card's name, power limit and SM clocks, read
in the same run.  Bytes from shapes (N voxels, nb blocks of 256, P points, T triangles):
  mesh count:    tsdf and weight once (8 N) + block counts (8 nb);       scans: 16 nb each
  point count:   8 N + 8 nb
  vertex pass:   8 N + the colours of both ends of each point's edge (24 P) + points, colours, normals (27 P) + first
                 vertex indices (4 P, at most)
  face pass:     8 N + the first vertex index of each triangle corner's owner (12 T) + faces (12 T)
Prints ONE JSON line.  Writes nothing to the tree.
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

HBM_DATASHEET_GBS = 3350.0
WALL = 0.05                     # the room's walls stand this far (metres) inside the volume's faces


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dims", type=int, nargs=3, default=[294, 217, 258])
    ap.add_argument("--voxel", type=float, default=0.01)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--cpu-repeats", type=int, default=3)
    ap.add_argument("--kernel-iters", type=int, default=20)
    run(ap.parse_args())


def room_sdf(x, extent):
    """Signed distance (metres, positive in free space) of a room [WALL, extent - WALL] per axis holding a few objects, at points
    x [..., 3] (torch float64)"""
    ex = torch.as_tensor(extent, dtype=x.dtype, device=x.device)
    d = torch.minimum(x - WALL, ex - WALL - x).min(-1).values        # inside the room: distance to the nearest wall

    def ball(c, r):
        return (x - torch.tensor(c, dtype=x.dtype, device=x.device)).norm(dim=-1) - r

    def box(c, h):
        q = (x - torch.tensor(c, dtype=x.dtype, device=x.device)).abs() - torch.tensor(h, dtype=x.dtype, device=x.device)
        return q.clamp(min=0).norm(dim=-1) + q.max(-1).values.clamp(max=0)

    def torus(c, R, r):
        p = x - torch.tensor(c, dtype=x.dtype, device=x.device)
        return torch.stack([p[..., 0].hypot(p[..., 1]) - R, p[..., 2]], -1).norm(dim=-1) - r

    w, h, z = extent
    objects = [ball((0.7 * w, 0.35 * h, 0.4 * z), 0.3), ball((0.3 * w, 0.7 * h, 0.65 * z), 0.22),
               box((0.5 * w, 0.2 * h, 0.5 * z), (0.45, 0.2, 0.3)), box((0.2 * w, 0.3 * h, 0.3 * z), (0.15, 0.3, 0.15)),
               torus((0.65 * w, 0.7 * h, 0.3 * z), 0.3, 0.08)]
    return torch.stack([d] + objects, 0).min(0).values


def build_volume(dims, voxel, dev):
    from unimatch_b200.fusion import TSDFVolume
    vol = TSDFVolume((0.0, 0.0, 0.0), voxel, dims, device=dev)
    X, Y, Z = dims
    extent = [n * vol.voxel_size for n in dims]
    axes = [(torch.arange(n, device=dev, dtype=torch.float64) + 0.5) * vol.voxel_size for n in dims]
    for k in range(Z):                                                # a plane at a time: bounded memory
        gy, gx = torch.meshgrid(axes[1], axes[0], indexing="ij")
        x = torch.stack([gx, gy, torch.full_like(gx, float(axes[2][k]))], -1)
        d = room_sdf(x, extent)
        seen = d >= -vol.trunc
        vol.tsdf[k] = torch.where(seen, (d / vol.trunc).clamp(max=1.0), torch.zeros_like(d)).float()
        vol.weight[k] = seen.float()
        for ch in range(3):
            vol.color[ch, k] = (x[..., ch] / extent[ch] * 255).float()
    return vol


def _event_ms(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def _kernel_ms(fn, iters):
    fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


@torch.no_grad()
def run(args):
    if not torch.cuda.is_available():
        raise SystemExit("mesh_bench: needs a CUDA device")
    import refops_mesh as RM
    ops = torch.ops.unimatch_sm100
    dev = torch.device("cuda", 0)
    vol = build_volume(tuple(args.dims), args.voxel, dev)
    torch.cuda.synchronize()
    N = vol.tsdf.numel()
    nb = -(-N // 256)

    def numpy_path():
        planes = {k: getattr(vol, k).cpu().numpy() for k in ("tsdf", "weight", "color")}
        return RM.mesh(planes, vol.origin, vol.voxel_size, np.float32)

    base = torch.cuda.memory_allocated(dev)
    torch.cuda.reset_peak_memory_stats(dev)
    mesh = vol.extract_mesh()                                         # warm-up
    peak = torch.cuda.max_memory_allocated(dev) - base
    vol.extract_points()
    ref = numpy_path()
    same = all(np.array_equal(g.cpu().numpy().view(np.uint8), np.ascontiguousarray(r).view(np.uint8))
               for g, r in zip(mesh, ref))
    P, T = int(mesh[0].shape[0]), int(mesh[3].shape[0])
    del mesh, ref

    times = {"extract_mesh": [], "extract_points": [], "download_and_numpy": []}
    for r in range(args.repeats):
        times["extract_mesh"].append(_event_ms(vol.extract_mesh))
        times["extract_points"].append(_event_ms(vol.extract_points))
        if r < args.cpu_repeats:
            times["download_and_numpy"].append(1000 * timed(numpy_path)[0])

    po = ops.tsdf_surface_count(vol.tsdf, vol.weight)
    fo = ops.tsdf_mesh_count(vol.tsdf, vol.weight)
    args_mesh = (vol.tsdf, vol.weight, vol.color, vol.origin, vol.voxel_size, po, P, fo)
    k_ms = {"point_count_and_scan": _kernel_ms(lambda: ops.tsdf_surface_count(vol.tsdf, vol.weight), args.kernel_iters),
            "mesh_count_and_scan": _kernel_ms(lambda: ops.tsdf_mesh_count(vol.tsdf, vol.weight), args.kernel_iters),
            "vertex_pass": _kernel_ms(lambda: ops.tsdf_mesh(*args_mesh, 0), args.kernel_iters)}
    k_ms["face_pass"] = _kernel_ms(lambda: ops.tsdf_mesh(*args_mesh, T), args.kernel_iters) - k_ms["vertex_pass"]
    nbytes = {"point_count_and_scan": 8 * N + 8 * nb + 16 * nb, "mesh_count_and_scan": 8 * N + 8 * nb + 16 * nb,
              "vertex_pass": 8 * N + (24 + 27 + 4) * P, "face_pass": 8 * N + 24 * T}
    kernels = {k: {"ms": round(ms, 4), "bytes": nbytes[k], "GB_s": round(nbytes[k] / ms / 1e6, 1),
                   "share_of_3350_GB_s": round(nbytes[k] / ms / 1e6 / HBM_DATASHEET_GBS, 4)} for k, ms in k_ms.items()}
    X, Y, Z = vol.dims
    print(json.dumps({
        "card": card(), "volume": {"dims": [X, Y, Z], "voxel_size": args.voxel, "voxels": N,
                                   "GiB": round(20 * N / 2 ** 30, 3)},
        "points": P, "faces": T, "repeats": args.repeats, "cpu_repeats": min(args.cpu_repeats, args.repeats),
        "ms_median": {k: round(statistics.median(v), 3) for k, v in times.items()},
        "ms": {k: [round(x, 3) for x in v] for k, v in times.items()},
        "kernels_ms_per_call": kernels, "extract_mesh_peak_device_memory_above_volume_MiB": round(peak / 2 ** 20, 1),
        "gpu_mesh_equals_numpy_statement": bool(same), "time": time.strftime("%Y-%m-%d %H:%M:%S")}))


if __name__ == "__main__":
    main()
