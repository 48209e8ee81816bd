#!/usr/bin/env python
"""Ray casting a TSDF volume at the fusion bench's shape, on one GPU.

    python tools/render_bench.py [--dims 294 217 258] [--voxel 0.01] [--views 8] [--size 480 640] [--repeats 5]
                                 [--kernel-iters 20] [--crop 32] [--bench-steps 5] [--bench-warmup 3]

The volume is `tools/mesh_bench.build_volume`'s analytic room with five objects.  `--views` cameras stand inside the room,
at half its height, each a tenth of the room behind its centre and facing outwards across it in the x-y plane towards the
walls and objects (fx = fy =
0.78 W).  Arms, alternated for `--repeats` rounds after a warm-up, each the median round (CUDA events):
  * `TSDFVolume.render()` end to end (the upload of the poses included);
  * what a user writes today: a torch-ops ray marcher on the GPU -- fixed half-voxel steps in t from 0 to the room's
    diagonal, `grid_sample` trilinear TSDF and weight (observed where the interpolated weight is > 0), the first change
    from >= 0 to < 0, linearly refined; depth only, steps in chunks of 32 to bound memory;
  * the numpy statement (tests/refops_render.py, float32 kernel order) on a `--crop` x `--crop` crop of the first view,
    reported as host time per ray.
Also: the kernel's time per call from CUDA events over `--kernel-iters` back-to-back launches and its rays/s; the mean
number of samples per ray (from the statement, on the crop); the peak device memory above the volume per GPU arm;
whether the kernel equals the statement bit for bit on the crop; the card's name, power limit and SM clocks, read in the
same run; and the JSON line of `bench.py --gpus 1 --steps K --warmup W`, run in the same session.
Prints ONE JSON line.  Writes nothing to the tree.
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from tools.common import card, timed  # noqa: E402
from tools.mesh_bench import _event_ms, _kernel_ms, build_volume  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dims", type=int, nargs=3, default=[294, 217, 258])
    ap.add_argument("--voxel", type=float, default=0.01)
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--size", type=int, nargs=2, default=[480, 640])
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--kernel-iters", type=int, default=20)
    ap.add_argument("--crop", type=int, default=32)
    ap.add_argument("--bench-steps", type=int, default=5)
    ap.add_argument("--bench-warmup", type=int, default=3)
    run(ap.parse_args())


def cameras(extent, n, h, w):
    """Intrinsics and n camera-to-world poses inside the room, facing outwards at angles 2 pi (k + 1/2) / n (camera y
    down = -z)"""
    K = np.array([[0.78 * w, 0, w / 2], [0, 0.78 * w, h / 2], [0, 0, 1]], np.float32)
    c = np.array(extent) / 2
    poses = []
    for k in range(n):
        a = 2 * math.pi * (k + 0.5) / n
        fwd = np.array([math.cos(a), math.sin(a), 0.0])
        down = np.array([0.0, 0.0, -1.0])
        P = np.eye(4)
        P[:3, 0], P[:3, 1], P[:3, 2] = np.cross(down, fwd), down, fwd
        P[:3, 3] = c - 0.1 * np.array(extent) * fwd                    # in free space, at least 17 cm from any surface
        poses.append(P.astype(np.float32))
    return K, poses


def torch_raycast(vol, K, poses, h, w, chunk=32):
    """The torch-ops ray marcher a user writes today: depth [n, h, w], 0 where no crossing is found"""
    dev = vol.device
    X, Y, Z = vol.dims
    P = torch.from_numpy(np.stack(poses)).to(dev)
    ys, xs = torch.meshgrid(torch.arange(h, device=dev, dtype=torch.float32),
                            torch.arange(w, device=dev, dtype=torch.float32), indexing="ij")
    cam = torch.stack([(xs - float(K[0, 2])) / float(K[0, 0]), (ys - float(K[1, 2])) / float(K[1, 1]), torch.ones_like(xs)], -1)
    d = torch.einsum("nij,hwj->nhwi", P[:, :3, :3], cam)                       # [n, h, w, 3]
    o = P[:, None, None, :3, 3]
    origin = torch.tensor(vol.origin, device=dev)
    size = torch.tensor([X, Y, Z], device=dev, dtype=torch.float32) * vol.voxel_size
    field = torch.stack([vol.tsdf, vol.weight])[None]                           # [1, 2, Z, Y, X]
    step = vol.voxel_size / 2
    t_max = float(size.norm())
    depth = torch.zeros(d.shape[:3], device=dev)
    found = torch.zeros(d.shape[:3], dtype=torch.bool, device=dev)
    prev_f = prev_ok = prev_t = None
    for k0 in range(0, int(t_max / step) + 1, chunk):
        t = (torch.arange(k0, k0 + chunk, device=dev, dtype=torch.float32) * step)[None, None, None, :]
        p = o[..., None, :] + t[..., None] * d[..., None, :]                    # [n, h, w, S, 3]
        g = (p - origin) / size * 2 - 1                                          # align_corners=False: voxel centres
        s = F.grid_sample(field, g.reshape(1, -1, chunk, 1, 3), mode="bilinear", align_corners=False)
        f, ok = s[0, 0].reshape(d.shape[:3] + (chunk,)), s[0, 1].reshape(d.shape[:3] + (chunk,)) > 0
        tt = t.expand(d.shape[:3] + (chunk,))
        if prev_f is not None:
            f, ok, tt = torch.cat([prev_f, f], -1), torch.cat([prev_ok, ok], -1), torch.cat([prev_t, tt], -1)
        cross = ok[..., :-1] & ok[..., 1:] & (f[..., :-1] >= 0) & (f[..., 1:] < 0)
        any_c = cross.any(-1) & ~found
        first = cross.float().argmax(-1, keepdim=True)
        fa, fb = f.gather(-1, first)[..., 0], f.gather(-1, first + 1)[..., 0]
        ta, tb = tt.gather(-1, first)[..., 0], tt.gather(-1, first + 1)[..., 0]
        depth = torch.where(any_c, ta + fa / (fa - fb) * (tb - ta), depth)
        found |= any_c
        prev_f, prev_ok, prev_t = f[..., -1:], ok[..., -1:], tt[..., -1:]
    return depth


@torch.no_grad()
def run(args):
    if not torch.cuda.is_available():
        raise SystemExit("render_bench: needs a CUDA device")
    import refops_render as RR
    from unimatch_b200.inference import _camera_to_world
    ops = torch.ops.unimatch_sm100
    dev = torch.device("cuda", 0)
    vol = build_volume(tuple(args.dims), args.voxel, dev)
    torch.cuda.synchronize()
    h, w = args.size
    extent = [n * vol.voxel_size for n in vol.dims]
    K, poses = cameras(extent, args.views, h, w)
    n_rays = args.views * h * w

    def peak(fn):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated(dev)
        torch.cuda.reset_peak_memory_stats(dev)
        out = fn()
        torch.cuda.synchronize()
        return out, torch.cuda.max_memory_allocated(dev) - base

    out, peak_render = peak(lambda: vol.render(K, poses, (h, w)))
    ref_torch, peak_torch = peak(lambda: torch_raycast(vol, K, poses, h, w))
    hits = out["depth"] > 0
    both = hits & (ref_torch > 0)
    agree = float((out["depth"] - ref_torch).abs()[both].median()) if both.any() else None

    c = args.crop
    y0, x0 = (h - c) // 2, (w - c) // 2
    Kc = K.copy()
    Kc[0, 2] -= x0
    Kc[1, 2] -= y0
    planes = {k: getattr(vol, k).cpu().numpy() for k in ("tsdf", "weight", "color")}
    rows = _camera_to_world(poses[:1])

    def statement():
        return RR.raycast(planes, vol.origin, vol.voxel_size, vol.trunc, rows, Kc, c, c, dtype=np.float32, counts=True)

    sd, sc, sn, samples = statement()
    crop = {k: out[k][0, y0:y0 + c, x0:x0 + c].cpu().numpy() for k in out}
    same = (np.array_equal(crop["depth"].view(np.uint32), sd[0].view(np.uint32)) and np.array_equal(crop["color"], sc[0])
            and np.array_equal(crop["normal"].view(np.uint32), sn[0].view(np.uint32)))

    times = {"render": [], "torch_ops": [], "numpy_statement_us_per_ray": []}
    for _ in range(args.repeats):
        times["render"].append(_event_ms(lambda: vol.render(K, poses, (h, w))))
        times["torch_ops"].append(_event_ms(lambda: torch_raycast(vol, K, poses, h, w)))
        times["numpy_statement_us_per_ray"].append(1e6 * timed(statement)[0] / (c * c))

    c2w = torch.from_numpy(_camera_to_world(poses)).to(dev)
    kargs = (vol.tsdf, vol.weight, vol.color, vol.origin, vol.voxel_size, vol.trunc, c2w, h, w, float(K[0, 0]),
             float(K[1, 1]), float(K[0, 2]), float(K[1, 2]), 0.0, float("inf"))
    kernel_ms = _kernel_ms(lambda: ops.tsdf_raycast(*kargs), args.kernel_iters)

    bench = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(args.bench_steps),
                            "--warmup", str(args.bench_warmup)], capture_output=True, text=True, cwd=ROOT)
    bench_line = next((ln for ln in reversed(bench.stdout.splitlines()) if ln.startswith("{")), None)
    X, Y, Z = vol.dims
    print(json.dumps({
        "card": card(), "volume": {"dims": [X, Y, Z], "voxel_size": args.voxel, "voxels": X * Y * Z},
        "views": args.views, "size": [h, w], "rays": n_rays, "repeats": args.repeats,
        "hit_share": round(float(hits.float().mean()), 4),
        "ms_median": {k: round(statistics.median(v), 3) for k, v in times.items()},
        "ms": {k: [round(x, 3) for x in v] for k, v in times.items()},
        "kernel_ms_per_call": round(kernel_ms, 4), "kernel_rays_per_s": round(n_rays / kernel_ms * 1e3),
        "mean_samples_per_ray_on_crop": round(float(samples.mean()), 2),
        "peak_device_memory_above_volume_MiB": {"render": round(peak_render / 2 ** 20, 1),
                                                "torch_ops": round(peak_torch / 2 ** 20, 1)},
        "torch_ops_median_abs_depth_difference_m": agree, "gpu_equals_numpy_statement_on_crop": bool(same),
        "bench_py": json.loads(bench_line) if bench_line else {"error": bench.stderr[-2000:]},
        "time": time.strftime("%Y-%m-%d %H:%M:%S")}))


if __name__ == "__main__":
    main()
