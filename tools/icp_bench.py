"""Measure ICP tracking against the fused volume (`TSDFVolume.track`, `DepthFusionRunner(track=True)`).

    python tools/icp_bench.py [--dims 294 217 258] [--voxel 0.01] [--views 8] [--size 480 640]

The room of tools/mesh_bench.py and the 8 cameras of tools/render_bench.py: the live depths are render() at the true
poses and tracking starts from poses moved by 2 cm and rotated by 2 degrees.  Reports track() end to end for all frames in
one call and one frame per call, per-op kernel times with the bytes their shapes imply against the 3.35 TB/s HBM3 figure,
a torch-ops ICP with the same model maps, association and solve (what a user writes today) with both paths' pose errors,
and tools/depth_fusion_bench.py's setup through DepthFusionRunner with track=True and track=False.  One JSON line, with
the card read in the same run.
"""
import argparse
import json
import math
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from tools.common import card, timed  # noqa: E402
from tools.mesh_bench import _kernel_ms, build_volume  # noqa: E402
from tools.render_bench import cameras  # noqa: E402

HBM_DATASHEET_GBS = 3350.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dims", type=int, nargs=3, default=[294, 217, 258])
    ap.add_argument("--voxel", type=float, default=0.01)
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--size", type=int, nargs=2, default=[480, 640])
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--kernel-iters", type=int, default=20)
    ap.add_argument("--fusion-frames", type=int, default=64)
    run(ap.parse_args())


def perturb(P, g, metres=0.02, degrees=2.0):
    axis = g.normal(size=3)
    axis /= np.linalg.norm(axis)
    a = math.radians(degrees)
    Kx = np.array([[0.0, -axis[2], axis[1]], [axis[2], 0.0, -axis[0]], [-axis[1], axis[0], 0.0]])
    R = np.eye(3) + math.sin(a) * Kx + (1 - math.cos(a)) * Kx @ Kx
    d = g.normal(size=3)
    Q = np.array(P, np.float64)
    Q[:3, :3] = R @ Q[:3, :3]
    Q[:3, 3] += metres * d / np.linalg.norm(d)
    return Q.astype(np.float32)


def pose_errors(true, est):
    out = []
    for P, Q in zip(true, est):
        P, Q = np.asarray(P, np.float64), np.asarray(Q, np.float64)
        c = np.clip((np.trace(P[:3, :3].T @ Q[:3, :3]) - 1) / 2, -1, 1)
        out.append((float(np.linalg.norm(P[:3, 3] - Q[:3, 3])), math.degrees(math.acos(c))))
    return {"max_translation_m": round(max(e[0] for e in out), 6), "max_rotation_deg": round(max(e[1] for e in out), 4)}


def torch_icp(vol, depths, K, poses, levels=3, iterations=(4, 5, 10), max_distance=0.1, max_angle=20.0):
    """Point-to-plane ICP in torch ops on the device, frame by frame: the model maps from render() at each level, the
    same pyramid, association, Jacobian and Cholesky solve, with a host read of each step's system."""
    from unimatch_b200.fusion import icp_levels
    cos_max = math.cos(math.radians(max_angle))
    out = []
    for d0, P0 in zip(depths, poses):
        lvs = icp_levels(torch.as_tensor(K).numpy(), d0.shape[0], d0.shape[1], levels)
        pyr = [d0]
        for _ in lvs[1:]:
            d = pyr[-1][: pyr[-1].shape[0] // 2 * 2, : pyr[-1].shape[1] // 2 * 2]
            blk = d.reshape(d.shape[0] // 2, 2, d.shape[1] // 2, 2).permute(0, 2, 1, 3).reshape(d.shape[0] // 2, -1, 4)
            ok = torch.isfinite(blk) & (blk > 0)
            lo = torch.where(ok, blk, torch.full_like(blk, float("inf"))).min(-1, keepdim=True).values
            use = ok & (blk - lo <= vol.trunc)
            pyr.append(torch.where(use.any(-1), (blk * use).sum(-1) / use.sum(-1).clamp(min=1), torch.zeros_like(lo[..., 0])))
        T = torch.as_tensor(np.asarray(P0, np.float64), device=d0.device)
        ref = T.clone()
        maps = []
        for (fx, fy, cx, cy, h, w), d in zip(lvs, pyr):
            r = vol.render(np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32), [np.asarray(P0)], (h, w))
            ys, xs = torch.meshgrid(torch.arange(h, device=d.device), torch.arange(w, device=d.device), indexing="ij")
            ray = torch.stack([(xs - cx) / fx, (ys - cy) / fy, torch.ones_like(xs, dtype=torch.float32)], -1)
            v = d[..., None] * ray
            n = torch.zeros_like(v)
            c = torch.cross(v[:-1, 1:] - v[:-1, :-1], v[1:, :-1] - v[:-1, :-1], dim=-1)
            c = c * torch.where((c * v[:-1, :-1]).sum(-1, keepdim=True) > 0, -1.0, 1.0)
            n[:-1, :-1] = torch.nn.functional.normalize(c, dim=-1)
            okd = torch.isfinite(d) & (d > 0)
            okn = torch.zeros_like(okd)
            okn[:-1, :-1] = okd[:-1, :-1] & okd[:-1, 1:] & okd[1:, :-1]
            q = (r["depth"][0][..., None] * ray) @ ref[:3, :3].float().T + ref[:3, 3].float()
            maps.append((v, n, okn, q, r["normal"][0], r["depth"][0] > 0, fx, fy, cx, cy, h, w))
        w2c = torch.linalg.inv(ref)
        for level in reversed(range(levels)):
            v, n, okn, q, m, okm, fx, fy, cx, cy, h, w = maps[level]
            for _ in range(iterations[::-1][level]):
                p = v @ T[:3, :3].float().T + T[:3, 3].float()
                nw = n @ T[:3, :3].float().T
                c = p @ w2c[:3, :3].float().T + w2c[:3, 3].float()
                u = torch.floor(fx * c[..., 0] / c[..., 2] + cx + 0.5)
                vv = torch.floor(fy * c[..., 1] / c[..., 2] + cy + 0.5)
                ok = okn & (c[..., 2] > 0) & (u >= 0) & (u < w) & (vv >= 0) & (vv < h)
                ui, vi = u.clamp(0, w - 1).long(), vv.clamp(0, h - 1).long()
                qq, mm = q[vi, ui], m[vi, ui]
                e = p - qq
                ok &= okm[vi, ui] & (e.norm(dim=-1) <= max_distance) & ((nw * mm).sum(-1) >= cos_max)
                a = torch.cat([torch.cross(p - ref[:3, 3].float(), mm, dim=-1), mm], -1)[ok].double()
                res = (mm * e).sum(-1)[ok].double()
                A, b = a.T @ a, a.T @ res
                if int(ok.sum()) < 36:
                    continue
                x = -torch.cholesky_solve(b[:, None], torch.linalg.cholesky(A))[:, 0]
                th = x[:3].norm()
                Kx = torch.zeros((3, 3), dtype=torch.float64, device=x.device)
                if th > 0:
                    k = x[:3] / th
                    Kx = torch.tensor([[0.0, -k[2], k[1]], [k[2], 0.0, -k[0]], [-k[1], k[0], 0.0]], dtype=torch.float64,
                                      device=x.device)
                dR = torch.eye(3, dtype=torch.float64, device=x.device) + torch.sin(th) * Kx + (1 - torch.cos(th)) * Kx @ Kx
                T = T.clone()
                T[:3, 3] = dR @ (T[:3, 3] - ref[:3, 3]) + ref[:3, 3] + x[3:]
                T[:3, :3] = dR @ T[:3, :3]
        out.append(T.cpu().numpy())
    return out


def run(args):
    from unimatch_b200 import ops
    from unimatch_b200.fusion import _ICP
    if not torch.cuda.is_available():
        raise SystemExit("icp_bench: needs a CUDA device")
    dev = torch.device("cuda", 0)
    h, w = args.size
    n = args.views
    vol = build_volume(tuple(args.dims), args.voxel, dev)
    extent = [d * vol.voxel_size for d in vol.dims]
    K, poses = cameras(extent, n, h, w)
    depths = vol.render(K, poses, (h, w))["depth"]
    g = np.random.default_rng(0)
    start = [perturb(P, g) for P in poses]

    vol.track(depths, K, start)                                     # warm-up
    batch_s = [timed(lambda: vol.track(depths, K, start))[0] for _ in range(args.repeats)]
    single_s = [timed(lambda: [vol.track(depths[i:i + 1], K, start[i:i + 1]) for i in range(n)])[0]
                for _ in range(args.repeats)]
    out = vol.track(depths, K, start)

    # per-op kernel times at the call's shapes
    icp = _ICP(vol, torch.as_tensor(K), n, h, w, 3, (4, 5, 10), 0.1, 20.0, 0.3, "icp_bench")
    pyr, nrm = icp.prepare(depths)
    poses64 = torch.from_numpy(np.stack(start).astype(np.float64)).to(dev)
    nv = torch.tensor([n], dtype=torch.int32, device=dev)
    torch.ops.unimatch_sm100.icp_init(poses64, None, nv, icp.state, icp.c2w, icp.w2c)
    ops_ = torch.ops.unimatch_sm100
    per_op, schedule = {}, {"tsdf_raycast": 0.0, "icp_reduce": 0.0, "icp_solve": 0.0}

    def record(name, fn, nbytes=None):
        ms = _kernel_ms(fn, args.kernel_iters)
        per_op[name] = {"ms": round(ms, 4)}
        if nbytes:
            per_op[name].update(bytes=nbytes, share_of_3350_GB_s=round(nbytes / ms / 1e6 / HBM_DATASHEET_GBS, 4))
        return ms

    px0 = n * h * w
    record("icp_downsample_level0", lambda: ops_.icp_downsample(depths, vol.trunc), 4 * px0 + px0)
    for level, (fx, fy, cx, cy, hl, wl) in enumerate(icp.levels):
        px, nb = n * hl * wl, ops.icp_blocks(hl, wl)
        maps = ops_.tsdf_raycast(vol.tsdf, vol.weight, vol.color, vol.origin, vol.voxel_size, vol.trunc, icp.c2w, hl, wl,
                                 fx, fy, cx, cy, 0.0, math.inf)
        record("icp_normals_level%d" % level, lambda: ops_.icp_normals(pyr[level], fx, fy, cx, cy), 16 * px)
        schedule["tsdf_raycast"] += record("tsdf_raycast_level%d" % level, lambda: ops_.tsdf_raycast(
            vol.tsdf, vol.weight, vol.color, vol.origin, vol.voxel_size, vol.trunc, icp.c2w, hl, wl, fx, fy, cx, cy, 0.0,
            math.inf))
        reduce_ms = record("icp_reduce_level%d" % level, lambda: ops_.icp_reduce(
            pyr[level], nrm[level], maps[0], maps[2], icp.state, icp.c2w, icp.w2c, fx, fy, cx, cy, icp.max_distance,
            icp.cos_max_angle, nv, icp.partials), 3 * 16 * px + 8 * 30 * nb * n)
        # repeated on the same partials: the estimate moves, the work per call does not
        solve_ms = record("icp_solve_level%d" % level, lambda: ops_.icp_solve(icp.partials, nb, nv, 36.0, 1e-2, False,
                                                                               icp.state), 8 * 30 * nb * n)
        steps = icp.iterations[level]
        schedule["icp_reduce"] += (steps + (level == 0)) * reduce_ms
        schedule["icp_solve"] += steps * solve_ms
    # the kernels of one track() call of the n frames, from the per-op times and the schedule's launch counts
    schedule = {k: round(v, 3) for k, v in schedule.items()}

    torch_s, torch_poses = timed(lambda: torch_icp(vol, depths, K, start))

    # the depth fusion bench's setup through the runner, with and without tracking
    from unimatch_b200.fusion import TSDFVolume
    from unimatch_b200.inference import DepthFusionRunner
    from unimatch_b200.synthetic import synthetic_model, synthetic_posed_sequence, workload_call
    model = "gmdepth-scale1-regrefine1"
    m, call = synthetic_model(model), workload_call(model)
    kw = {k: v for k, v in call.items() if k not in ("min_depth", "max_depth", "num_depth_candidates", "task")}
    frames, Kf, fposes = synthetic_posed_sequence(args.fusion_frames, 480, 640, seed=2017)
    items = list(zip(frames.numpy(), fposes.numpy()))
    fps = {}
    for track in (False, True):
        fv = TSDFVolume.covering(Kf, fposes.numpy(), (480, 640), 3.0, 0.01, device=dev)
        runner = DepthFusionRunner(m, (480, 640), 8, dev, Kf, fv, return_depth=False, track=track, **kw)

        def arm():
            fv.reset()
            if track:
                runner.pose_correction.copy_(torch.eye(4, dtype=torch.float64, device=dev))
            for _ in runner.run(items):
                pass
        timed(arm)
        secs = [timed(arm)[0] for _ in range(args.repeats)]
        fps["track" if track else "no_track"] = round((len(items) - 1) / statistics.median(secs), 2)

    print(json.dumps({
        "card": card(), "volume": {"dims": list(vol.dims), "voxel_size": args.voxel}, "views": n, "frame_size": [h, w],
        "track_ms": {"all_frames_one_call_median": round(1000 * statistics.median(batch_s), 3),
                     "one_frame_per_call_median_total": round(1000 * statistics.median(single_s), 3)},
        "tracked": int(out["tracked"].sum()), "inliers_min": int(out["inliers"].min()),
        "pose_error": {"start": pose_errors(poses, start), "track": pose_errors(poses, out["pose"].numpy()),
                       "torch_ops": pose_errors(poses, torch_poses)},
        "torch_ops_icp_ms": round(1000 * torch_s, 3),
        "per_op": per_op, "schedule_ms_from_per_op": schedule,
        "depth_fusion_runner_frames_per_s": fps, "time": time.strftime("%Y-%m-%d %H:%M:%S")}))


if __name__ == "__main__":
    main()
