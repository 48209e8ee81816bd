"""The mesh rasteriser, point visibility and the 2D depth metrics on the device: `render_mesh` against the float32
statement (tests/refops_raster.py) bit for bit -- depth bits, face ids and colours -- on random triangle soups,
icospheres seen from inside and outside, the mesh of a fused random clip, a coarse bench room, batches mixing cameras
inside, outside, facing away and straddling the mesh, an empty mesh, no cameras, and faces covering whole frames; the
same output from a second call; `visible_points` exactly and `depth_metrics` counts exactly and means to 1e-12 against
the statement; and end to end, a rendered analytic mesh fused and scored, and visibility culling restoring recall."""
import math

import numpy as np
import pytest
import torch

import refops_fusion as RF
import refops_raster as RS
from test_fusion_cpu import covering_scene
from test_fusion_gpu import DIMS, ORIGIN, VS, _random_clip
from test_fusion_gpu import K as KF
from test_render_cpu import _depth_bound
from unimatch_b200.evaluation import depth_metrics, depth_metrics_from_sums, reconstruction_metrics
from unimatch_b200.fusion import TSDFVolume, fuse_depths, render_mesh, visible_points
from unimatch_b200.inference import _world_to_camera

pytestmark = pytest.mark.gpu


def _np(x):
    return x.cpu().numpy() if torch.is_tensor(x) else np.asarray(x)


def _check(points, faces, K, poses, h, w, colors=None, near=0.01, far=None, min_hits=1):
    """render_mesh against the float32 statement; returns the output"""
    out = render_mesh(points, faces, K, poses, (h, w), colors=colors, near=near, far=far)
    n = len(poses)
    assert out["depth"].shape == (n, h, w) and out["face"].dtype == torch.int32 and out["depth"].is_cuda
    w2c = _world_to_camera([np.asarray(p, np.float32) for p in poses])
    rd, rf, rc = RS.raster(_np(points).astype(np.float32), _np(faces), w2c, np.asarray(K, np.float32), h, w,
                           colors=colors, near=near, far=np.inf if far is None else far)
    assert np.array_equal(out["depth"].cpu().numpy().view(np.uint32), rd.view(np.uint32))
    assert np.array_equal(out["face"].cpu().numpy(), rf)
    if colors is not None:
        assert np.array_equal(out["color"].cpu().numpy(), rc)
    else:
        assert "color" not in out
    assert (rf >= 0).sum() >= min_hits
    again = render_mesh(points, faces, K, poses, (h, w), colors=colors, near=near, far=far)
    for k in out:
        assert torch.equal(out[k], again[k])
    return out


def _colors(n, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, 3), dtype=np.uint8)


K = np.array([[30.0, 0, 27.5], [0, 30.0, 19.5], [0, 0, 1]], np.float32)
H, W = 40, 56


@pytest.mark.parametrize("seed", [0, 1])
def test_random_triangle_soup(seed):
    g = np.random.default_rng(seed)
    pts = g.uniform(-1, 1, (600, 3)).astype(np.float32)
    pts[:, 2] += 2.5
    faces = g.integers(0, 600, (400, 3)).astype(np.int32)
    poses = [RS.pose(np.eye(3), g.uniform(-0.3, 0.3, 3)) for _ in range(3)]
    _check(pts, faces, K, poses, H, W, colors=_colors(600, seed), min_hits=100)
    _check(torch.from_numpy(pts).cuda(), torch.from_numpy(faces.astype(np.int64)), K, poses, H, W, far=2.6, min_hits=10)


def test_icospheres_inside_and_outside():
    pts, tri = RS.icosphere(3, 1.0, jitter=0.03, seed=2)
    g = np.random.default_rng(3)
    inside = [RS.pose(RS.random_rotation(g), g.uniform(-0.3, 0.3, 3)) for _ in range(3)]
    out = _check(pts, tri, K, inside, H, W, colors=_colors(len(pts), 1))
    assert (out["face"] >= 0).all()
    outside = [RS.look_at(3.0 * np.array([math.cos(a), math.sin(a), 0.3]), (0, 0, 0)) for a in (0.0, 2.0, 4.0)]
    _check(pts, tri, K, outside, H, W, colors=_colors(len(pts), 2), min_hits=500)


def test_mesh_of_a_fused_random_clip():
    d, frames, poses = _random_clip(6, 40, 56, seed=5)
    vol = TSDFVolume(ORIGIN, VS, DIMS, device="cuda")
    fuse_depths(vol, torch.from_numpy(d).cuda(), torch.from_numpy(frames).cuda(), KF, poses)
    pts, cols, _, tri = vol.extract_mesh()
    assert tri.shape[0] > 100
    _check(pts, tri, KF, poses[:3], 40, 56, colors=cols.cpu().numpy(), min_hits=100)


def test_coarse_bench_room():
    from tools.mesh_bench import build_volume
    from tools.render_bench import cameras
    vol = build_volume((60, 44, 52), 0.05, torch.device("cuda", 0))
    pts, cols, _, tri = vol.extract_mesh()
    extent = [n * vol.voxel_size for n in vol.dims]
    Kc, poses = cameras(extent, 2, 24, 32)
    out = _check(pts, tri, Kc, poses, 24, 32, colors=cols.cpu().numpy())
    assert (out["face"] >= 0).float().mean() > 0.95


def test_mixed_batch_and_whole_frame_faces():
    pts, tri = RS.icosphere(2, 1.0, centre=(0, 0, 3.0), jitter=0.05, seed=4)
    big = np.array([[-50, -50, 5.0], [50, -50, 5.0], [0, 60, 5.0], [-50, -50, 1.2], [50, -50, 1.4], [0, 60, 1.3]],
                   np.float32)
    pts2 = np.concatenate([pts, big])
    tri2 = np.concatenate([tri, len(pts) + np.array([[0, 1, 2], [3, 4, 5]], np.int32)])
    poses = [RS.pose(np.eye(3), (0, 0, 3.0)),                             # inside the sphere
             RS.pose(np.eye(3), (0.1, 0.0, 0.0)),                         # outside, facing it
             RS.pose(RF.rot("y", math.pi), (0, 0, 0.0)),                  # facing away
             RS.pose(np.eye(3), (0.0, 0.0, 2.0))]                         # straddling: inside the sphere's near cap
    _check(pts2, tri2, K, poses, H, W, colors=_colors(len(pts2), 5), min_hits=1000)


def test_empty_mesh_and_no_cameras():
    P = [np.eye(4, dtype=np.float32)]
    out = render_mesh(np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32), K, P, (H, W))
    assert (out["depth"] == 0).all() and (out["face"] == -1).all()
    pts, tri = RS.icosphere(0, 1.0, centre=(0, 0, 3))
    out = render_mesh(pts, tri, K, [], (H, W), colors=_colors(len(pts), 0))
    assert out["depth"].shape == (0, H, W) and out["color"].shape == (0, H, W, 3)
    out = render_mesh(pts, np.zeros((0, 3), np.int64), K, P, (H, W), colors=_colors(len(pts), 0))
    assert (out["face"] == -1).all() and (out["color"] == 0).all()


def test_visible_points_matches_the_statement():
    pts, tri = RS.icosphere(3, 1.0, centre=(0, 0, 3.0), jitter=0.02, seed=6)
    poses = [RS.pose(np.eye(3), (0.2 * i - 0.2, 0.0, 0.0)) for i in range(3)]
    depth = render_mesh(pts, tri, K, poses, (H, W))["depth"]
    g = np.random.default_rng(7)
    q = np.concatenate([pts, g.uniform(-2, 2, (2000, 3)).astype(np.float32) + np.float32([0, 0, 3])])
    q[5] = np.nan
    for tol in (0.0, 0.05, 0.5):
        vis = visible_points(q, depth, K, poses, tolerance=tol)
        w2c = _world_to_camera([np.asarray(p, np.float32) for p in poses])
        ref = RS.visible(q, depth.cpu().numpy(), w2c, K, tol)
        assert vis.dtype == torch.bool and np.array_equal(vis.cpu().numpy(), ref)
        assert 0 < ref.sum() < len(q)


def test_depth_metrics_match_the_statement():
    g = np.random.default_rng(8)
    gt = g.uniform(0.2, 12.0, (5, 37, 61)).astype(np.float32)
    pred = (gt * g.uniform(0.6, 1.5, gt.shape)).astype(np.float32)
    pred[g.random(pred.shape) < 0.1] = 0
    pred[g.random(pred.shape) < 0.02] = np.nan
    gt[g.random(gt.shape) < 0.05] = np.inf
    pred[3] = 0
    out = depth_metrics(torch.from_numpy(pred).cuda(), torch.from_numpy(gt).cuda())
    ref = depth_metrics_from_sums(RS.depth_sums(pred, gt), 37 * 61)
    assert out["n_frames"] == ref["n_frames"] == 4
    assert np.array_equal(out["per_frame"]["n_masked"], ref["per_frame"]["n_masked"])
    for k in ("r1", "r2", "r3", "complete"):
        assert np.array_equal(out["per_frame"][k], ref["per_frame"][k], equal_nan=True)
    for k in ("AbsRel", "AbsDiff", "SqRel", "RMSE", "LogRMSE"):
        np.testing.assert_allclose(out["per_frame"][k], ref["per_frame"][k], rtol=1e-12, equal_nan=True)
        assert abs(out[k] - ref[k]) <= 1e-12 * abs(ref[k])
    again = depth_metrics(torch.from_numpy(pred).cuda(), torch.from_numpy(gt).cuda())
    assert all(out[k] == again[k] for k in ("AbsRel", "RMSE", "LogRMSE", "complete"))


def _sphere_mesh(scene, subdivisions=5):
    pts, tri = RS.icosphere(subdivisions, scene[2], centre=scene[1])
    c = pts[tri].astype(np.float64).mean(1)
    sag = float(scene[2] - np.linalg.norm(c - np.asarray(scene[1]), axis=1).min())     # the mesh's largest gap
    return pts, tri, sag


def test_rendered_mesh_fused_and_scored():
    """The sphere clip's sphere as an icosphere (max gap `sag` from the sphere), rendered at the clip's poses, fused and
    extracted: each extracted point lies within the render tests' footprint bound of the sphere, so the accuracy against
    the mesh's vertices stays below that bound plus the gap plus the vertex spacing."""
    vs, trunc, h, w, scale = 0.01, 0.04, 48, 64, 8
    scene, Kx, poses = RF.sphere_clip(h=h * scale, w=w * scale)
    Kr = RF.sphere_clip(h=h, w=w)[1]
    pts, tri, sag = _sphere_mesh(scene)
    origin, dims = covering_scene(scene)
    vol = TSDFVolume(origin, vs, dims, trunc=trunc, device="cuda")
    P32 = [P.astype(np.float32) for P in poses]
    depth = render_mesh(pts, tri, np.asarray(Kx, np.float32), P32, (h * scale, w * scale))["depth"]
    assert (depth > 0).all()
    frames = torch.zeros(depth.shape + (3,), dtype=torch.uint8, device="cuda")
    fuse_depths(vol, depth, frames, np.asarray(Kx, np.float32), P32)
    pred = vol.extract_points()[0]
    lo, hi = np.array(origin) - trunc, np.array(origin) + vs * np.array(dims) + trunc
    tol = _depth_bound(scene, Kx, poses, Kr, poses, vs, lo, hi, h, w, scale)
    edge = float(np.linalg.norm(pts[tri[:, 0]] - pts[tri[:, 1]], axis=1).max())
    m = reconstruction_metrics(pred, pts, down_sample=None)
    assert m["n_pred"] > 1000 and m["acc"] < tol + sag + edge, (m, tol, sag, edge)


def test_visibility_culling_restores_recall():
    """GT: the whole sphere (an icosphere's vertices), of which the clip's cameras see only the near cap.  The
    prediction, a full reconstruction of the seen side (every rendered depth back-projected), scores a low recall
    against all of it; culling both sets to what the cameras saw (`visible_points` in the GT mesh's rendered depths)
    brings recall near 1."""
    h, w = 96, 128
    scene, Kx, poses = RF.sphere_clip(h=h, w=w)
    pts, tri, _ = _sphere_mesh(scene)
    P32 = [P.astype(np.float32) for P in poses]
    K32 = np.asarray(Kx, np.float32)
    depth = render_mesh(pts, tri, K32, P32, (h, w))["depth"]
    assert (depth > 0).all()
    d = depth.cpu().numpy().astype(np.float64)
    pred = np.concatenate([P[:3, 3] + (RF.rays(Kx, h, w) @ P[:3, :3].T) * di[..., None] for P, di in zip(poses, d)])
    pred = torch.from_numpy(pred.reshape(-1, 3).astype(np.float32)).cuda()
    gt = torch.from_numpy(pts).cuda()
    raw = reconstruction_metrics(pred, gt)
    vis_p, vis_g = visible_points(pred, depth, K32, P32), visible_points(gt, depth, K32, P32)
    assert bool(vis_p.all()) and 0 < int(vis_g.sum()) < len(pts) // 2
    culled = reconstruction_metrics(pred[vis_p], gt[vis_g])
    assert raw["recall"] < 0.5 and culled["recall"] > 0.97 and culled["prec"] > 0.97, (raw, culled)
