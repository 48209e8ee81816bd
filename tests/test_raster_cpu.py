"""The mesh rasteriser, point visibility and the 2D depth metrics without a GPU: the numpy statement
(tests/refops_raster.py) on closed meshes seen from inside (no pixel misses, including vertices and edges exactly on
pixel centres), float32 against float64 on analytic polyhedra, hand-made cases (colour, ties, degenerate faces, faces
crossing near, z = 0 or the camera, far cuts, large faces, odd frame sizes), the pixel rectangle shown to change nothing,
`visible_points` and `depth_metrics` hand cases, and the argument refusals of all three functions."""
import math

import numpy as np
import pytest
import torch

import refops_mesh as RM
import refops_raster as RS
from unimatch_b200.evaluation import depth_metrics, depth_metrics_from_sums
from unimatch_b200.fusion import render_mesh, visible_points
from unimatch_b200.inference import _world_to_camera

K = np.array([[20.0, 0, 12.5], [0, 20.0, 9.5], [0, 0, 1]], np.float32)
H, W = 20, 25


def _w2c(poses):
    return _world_to_camera([np.asarray(p, np.float32) for p in poses])


def _rasters(points, faces, poses, Kc=K, h=H, w=W, **kw):
    """The float32 statement with and without the rectangle; asserts they agree and returns the first"""
    w2c = _w2c(poses)
    a = RS.raster(points, faces, w2c, Kc, h, w, **kw)
    b = RS.raster(points, faces, w2c, Kc, h, w, rect=False, **kw)
    for x, y in zip(a, b):
        if x is not None:
            assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))
    return a


def _inside_poses(centre, n, seed, spread=0.2):
    g = np.random.default_rng(seed)
    return [RS.pose(RS.random_rotation(g), np.asarray(centre) + g.uniform(-spread, spread, 3)) for _ in range(n)]


def torus_mesh():
    vol = RM.sdf_volume(RM.torus((0, 0, 0), 0.6, 0.25), (-1, -1, -0.5), 0.05, (40, 40, 20), 0.2)
    pts, _, _, tri = RM.mesh(vol, (-1, -1, -0.5), 0.05, np.float32)
    return pts.astype(np.float32), tri


def sphere_mesh():
    vol = RM.sdf_volume(RM.sphere((0.02, -0.01, 0.03), 0.7), (-1, -1, -1), 0.1, (20, 20, 20), 0.4)
    pts, _, _, tri = RM.mesh(vol, (-1, -1, -1), 0.1, np.float32)
    return pts.astype(np.float32), tri


def closed_scenes():
    """(name, points, faces, camera poses inside)"""
    ico = RS.icosphere(2, 1.0, jitter=0.05, seed=1)
    tor = torus_mesh()
    sph = sphere_mesh()
    box = RS.room_box((-1.5, -1.0, -0.75), (1.5, 1.0, 0.75), n=3)
    around_core = [RS.pose(RS.random_rotation(np.random.default_rng(s)), [0.6 * math.cos(s), 0.6 * math.sin(s), 0.02])
                   for s in range(3)]
    return [("icosphere", *ico, _inside_poses((0, 0, 0), 3, 0)), ("torus", *tor, around_core),
            ("sphere", *sph, _inside_poses((0, 0, 0), 3, 1)), ("room", *box, _inside_poses((0, 0, 0), 3, 2, 0.5))]


@pytest.mark.parametrize("scene", range(4))
def test_camera_inside_a_closed_mesh_has_no_miss(scene):
    name, pts, tri, poses = closed_scenes()[scene]
    assert not RM.unmatched_edges(tri), name
    d, f, _ = _rasters(pts, tri, poses)
    assert (f >= 0).all() and (d > 0).all(), name


def _dyadic_views():
    """Axis-aligned cameras at the centre of the box [-1, 1]^3 with integer intrinsics: every box vertex in view projects
    exactly onto a pixel centre, and the squares' edges and diagonals run exactly through pixel centres"""
    Kd = np.array([[8.0, 0, 8], [0, 8.0, 8], [0, 0, 1]], np.float32)
    Rs = [np.eye(3), np.array([[0, 0, 1], [0, 1, 0], [-1, 0, 0.0]]), np.array([[1, 0, 0], [0, 0, -1], [0, 1, 0.0]]),
          np.diag([-1.0, 1, -1])]
    return Kd, [RS.pose(R, (0, 0, 0)) for R in Rs]


@pytest.mark.parametrize("n", [1, 2, 4])
def test_watertight_on_vertices_and_edges_through_pixel_centres(n):
    pts, tri = RS.room_box(n=n)
    Kd, poses = _dyadic_views()
    d, f, _ = _rasters(pts, tri, poses, Kd, 17, 17)
    assert (f >= 0).all()
    assert np.array_equal(d[:, 8, 8], np.ones(4, np.float32))           # the wall straight ahead at 1
    assert (d[:, 0, 0] == 1).all() and (d[:, 16, 16] == 1).all()        # the corners, exactly on vertices


def test_float32_agrees_with_float64_within_a_derived_bound():
    """Analytic polyhedra (an icosahedron from inside and outside, the room box): where both forms pick one face, the
    float32 depth is within its rounding bound of the float64 one.  t = det / S; with u = 2^-24: the float32 camera
    coordinates are within 3u (|M| |p| + |t|) <= 6u |V| of the float64 ones here (cameras within 0.5 of the centre,
    every vertex at least 0.5 away), which moves det by at most 18u and S by at most 12u of their absolute-value forms;
    each cross product adds 2u of its absolute products, each dot product 3u and the sum of three edge values 2u.  So
    |det - det64| <= 24u det_abs, |S - S64| <= 24u S_abs, and |t - t64| / |t64| <= 24u (det_abs / |det| + S_abs / |S|)
    + u (the division)."""
    u = 2.0 ** -24
    scenes = [(*RS.icosphere(0, 1.0), _inside_poses((0, 0, 0), 3, 5)),
              (*RS.icosphere(0, 1.0), [RS.look_at((2.5, 0.3, 0.4), (0, 0, 0)), RS.look_at((-0.5, 2.2, 1.0), (0, 0, 0))]),
              (*RS.room_box(n=2), _inside_poses((0, 0, 0), 3, 6, 0.4))]
    for pts, tri, poses in scenes:
        w2c32 = _w2c(poses)
        w2c64 = np.stack([np.linalg.inv(np.asarray(p, np.float32).astype(np.float64)) for p in poses])[:, :3]
        d32, f32, _ = RS.raster(pts, tri, w2c32, K, H, W, dtype=np.float32)
        d64, f64, _ = RS.raster(pts, tri, w2c64, K, H, W, dtype=np.float64)
        assert np.array_equal(f32 >= 0, f64 >= 0)
        same = (f32 == f64) & (f32 >= 0)
        assert same.mean() > 0.9 * (f32 >= 0).mean()
        ys, xs = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
        xc, yc = (xs - K[0, 2]) / K[0, 0], (ys - K[1, 2]) / K[1, 1]
        for v in range(len(poses)):
            V = RS.camera_vertices(pts, w2c64[v], np.float64)
            fi = tri[np.where(same[v], f64[v], 0)].astype(np.int64)
            A, B, C = V[fi[..., 0]], V[fi[..., 1]], V[fi[..., 2]]
            dvec = np.stack([xc, yc, np.ones_like(xc)], -1)
            n = np.cross(B - A, C - A)
            S = (n * dvec).sum(-1)

            def abscross(a, b):
                return np.stack([np.abs(a[..., 1] * b[..., 2]) + np.abs(a[..., 2] * b[..., 1]),
                                 np.abs(a[..., 2] * b[..., 0]) + np.abs(a[..., 0] * b[..., 2]),
                                 np.abs(a[..., 0] * b[..., 1]) + np.abs(a[..., 1] * b[..., 0])], -1)
            S_abs = ((abscross(A, B) + abscross(B, C) + abscross(C, A)) * np.abs(dvec)).sum(-1)
            det = (A * np.cross(B, C)).sum(-1)
            det_abs = (np.abs(A) * abscross(B, C)).sum(-1)
            bound = 24 * u * (det_abs / np.abs(det) + S_abs / np.abs(S)) + u
            rel = np.abs(d32[v].astype(np.float64) - d64[v]) / np.where(same[v], d64[v], 1.0)
            assert (rel[same[v]] <= bound[same[v]]).all(), (rel[same[v]].max(), bound[same[v]].min())


def _one_triangle(z=2.0):
    return np.array([[-1, -1, z], [1, -1, z], [0, 1, z]], np.float32), np.array([[0, 1, 2]], np.int32)


def test_colour_of_one_triangle_is_hand_computed():
    pts, tri = _one_triangle()
    Kc = np.array([[4.0, 0, 2], [0, 4.0, 2], [0, 0, 1]], np.float32)
    cols = np.array([[255, 0, 0], [0, 255, 0], [0, 0, 255]], np.uint8)
    d, f, c = _rasters(pts, tri, [np.eye(4)], Kc, 5, 5, colors=cols)
    # pixel (2, 2): ray (0, 0, 1) hits (0, 0, 2): barycentrics (1/4, 1/4, 1/2)
    assert d[0, 2, 2] == 2.0 and f[0, 2, 2] == 0
    assert c[0, 2, 2].tolist() == [64, 64, 128]                 # rint(63.75), rint(63.75), rint(127.5) (half to even)
    # pixel (2, 1): ray (0, -1/4, 1) hits (0, -1/2, 2): barycentrics (3/8, 3/8, 1/4)
    assert c[0, 1, 2].tolist() == [96, 96, 64]                  # rint(95.625), rint(95.625), rint(63.75)
    assert f[0, 0, 0] == 0 and c[0, 0, 0].tolist() == [255, 0, 0]     # the ray through vertex A
    assert f[0, 4, 0] == -1 and d[0, 4, 0] == 0 and c[0, 4, 0].tolist() == [0, 0, 0]   # (-1, 1, 2): outside


def test_coincident_and_duplicated_faces_go_to_the_least_index():
    pts, tri = _one_triangle()
    pts = np.concatenate([pts, pts])                                   # the same triangle through other vertices
    faces = np.array([[3, 4, 5], [0, 1, 2], [2, 1, 0], [0, 1, 2]], np.int32)
    cols = np.zeros((6, 3), np.uint8)
    cols[:3] = 200
    cols[3:] = 50
    d, f, c = _rasters(pts, faces, [np.eye(4)], np.array([[4.0, 0, 2], [0, 4.0, 2], [0, 0, 1]], np.float32), 5, 5,
                       colors=cols)
    hit = f >= 0
    assert hit.sum() > 3 and (f[hit] == 0).all() and (c[hit] == 50).all()


def test_degenerate_faces_are_never_hit():
    # repeated indices; vertices 0 and 3 coincide; 1, 4 and 5 are collinear (exact small integers, so S is exactly 0)
    pts = np.array([[-1, -1, 2], [1, -1, 2], [0, 1, 2], [-1, -1, 2], [3, -1, 2], [2, -1, 2]], np.float32)
    faces = np.array([[0, 0, 1], [0, 1, 1], [2, 2, 2], [0, 3, 1], [1, 4, 5], [1, 5, 4]], np.int32)
    Kc = np.array([[4.0, 0, 2], [0, 4.0, 2], [0, 0, 1]], np.float32)
    d, f, _ = _rasters(pts, faces, [np.eye(4)], Kc, 5, 9)
    assert (f == -1).all() and (d == 0).all()


def test_faces_crossing_near_zero_behind_and_around_the_camera():
    Kc = np.array([[6.0, 0, 4.5], [0, 6.0, 3.5], [0, 0, 1]], np.float32)
    g = np.random.default_rng(4)
    cases = {
        "crosses near": np.array([[-1, -1, 0.005], [1, -1, 0.5], [0, 1, 0.2]], np.float32),
        "crosses z = 0": np.array([[-1, -1, -0.5], [1, -0.5, 0.8], [0, 1, 0.3]], np.float32),
        "behind": np.array([[-1, -1, -1], [1, -1, -1], [0, 1, -1]], np.float32),
        "around the camera": np.array([[-3, -3, -1], [3, -3, 1], [0, 3, 0.1]], np.float32),
    }
    for name, pts in cases.items():
        d, f, _ = _rasters(pts, np.array([[0, 1, 2]], np.int32), [np.eye(4)], Kc, 8, 10, near=0.01)
        assert ((d >= np.float32(0.01)) | (f < 0)).all(), name
        if name == "behind":
            assert (f < 0).all()
        if name == "crosses z = 0":
            assert (f == 0).any()
    soup = g.uniform(-1, 1, (60, 3)).astype(np.float32)
    soup[:, 2] = g.uniform(-0.3, 0.6, 60)
    d, f, _ = _rasters(soup, np.arange(60, dtype=np.int32).reshape(20, 3), [np.eye(4)], Kc, 8, 10, near=0.05)
    assert (d[f >= 0] >= np.float32(0.05)).all()


def test_far_cuts_and_faces_larger_than_the_frame():
    pts, tri = _one_triangle(3.0)
    pts = pts * np.float32([40, 40, 1])                                 # much larger than the frame
    Kc = np.array([[6.0, 0, 4.5], [0, 6.0, 3.5], [0, 0, 1]], np.float32)
    d, f, _ = _rasters(pts, tri, [np.eye(4)], Kc, 8, 10)
    assert (f == 0).all() and (d == 3).all()
    d, f, _ = _rasters(pts, tri, [np.eye(4)], Kc, 8, 10, far=2.5)
    assert (f == -1).all()
    d, f, _ = _rasters(pts, tri, [np.eye(4)], Kc, 8, 10, far=3.0)
    assert (f == 0).all()


@pytest.mark.parametrize("hw", [(1, 1), (17, 33), (31, 18)])
def test_small_and_odd_frames(hw):
    h, w = hw
    pts, tri = RS.icosphere(1, 1.0, jitter=0.1, seed=3)
    Kc = np.array([[0.8 * w + 1, 0, (w - 1) / 2], [0, 0.8 * w + 1, (h - 1) / 2], [0, 0, 1]], np.float32)
    d, f, _ = _rasters(pts, tri, _inside_poses((0, 0, 0), 2, 7), Kc, h, w)
    assert (f >= 0).all()
    d, f, _ = _rasters(pts, tri, [RS.look_at((0.3, -3.0, 0.4), (0, 0, 0))], Kc, h, w)
    assert (d[f >= 0] > 1.5).all()


def test_rectangles_hold_tile_counts():
    pts, tri = RS.icosphere(1, 1.0)
    w2c = _w2c(_inside_poses((0, 0, 0), 2, 8))
    x0, x1, y0, y1, ok = RS.rectangles(pts, tri, w2c[0], K, H, W, 0.01)
    assert 0 < ok.sum() < len(tri)                                      # faces behind the camera get none
    assert (x0[ok] >= 0).all() and (x1[ok] <= W - 1).all() and (x0[ok] <= x1[ok]).all() and (y0[ok] <= y1[ok]).all()
    assert RS.bin_entries(pts, tri, w2c[:1], K, H, W, 0.01) >= ok.sum()


# ---- visible_points ---------------------------------------------------------------------------------------------------
def test_visible_points_hand_cases():
    Kc = np.array([[4.0, 0, 2], [0, 4.0, 2], [0, 0, 1]], np.float32)
    depth = np.full((1, 5, 5), 2.0, np.float32)
    depth[0, 0, 0] = 0.0
    depth[0, 4, 4] = np.nan
    pts = np.array([[0, 0, 1.0],          # in front of the surface: seen
                    [0, 0, 3.0],          # occluded
                    [0, 0, 2.04],         # behind, within tolerance
                    [0, 0, 2.06],         # behind, beyond tolerance
                    [5, 0, 1.0],          # outside the frame
                    [0, 0, -1.0],         # behind the camera
                    [-1, -1, 2.0],        # on the pixel with depth 0
                    [1, 1, 2.0]], np.float32)   # on the NaN pixel
    vis = RS.visible(pts, depth, _w2c([np.eye(4)]), Kc, 0.05)
    assert vis.tolist() == [True, False, True, False, False, False, False, False]
    two = np.concatenate([depth, np.full((1, 5, 5), 5.0, np.float32)])
    assert RS.visible(pts, two, _w2c([np.eye(4), np.eye(4)]), Kc, 0.05).tolist() == \
        [True, True, True, True, False, False, True, True]


# ---- depth_metrics ------------------------------------------------------------------------------------------------
def test_depth_metrics_against_a_float64_formula():
    g = np.random.default_rng(9)
    gt = g.uniform(0.3, 12.0, (4, 6, 7)).astype(np.float32)
    pred = (gt * g.uniform(0.7, 1.4, gt.shape)).astype(np.float32)
    pred[0, 0, :3] = [0, -1, np.inf]
    gt[0, 1, :2] = [np.nan, 0]
    pred[2] = 0                                                          # no estimate anywhere: a NaN frame
    pred[3, :2] = np.nan
    out = depth_metrics_from_sums(RS.depth_sums(pred, gt), 42)
    assert out["n_frames"] == 3 and math.isnan(out["per_frame"]["AbsRel"][2])
    rows = []
    for p, t in zip(pred, gt):
        has = np.isfinite(p) & (p > 0)
        m = has & np.isfinite(t) & (t > 0) & (t < 10)
        pp, tt = p[m].astype(float), t[m].astype(float)
        r = np.maximum(tt / pp, pp / tt)
        rows.append([np.mean(np.abs(pp - tt) / tt), np.mean(np.abs(pp - tt)), np.mean((pp - tt) ** 2 / tt),
                     np.sqrt(np.mean((pp - tt) ** 2)), np.sqrt(np.mean((np.log(pp) - np.log(tt)) ** 2)),
                     np.mean(r < 1.25), np.mean(r < 1.25 ** 2), np.mean(r < 1.25 ** 3), has.mean()] if m.any() else
                    [np.nan] * 8 + [has.mean()])
    rows = np.array(rows)
    for k, key in enumerate(("AbsRel", "AbsDiff", "SqRel", "RMSE", "LogRMSE", "r1", "r2", "r3", "complete")):
        np.testing.assert_allclose(out["per_frame"][key], rows[:, k], rtol=1e-12, equal_nan=True)
        want = np.nanmean(rows[:, k]) if key != "complete" else rows[:, k].mean()
        assert abs(out[key] - want) <= 1e-12 * abs(want)
    assert out["complete"] < 1 and out["per_frame"]["complete"][2] == 0


# ---- argument refusals --------------------------------------------------------------------------------------------
def _mesh():
    pts, tri = _one_triangle()
    return pts, tri


@pytest.mark.parametrize("case", ["nan_vertex", "index_high", "index_negative", "float_faces", "bad_k", "nan_pose",
                                  "near0", "far_le_near", "views", "pixels", "colors", "points_shape"])
def test_render_mesh_refusals(case):
    pts, tri = _mesh()
    kw = dict(points=pts, faces=tri, intrinsics=K, poses=[np.eye(4, dtype=np.float32)], frame_size=(H, W), device="cpu")
    if case == "nan_vertex":
        kw["points"] = pts.copy()
        kw["points"][1, 2] = np.nan
    elif case == "index_high":
        kw["faces"] = np.array([[0, 1, 3]], np.int32)
    elif case == "index_negative":
        kw["faces"] = np.array([[0, -1, 2]], np.int64)
    elif case == "float_faces":
        kw["faces"] = tri.astype(np.float32)
    elif case == "bad_k":
        Kb = K.copy()
        Kb[0, 0] = 0
        kw["intrinsics"] = Kb
    elif case == "nan_pose":
        P = np.eye(4, dtype=np.float32)
        P[0, 3] = np.nan
        kw["poses"] = [P]
    elif case == "near0":
        kw["near"] = 0.0
    elif case == "far_le_near":
        kw["near"], kw["far"] = 1.0, 1.0
    elif case == "views":
        kw["poses"] = [np.eye(4, dtype=np.float32)] * 65536
    elif case == "pixels":
        kw["frame_size"] = (65536, 32768)
    elif case == "colors":
        kw["colors"] = np.zeros((3, 3), np.float32)
    elif case == "points_shape":
        kw["points"] = pts[:, :2]
    match = {"nan_vertex": "finite", "index_high": "face indices", "index_negative": "face indices",
             "float_faces": "integer faces", "bad_k": "fx, fy", "nan_pose": "poses must be finite", "near0": "near",
             "far_le_near": "near", "views": "65535", "pixels": "2\\^31", "colors": "colors",
             "points_shape": "points"}[case]
    with pytest.raises(ValueError, match=match):
        render_mesh(**kw)


def test_visible_points_and_depth_metrics_refusals():
    d = torch.zeros((1, 4, 4))
    with pytest.raises(ValueError):
        visible_points(np.zeros((3, 3), np.float32), d, K, [np.eye(4)])            # host depths
    with pytest.raises(ValueError):
        depth_metrics(d, d)                                                          # host tensors
    with pytest.raises(ValueError):
        depth_metrics(np.zeros((1, 4, 4), np.float32), np.zeros((1, 4, 4), np.float32))
