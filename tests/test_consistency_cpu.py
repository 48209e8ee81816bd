"""The multi-view consistency filter's statement (tests/refops_consistency.py) on analytic clips and hand-made cases, its
effect on fusion, the host helpers (`sequence_sources`, the refusals of `filter_depths`, `depth_points` and
`DepthFusionRunner`) and the C entries' argument checks, all without a GPU."""
import ctypes
import math

import numpy as np
import pytest
import torch

import refops_consistency as RC
import refops_fusion as RF
from unimatch_b200 import ops
from unimatch_b200.fusion import _consistency_args, depth_points, filter_depths, sequence_sources
from unimatch_b200.inference import _camera_to_world, _world_to_camera

U32 = 2.0 ** -24                     # float32 unit roundoff


def _rows(P):
    ps = [np.asarray(p, np.float32) for p in P]
    return _camera_to_world(ps), _world_to_camera(ps)


def _second_difference(D):
    """The largest |second difference| of the valid depths along x and along y (both neighbours valid)"""
    ok = D > 0
    ddx = np.abs(D[:, :, 2:] - 2 * D[:, :, 1:-1] + D[:, :, :-2])[ok[:, :, 2:] & ok[:, :, 1:-1] & ok[:, :, :-2]]
    ddy = np.abs(D[:, 2:] - 2 * D[:, 1:-1] + D[:, :-2])[ok[:, 2:] & ok[:, 1:-1] & ok[:, :-2]]
    return float(ddx.max()), float(ddy.max())


@pytest.mark.parametrize("name", ["sphere", "tilted"])
def test_exact_depths_are_consistent_wherever_the_taps_are_valid(name):
    """Bilinear interpolation of a C2 function on a unit cell errs by at most (ax (1 - ax) M_xx + ay (1 - ay) M_yy) / 2
    <= (M_xx + M_yy) / 8, M the largest second derivatives over the cell; on these smooth surfaces the second difference
    over the pixel grid bounds them up to a factor 2, which we allow.  With the float32 storage of the taps (half an ulp
    of the depth) the sampled source depth errs by e <= (M_xx + M_yy) / 4 + d_max 2^-24.  That moves the back-projected
    point by at most e |r_s| along the source ray (|r_s| = |((u - cx) / fx, (v - cy) / fy, 1)| <= R), so its reference
    depth by at most e R and its reprojection by at most f e R (1 + R) / z_min per axis (the projection's Jacobian
    f / z (I, -x / z) with |x / z| <= R).  The bounds below are far inside 1 px and 1 %, so every pixel whose four taps
    in a source are valid must be consistent with it (the exact reprojection of an exact depth has no error, and the
    float32 pipeline adds far less than the margin: see test_float32_against_float64)."""
    D, K, P, _ = RC.clip_depths(name)
    c2w, w2c = _rows(P)
    n, h, w = D.shape
    mxx, myy = _second_difference(D)
    e = (mxx + myy) / 4 + float(D.max()) * U32
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    R = math.sqrt(max(cx, w - 1 - cx) ** 2 / fx ** 2 + max(cy, h - 1 - cy) ** 2 / fy ** 2 + 1)
    z_min = float(D[D > 0].min()) * 0.9                     # the reference depth of the moved point, with room
    px_bound = math.sqrt(2) * max(fx, fy) * e * R * (1 + R) / z_min
    rel_bound = e * R / z_min
    assert px_bound < 0.5 and rel_bound < 0.005
    checked = 0
    for r in range(n):
        for s in range(n):
            if r != s:
                ok, taps = RC.source_check(D, c2w, w2c, K, r, s)
                assert np.array_equal(ok, taps), (r, s)
                checked += taps.sum()
    assert checked > 0.5 * n * (n - 1) * h * w                # the frames overlap by more than half


def test_occluded_pixels_are_not_consistent():
    """Corner clip: a reference pixel on a wall or the floor whose point is hidden from a source by the sphere, with all
    four of its taps there on the sphere at under 97 % of the point's source depth, samples a depth at least 3 % short;
    with camera baselines of centimetres the source ray is within a few degrees of the reference ray, so
    back-projecting it misses the reference depth by about 3 %, three times the 1 % allowed."""
    D, K, P, scenes = RC.clip_depths("corner", n=8)
    c2w, w2c = _rows(P)
    n, h, w = D.shape
    sphere = scenes[-1]
    fx, fy, cx, cy = (float(v) for v in (K[0, 0], K[1, 1], K[0, 2], K[1, 2]))
    ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    found = 0
    for r in range(n):
        X = RF.rays(K, h, w) @ P[r, :3, :3].T.astype(np.float64) * D[r][..., None] + P[r, :3, 3]
        on_sphere = np.abs(RF.distance(sphere, X)) < 1e-6
        for s in range(n):
            if s == r:
                continue
            Pi = np.linalg.inv(P[s].astype(np.float64))
            c = X @ Pi[:3, :3].T + Pi[:3, 3]
            u, v = fx * c[..., 0] / c[..., 2] + cx, fy * c[..., 1] / c[..., 2] + cy
            inside = (u >= 0) & (u <= w - 1) & (v >= 0) & (v <= h - 1) & (D[r] > 0)
            x0 = np.clip(np.floor(u), 0, w - 1).astype(int)
            y0 = np.clip(np.floor(v), 0, h - 1).astype(int)
            x1, y1 = np.minimum(x0 + 1, w - 1), np.minimum(y0 + 1, h - 1)
            taps = np.stack([D[s][y0, x0], D[s][y0, x1], D[s][y1, x0], D[s][y1, x1]])
            hidden = inside & ~on_sphere & (taps < 0.97 * c[..., 2]).all(0) & (taps > 0).all(0)
            ok, _ = RC.source_check(D, c2w, w2c, K, r, s)
            assert not (ok & hidden).any()
            found += hidden.sum()
    assert found > 30


def test_corrupted_depths_are_removed():
    """Corner clip with 2 % outliers (uniform in [0.5, 4] m) and an 8 x 8 patch per frame scaled by 1.3, filtered with
    two sources on each side and min_views 2.  A corrupted pixel is kept only if two sources agree with it to 1 % of
    depth, which for an outlier needs its value within about 1 % of the true depth d: probability at most
    2 (0.01 + 1e-3) d_max / 3.5 < 1.7 % with d_max = 2.6 m.  A scaled patch agrees only with another frame's patch over
    the same points.  So at most 2 % of the corrupted pixels may stay, and every one that stays is within 2 % of the
    true depth (a clean source bounds it to 1 % plus the interpolation error)."""
    D, K, P, _ = RC.clip_depths("corner", n=8)
    assert D.max() < 2.6
    Dc, mask = RC.corrupt(D, seed=0)
    c2w, w2c = _rows(P)
    views, f = RC.consistency(Dc, c2w, w2c, K, range(8), sequence_sources(8, 2, 2))
    kept = (f > 0) & mask
    assert mask.sum() > 500
    assert kept.sum() <= 0.02 * mask.sum()
    assert (np.abs(Dc - D)[kept] / D[kept]).max(initial=0) < 0.02
    clean = (D > 0) & ~mask
    assert ((f > 0) & clean).sum() >= 0.7 * clean.sum()


def test_filtering_removes_the_floaters_from_fusion():
    """Fusing the corrupted corner clip: extracted points more than two voxels from the true surface (floaters) drop by
    at least an order of magnitude with the filter, and the filter keeps at least 90 % of the near-surface points that
    fusing the exact depths gives."""
    D, K, P, scenes = RC.clip_depths("corner", n=8)
    Dc, _ = RC.corrupt(D, seed=0)
    c2w, w2c = _rows(P)
    _, f = RC.consistency(Dc, c2w, w2c, K, range(8), sequence_sources(8, 2, 2))
    origin, vs, dims = (-0.6, -0.45, 1.3), 0.02, (70, 53, 58)
    frames = np.zeros(D.shape + (3,), np.uint8)

    def fused(d):
        vol = RF.integrate(RF.empty_volume(dims), origin, vs, 4 * vs, d, frames, w2c, K)
        p, _ = RF.extract(vol, origin, vs)
        dist = np.min(np.stack([RF.distance(s, p) for s in scenes]), 0)
        return (dist > 2 * vs).sum(), (dist <= 2 * vs).sum()

    far_raw, _ = fused(Dc)
    far_filtered, near_filtered = fused(f)
    _, near_clean = fused(D)
    assert far_raw >= 100 and 10 * far_filtered <= far_raw
    assert near_filtered >= 0.9 * near_clean


# ---- hand-made cases ------------------------------------------------------------------------------------------------
K1 = np.array([[4.0, 0, 1.5], [0, 4.0, 1.5], [0, 0, 1]], np.float32)


def _pair(d_ref, d_src, src_pose):
    D = np.stack([d_ref, d_src]).astype(np.float32)
    return D, _rows([np.eye(4), src_pose])


def _shift(x=0.0, y=0.0, z=0.0):
    P = np.eye(4)
    P[:3, 3] = (x, y, z)
    return P


def test_behind_the_camera_outside_the_frame_and_the_last_row():
    flat = np.full((4, 4), 2.0)
    back = RF.pose(RF.rot("y", math.pi), [0.0, 0.0, 4.0])          # looks back at the plane from behind it: c.z > 0 ...
    D, (c2w, w2c) = _pair(flat, flat, RF.pose(RF.rot("y", math.pi), [0.0, 0.0, 0.0]))
    ok, taps = RC.source_check(D, c2w, w2c, K1, 0, 1)
    assert not taps.any()                                       # ... this one looks away: every point has c.z < 0
    D, (c2w, w2c) = _pair(flat, flat, _shift(x=0.5))                # half a metre at 2 m: 1 px of 4 shifts off the frame
    ok, taps = RC.source_check(D, c2w, w2c, K1, 0, 1)
    assert not taps[:, 0].any() and taps[:, 1:].all() and ok[:, 1:].all()
    D, (c2w, w2c) = _pair(flat, flat, _shift())                     # same camera: u = x lands on the last column / row
    ok, taps = RC.source_check(D, c2w, w2c, K1, 0, 1)
    assert ok.all()
    del back


def test_an_invalid_tap_drops_the_source():
    flat = np.full((4, 4), 2.0)
    src = flat.copy()
    src[2, 2] = np.nan
    D, (c2w, w2c) = _pair(flat, src, _shift(x=0.25))               # u = x - 0.5: taps x - 1 and x, rows y and y + 1
    ok, taps = RC.source_check(D, c2w, w2c, K1, 0, 1)
    assert not taps[1:3, 2:4].any()                                 # the pixels whose taps include (2, 2)
    assert taps[0, 1:].all() and taps[3, 1:].all() and ok[0, 1:].all()
    assert not taps[:, 0].any()                                     # u = -0.5 is outside


def test_table_entries_and_min_views_boundaries():
    flat = np.full((3, 4, 4), 2.0, np.float32)
    c2w, w2c = _rows([np.eye(4)] * 3)
    table = [[1, 2, -1, 7], [0, -1, -1, -1], [0, 0, 1, 1]]
    for m, want in ((1, [True, True, True]), (2, [True, False, True]), (3, [False, False, True]),
                    (4, [False, False, True])):
        views, out = RC.consistency(flat, c2w, w2c, K1, range(3), table, min_views=m)
        assert [int(views[i].min()) for i in range(3)] == [2, 1, 4]      # -1 and 7 are no source; duplicates count twice
        assert [bool((views[i] >= m).all()) for i in range(3)] == want
        assert all(np.array_equal(out[i], np.where(views[i] >= m, flat[i], 0)) for i in range(3))
    views, _ = RC.consistency(flat, c2w, w2c, K1, [5, -1], [[0, 1], [0, 1]], min_views=1)
    assert not views.any()                                          # references outside [0, n) have no valid depth


def test_float32_against_float64():
    """Per source, the float32 statement's reprojection error and relative depth difference against float64's, on the
    three clips.  Each is some 40 float32 operations on coordinates below 2 w and depths below 3 m with a coefficient
    chain of magnitude f R (1 + R) / z <= 300: 40 x 2^-24 x 300 ~ 7e-4 px, and 40 x 2^-24 ~ 2.4e-6 in the ratio.  The
    decisions agree wherever float64 is further than that from a threshold."""
    for name in ("sphere", "tilted", "corner"):
        D, K, P, _ = RC.clip_depths(name)
        c2w, w2c = _rows(P)
        for r, s in ((0, 1), (2, 4), (3, 0)):
            o32, t32, e32, r32 = RC.source_check(D, c2w, w2c, K, r, s, details=True)
            o64, t64, e64, r64 = RC.source_check(D, c2w, w2c, K, r, s, dtype=np.float64, details=True)
            both = t32 & t64 & np.isfinite(e64)
            assert np.abs(e32 - e64)[both].max(initial=0) <= 7e-4
            assert np.abs(r32 - r64)[both].max(initial=0) <= 2.4e-6
            clear = both & (np.abs(e64 - 1.0) > 7e-4) & (np.abs(r64 - 0.01) > 2.4e-6)
            assert np.array_equal(o32[clear], o64[clear])
            assert (t32 != t64).sum() <= 0.001 * t64.size      # only a tap bound met to the last bit may differ


def test_points_statement_back_projects_along_the_pixel_rays():
    D, K, P, scenes = RC.clip_depths("sphere")
    pts, cols = RC.points(D, np.zeros(D.shape + (3,), np.uint8), _rows(P)[0], K)
    assert pts.shape == ((D > 0).sum(), 3)
    assert RF.distance(scenes[0], pts.astype(np.float64)).max() < 1e-5


# ---- host helpers and refusals --------------------------------------------------------------------------------------
def test_sequence_sources():
    for n, b, a in ((1, 2, 2), (5, 2, 0), (5, 0, 3), (7, 3, 2), (0, 2, 2)):
        got = sequence_sources(n, b, a)
        assert got.dtype == np.int32 and got.shape == (n, b + a)
        assert np.array_equal(got, RC.sequence_sources(n, b, a))
    assert sequence_sources(4, 2, 1).tolist() == [[-1, -1, 1], [0, -1, 2], [1, 0, 3], [2, 1, -1]]
    with pytest.raises(ValueError):
        sequence_sources(4, -1, 0)


def test_consistency_arguments_are_checked():
    good = sequence_sources(4, 1, 1)
    src, mp, mr, mv = _consistency_args(4, good, 1.0, 0.01, 2, "f")
    assert src.dtype == np.int32 and (mp, mr, mv) == (1.0, float(np.float32(0.01)), 2)
    for bad, match in ((np.array([[0, 1]] * 4), "own source"), (np.array([[1], [2], [3], [4]]), r"\[-1, 4\)"),
                       (np.array([[-2], [0], [1], [2]]), r"\[-1, 4\)"), (np.zeros((4, 0), np.int32), "1 .. 255"),
                       (np.ones((4, 256), np.int32), "1 .. 255"), (np.zeros((3, 1), np.int32), "one row"),
                       (np.zeros((4, 1)), "integer")):
        with pytest.raises(ValueError, match=match):
            _consistency_args(4, bad, 1.0, 0.01, 1, "f")
    for kw, match in (({"max_pixel": 0.0}, "max_pixel"), ({"max_pixel": float("inf")}, "max_pixel"),
                      ({"max_relative": 1e-46}, "max_relative"), ({"max_relative": -1.0}, "max_relative"),
                      ({"min_views": 0}, "min_views"), ({"min_views": 3}, "min_views"), ({"min_views": True}, "min_views")):
        args = dict(max_pixel=1.0, max_relative=0.01, min_views=2)
        args.update(kw)
        with pytest.raises(ValueError, match=match):
            _consistency_args(4, good, args["max_pixel"], args["max_relative"], args["min_views"], "f")


def test_public_functions_refuse_bad_inputs(monkeypatch):
    class FakeDepth:                                    # passes the device checks without a GPU
        is_cuda, dtype, shape, device = True, torch.float32, (2, 8, 8), torch.device("cuda", 0)

        def dim(self):
            return 3

    import unimatch_b200.fusion as fusion
    real = torch.is_tensor
    monkeypatch.setattr(fusion.torch, "is_tensor", lambda t: isinstance(t, FakeDepth) or real(t))
    d, K = FakeDepth(), np.array([[10.0, 0, 4], [0, 10.0, 4], [0, 0, 1]])
    src = sequence_sources(2, 1, 0)
    with pytest.raises(ValueError, match="depths"):
        filter_depths(np.zeros((2, 8, 8), np.float32), K, [np.eye(4)] * 2, src)
    with pytest.raises(ValueError, match="poses"):
        filter_depths(d, K, [np.eye(4)], src)
    with pytest.raises(ValueError, match="finite"):
        filter_depths(d, K, [np.eye(4), np.full((4, 4), np.nan)], src)
    with pytest.raises(ValueError, match="fx"):
        filter_depths(d, np.diag([0.0, 1.0, 1.0]), [np.eye(4)] * 2, src)
    with pytest.raises(ValueError, match="own source"):
        filter_depths(d, K, [np.eye(4)] * 2, [[0], [0]], min_views=1)
    with pytest.raises(ValueError, match="min_views"):
        filter_depths(d, K, [np.eye(4)] * 2, src)
    with pytest.raises(ValueError, match="frames"):
        depth_points(d, np.zeros((2, 8, 8, 3), np.uint8), K, [np.eye(4)] * 2)


def test_runner_options_are_checked():
    from unimatch_b200.inference import DepthFusionRunner
    for kw, match in (({"consistency_views": -1}, "consistency_views"), ({"consistency_views": 256}, "consistency_views"),
                      ({"consistency_views": 2.0}, "consistency_views"),
                      ({"consistency_views": 2, "consistency_min_views": 3}, "consistency_min_views"),
                      ({"consistency_views": 2, "consistency_min_views": 0}, "consistency_min_views")):
        with pytest.raises(ValueError, match=match):
            DepthFusionRunner(None, (8, 8), 1, "cuda", np.eye(3), None, **kw)


def test_c_entries_check_arguments_without_a_gpu():
    p = [ctypes.c_void_p(4096 * (i + 1)) for i in range(12)]
    err = ops.LIB.um_last_error
    a = dict(depth=p[0], n=2, h=4, w=4, fx=1.0, fy=1.0, cx=0.0, cy=0.0, c2w=p[1], w2c=p[2], refs=p[3], r=2, src=p[4], s=1,
             mp=1.0, mr=0.01, mv=1, views=p[5], out=p[6])

    def cons(**kw):
        b = dict(a, **kw)
        return ops.LIB.um_depth_consistency(*b.values(), None)

    assert cons(depth=None) == -22 and b"NULL" in err()
    assert cons(n=0) == -22 and b"bad depths" in err()
    assert cons(h=0) == -22 and b"bad depths" in err()
    assert cons(r=0) == -22 and b"reference count" in err()
    assert cons(s=0) == -22 and b"source count" in err()
    assert cons(s=256, mv=1) == -22 and b"source count" in err()
    assert cons(mv=0) == -22 and b"min_views" in err()
    assert cons(mv=2) == -22 and b"min_views" in err()
    assert cons(mp=0.0) == -22 and b"max_pixel" in err()
    assert cons(mr=float("nan")) == -22 and b"max_relative" in err()
    assert cons(mp=float("inf")) == -22 and b"max_pixel" in err()
    assert cons(fx=0.0) == -22 and b"fx" in err()
    assert cons(refs=ctypes.c_void_p(4 * 4096 + 2)) == -22 and b"aligned" in err()
    assert cons(out=ctypes.c_void_p(4096 + 8)) == -22 and b"overlap" in err()
    assert cons(views=p[6]) == -22 and b"overlap" in err()
    assert ops.LIB.um_depth_points_count(None, 1, 4, 4, p[1], None) == -22 and b"NULL" in err()
    assert ops.LIB.um_depth_points_count(p[0], 0, 4, 4, p[1], None) == -22 and b"bad depths" in err()
    assert ops.LIB.um_depth_points_count(p[0], 1, 4, 4, ctypes.c_void_p(2 * 4096 + 4), None) == -22 and b"aligned" in err()
    assert ops.LIB.um_depth_points_count(p[0], 1, 4, 4, ctypes.c_void_p(4096 + 8), None) == -22 and b"overlap" in err()

    def pts(**kw):
        b = dict(depth=p[0], frames=p[1], n=1, h=4, w=4, fx=1.0, fy=1.0, cx=0.0, cy=0.0, c2w=p[2], offsets=p[3], np_=3,
                 points=p[4], colors=p[5])
        b.update(kw)
        return ops.LIB.um_depth_points(*b.values(), None)

    assert pts(c2w=None) == -22 and b"NULL" in err()
    assert pts(points=None) == -22 and b"NULL" in err()
    assert pts(np_=17) == -22 and b"point count" in err()
    assert pts(fy=0.0) == -22 and b"fx" in err()
    assert pts(offsets=ctypes.c_void_p(4 * 4096 + 4)) == -22 and b"aligned" in err()
    assert pts(colors=ctypes.c_void_p(4096 * 5 + 4)) == -22 and b"overlap" in err()
