"""ICP tracking without a GPU: the statement (tests/refops_icp.py) on volumes fused from the exact depths of analytic scenes
(the corner clip recovers perturbed poses, the constant-plane clip is degenerate, an empty volume tracks nothing, and
track-then-fuse keeps a drifting clip's poses bounded), hand-made depth maps for the pyramid and normal rules, the
choice of min_pivot, and the argument checks of `TSDFVolume.track` and the C entries."""
import ctypes
import math

import numpy as np
import pytest
import torch

import refops_fusion as RF
import refops_icp as RI
from unimatch_b200 import ops
from unimatch_b200.fusion import ICP_MIN_INLIERS, ICP_MIN_PIVOT, TSDFVolume, icp_levels

H, W = 48, 64
CORNER_VS = 0.02
CORNER_BOX = ((-0.6, -0.45, 1.3), (70, 53, 58))          # 2 cm voxels around what the corner clip's cameras see


def _fuse(scenes, K, poses, origin, vs, dims, h=H, w=W):
    depths = np.stack([RI.render_union(scenes, K, P, h, w) for P in poses])
    frames = np.full(depths.shape + (3,), 128, np.uint8)
    w2c = np.stack([np.linalg.inv(P)[:3] for P in poses])
    return RF.integrate(RF.empty_volume(dims), origin, vs, 4 * vs, depths, frames, w2c, K), depths


def test_constants_match_the_statement():
    assert (ICP_MIN_INLIERS, ICP_MIN_PIVOT) == (RI.MIN_INLIERS, RI.MIN_PIVOT)
    assert (ops.ICP_TERMS, ops.ICP_STATE) == (RI.TERMS, RI.STATE)
    K = np.array([[50.0, 0, 31.7], [0, 40.0, 23.3], [0, 0, 1]], np.float32)
    assert [tuple(map(float, lv)) for lv in RI.levels(K, 48, 65, 3)] == [tuple(map(float, lv)) for lv in
                                                                        icp_levels(K, 48, 65, 3)]


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_corner_clip_recovers_perturbed_poses(dtype):
    """Each frame of the corner clip, fused from exact depths at 2 cm, is tracked from a pose moved by up to 2 cm and
    rotated by up to 2 degrees.  The bound: the fused surface is the exact one up to the render tests' depth bound
    (below one voxel: nearest-pixel footprint, truncation and secant error, tests/test_render_cpu.py).  A point-to-plane
    fit to the floor and the two walls, each offset along its normal by at most half that, moves the camera by at most
    the offsets along the three orthogonal normals, sqrt(3) / 2 voxel at worst, and rotates it by that over the
    scene's lever (about 1 m): we require half a voxel and half a degree, and every frame must end closer than it
    started."""
    scenes, K, poses = RI.corner_clip()
    origin, dims = CORNER_BOX
    vol, depths = _fuse(scenes, K, poses, origin, CORNER_VS, dims)
    assert (depths > 0).all()
    g = np.random.default_rng(0)
    start = np.stack([RI.perturb(P, g) for P in poses])
    out = RI.track(vol, origin, CORNER_VS, 4 * CORNER_VS, depths, K, start, dtype=dtype)
    assert out["tracked"].all()
    assert (out["inliers"] >= 0.3 * out["valid"]).all()
    for P, Q, T in zip(poses, start, out["T"]):
        dt0, dr0 = RI.pose_error(P, Q)
        dt, dr = RI.pose_error(P, T)
        assert dt <= CORNER_VS / 2 and dr <= 0.5, (dt, dr)
        assert dt < dt0 / 2 and dr < dr0 / 2
    assert (out["rmse"] < CORNER_VS / 4).all()


def test_min_pivot_separates_the_corner_from_a_plane():
    """min_pivot = 1e-2: the corner clip's smallest scaled pivot at its last solve is above 5e-2 on every frame; a plane
    leaves three unknowns unconstrained, so the constant-plane clip (axis-aligned normals) has zero pivots and the
    tilted-plane clip, whose fused normals bend only at the volume's edges, stays below 5e-3."""
    scenes, K, poses = RI.corner_clip()
    origin, dims = CORNER_BOX
    vol, depths = _fuse(scenes, K, poses, origin, CORNER_VS, dims)
    hist = []
    RI.track(vol, origin, CORNER_VS, 4 * CORNER_VS, depths, K, poses, history=hist)
    assert min(RI.scaled_pivots(S).min() for S in hist[-1][1]) > 5 * RI.MIN_PIVOT
    scene, Kt, pt = RF.tilted_plane_clip()
    o, d = (-0.35, -0.3, 1.05), (70, 60, 75)
    vt, dt = _fuse([scene], Kt, pt, o, 0.01, d)
    hist = []
    out = RI.track(vt, o, 0.01, 0.04, dt, Kt, pt, min_pivot=1e-9, history=hist)       # every step taken
    pivots = [np.nanmin(RI.scaled_pivots(S)) for S in hist[-1][1]]
    assert max(pivots) < RI.MIN_PIVOT / 2
    assert not RI.track(vt, o, 0.01, 0.04, dt, Kt, pt)["tracked"].any()


def test_constant_plane_is_degenerate():
    scene, K, poses = RF.constant_plane_clip()
    origin, dims, vs = (-0.3, -0.3, 0.903), (30, 30, 10), 0.02
    vol, depths = _fuse([scene], K, poses, origin, vs, dims, h=24, w=32)
    g = np.random.default_rng(1)
    start = np.stack([RI.perturb(P, g) for P in poses])
    out = RI.track(vol, origin, vs, 4 * vs, depths, K, start)
    assert not out["tracked"].any()
    assert (out["inliers"] > 0).all()
    assert np.array_equal(out["pose"], start.astype(np.float32))


def test_empty_volume_is_not_tracked():
    scenes, K, poses = RI.corner_clip(n=2)
    origin, dims = CORNER_BOX
    depths = np.stack([RI.render_union(scenes, K, P, H, W) for P in poses])
    out = RI.track(RF.empty_volume(dims), origin, CORNER_VS, 4 * CORNER_VS, depths, K, poses)
    assert not out["tracked"].any() and (out["inliers"] == 0).all() and (out["rmse"] == 0).all()
    assert np.array_equal(out["pose"], poses.astype(np.float32))


def test_track_then_fuse_bounds_a_drifting_clip():
    """The given poses of a 6-frame corner clip carry an accumulated random walk (0.8 cm and 0.8 degrees per frame).
    Fusing them as given lets the error grow with the walk; tracking each frame against the frames fused before it,
    with the carried correction C = T P^-1, and fusing it at the tracked pose keeps every frame within a voxel and a
    degree of the first frame's frame of reference."""
    scenes, K, poses = RI.corner_clip(n=6, seed=7)
    origin, dims = CORNER_BOX
    g = np.random.default_rng(2)
    drift, given = np.eye(4), []
    for P in poses:
        given.append(drift @ P)
        drift = RI.perturb(np.eye(4), g, 0.008, 0.8) @ drift
    given = np.stack(given)
    depths = np.stack([RI.render_union(scenes, K, P, H, W) for P in poses])
    frames = np.full((1, H, W, 3), 128, np.uint8)
    vol = RF.empty_volume(dims)
    C = np.eye(4)
    errors, plain = [], []
    for t in range(len(poses)):
        out = RI.track(vol, origin, CORNER_VS, 4 * CORNER_VS, depths[t:t + 1], K, given[t:t + 1], correction=C)
        T = out["T"][0]
        assert out["tracked"][0] == (t > 0)
        if out["tracked"][0]:
            C = RI.correction_after(T, given[t])
        w2c = RI.rigid_inverse_rows(T)[None].astype(np.float64)
        vol = RF.integrate(vol, origin, CORNER_VS, 4 * CORNER_VS, depths[t:t + 1], frames, w2c, K)
        errors.append(RI.pose_error(poses[t], T))
        plain.append(RI.pose_error(poses[t], given[t]))
    assert max(e[0] for e in errors) <= CORNER_VS and max(e[1] for e in errors) <= 1.0, errors
    assert plain[-1][0] > 2 * max(e[0] for e in errors[1:]) or plain[-1][1] > 2 * max(e[1] for e in errors[1:])


# ---- hand-made depth maps ---------------------------------------------------------------------------------------------
def test_pyramid_rule_on_a_4x4_map():
    """Blocks: all valid and within trunc (the mean); one depth beyond trunc of the smallest (left out); invalid depths
    (0, negative, NaN, inf; left out); nothing valid (0)."""
    d = np.array([[[1.0, 1.5, 2.0, 2.0],
                   [1.25, 1.75, 2.0, 3.5],
                   [0.0, -1.0, np.nan, np.inf],
                   [3.0, np.nan, 0.0, -np.inf]]], np.float32)
    out = RI.downsample(d, 1.0)
    assert out.shape == (1, 2, 2)
    assert out[0].tolist() == [[1.375, 2.0], [3.0, 0.0]]
    assert RI.downsample(d, 2.0)[0, 0, 1] == np.float32(9.5 / 4)
    odd = np.ones((1, 5, 7), np.float32)
    assert RI.downsample(odd, 1.0).shape == (1, 2, 3)


def test_normal_rule_on_a_4x4_map():
    """A plane z = 2 seen along its normal gives (0, 0, -1) (towards the camera); the last row and column and pixels
    next to an invalid depth get 0; a slanted plane gives its unit normal facing the camera."""
    d = np.full((1, 4, 4), 2.0, np.float32)
    d[0, 1, 2] = 0.0
    n = RI.normals(d, 2.0, 2.0, 1.5, 1.5)
    assert n[0, 0, 0].tolist() == [0.0, 0.0, -1.0]
    assert not n[0, 3].any() and not n[0, :, 3].any()
    assert not n[0, 1, 2].any() and not n[0, 1, 1].any() and not n[0, 0, 2].any()
    xs = np.arange(4, dtype=np.float64)
    slant = (2.0 / (1 - 0.5 * (xs - 1.5) / 2.0))[None, None, :].repeat(4, 1).astype(np.float32)    # z = 2 + 0.5 x
    ns = RI.normals(slant, 2.0, 2.0, 1.5, 1.5, dtype=np.float64)
    np.testing.assert_allclose(ns[0, :3, :3].reshape(-1, 3), np.broadcast_to(np.array([0.5, 0, -1]) / math.sqrt(1.25),
                                                                             (9, 3)), atol=1e-6)
    n32 = RI.normals(slant, 2.0, 2.0, 1.5, 1.5)
    assert n32.dtype == np.float32 and np.abs(n32 - ns).max() < 1e-6


def test_levels_follow_the_pixel_centre_convention():
    """A pixel-centre ray at level l + 1 is the mean of its 2 x 2 block's rays at level l"""
    K = np.array([[50.0, 0, 31.5], [0, 50.0, 23.5], [0, 0, 1]], np.float32)
    (fx, fy, cx, cy, h, w), (fx1, fy1, cx1, cy1, h1, w1) = RI.levels(K, 48, 64, 2)
    assert (h1, w1) == (24, 32) and (fx1, fy1) == (25.0, 25.0)
    x1 = 5
    assert (x1 - cx1) / fx1 == pytest.approx(((2 * x1 - cx) / fx + (2 * x1 + 1 - cx) / fx) / 2)


# ---- argument checks ------------------------------------------------------------------------------------------------
def test_track_arguments_are_checked(monkeypatch):
    vol = object.__new__(TSDFVolume)
    vol.device = torch.device("cuda", 0)
    K = np.array([[10.0, 0, 4], [0, 10.0, 4], [0, 0, 1]])

    class FakeDepth:                                    # passes the device checks without a GPU
        is_cuda, dtype, shape, device = True, torch.float32, (1, 16, 16), torch.device("cuda", 0)

        def dim(self):
            return 3

    import unimatch_b200.fusion as fusion
    real = torch.is_tensor
    monkeypatch.setattr(fusion.torch, "is_tensor", lambda t: isinstance(t, FakeDepth) or real(t))
    d = FakeDepth()
    with pytest.raises(ValueError, match="depths"):
        vol.track(np.zeros((1, 16, 16), np.float32), K, [np.eye(4)])
    with pytest.raises(ValueError, match="intrinsics"):
        vol.track(d, np.eye(4), [np.eye(4)])
    with pytest.raises(ValueError, match="poses"):
        vol.track(d, K, [np.eye(4), np.eye(4)])
    with pytest.raises(ValueError, match="finite"):
        vol.track(d, K, [np.full((4, 4), np.nan)])
    with pytest.raises(ValueError, match="levels"):
        vol.track(d, K, [np.eye(4)], levels=0)
    with pytest.raises(ValueError, match="iterations"):
        vol.track(d, K, [np.eye(4)], iterations=(1, 2))
    with pytest.raises(ValueError, match="iterations"):
        vol.track(d, K, [np.eye(4)], iterations=(1, 2, 0))
    with pytest.raises(ValueError, match="too small"):
        vol.track(d, K, [np.eye(4)], levels=5, iterations=(1, 1, 1, 1, 1))
    with pytest.raises(ValueError, match="max_distance"):
        vol.track(d, K, [np.eye(4)], max_distance=0.0)
    with pytest.raises(ValueError, match="max_distance"):
        vol.track(d, K, [np.eye(4)], max_distance=1e-46)         # positive, but 0 in float32
    with pytest.raises(ValueError, match="max_angle"):
        vol.track(d, K, [np.eye(4)], max_angle=float("nan"))
    with pytest.raises(ValueError, match="min_inlier_fraction"):
        vol.track(d, K, [np.eye(4)], min_inlier_fraction=1.5)
    with pytest.raises(ValueError, match="fx"):
        vol.track(d, np.diag([0.0, 1.0, 1.0]), [np.eye(4)])


def test_c_entries_check_arguments_without_a_gpu():
    p = [ctypes.c_void_p(4096 * (i + 1)) for i in range(12)]
    err = ops.LIB.um_last_error
    assert ops.LIB.um_icp_downsample(None, p[1], 1, 4, 4, 0.1, None) == -22
    assert b"NULL" in err()
    assert ops.LIB.um_icp_downsample(p[0], p[1], 1, 1, 4, 0.1, None) == -22 and b"bad depths" in err()
    assert ops.LIB.um_icp_downsample(p[0], p[1], 1, 4, 4, 0.0, None) == -22 and b"trunc" in err()
    assert ops.LIB.um_icp_downsample(p[0], ctypes.c_void_p(4098), 1, 4, 4, 0.1, None) == -22 and b"aligned" in err()
    assert ops.LIB.um_icp_downsample(p[0], ctypes.c_void_p(4096 + 4), 1, 4, 4, 0.1, None) == -22 and b"overlap" in err()
    assert ops.LIB.um_icp_normals(p[0], p[1], 1, 4, 4, 0.0, 1.0, 0.0, 0.0, None) == -22 and b"fx" in err()
    assert ops.LIB.um_icp_normals(p[0], p[1], 0, 4, 4, 1.0, 1.0, 0.0, 0.0, None) == -22 and b"bad depths" in err()
    assert ops.LIB.um_icp_init(p[0], None, 1, None, p[2], p[3], p[4], None) == -22 and b"NULL" in err()
    assert ops.LIB.um_icp_init(p[0], None, 0, p[1], p[2], p[3], p[4], None) == -22 and b"frame count" in err()
    assert ops.LIB.um_icp_init(p[0], ctypes.c_void_p(4100), 1, p[1], p[2], p[3], p[4], None) == -22 and b"aligned" in err()
    assert ops.LIB.um_icp_init(p[0], None, 1, p[1], p[2], p[2], p[4], None) == -22 and b"overlap" in err()

    def reduce(**kw):
        a = dict(n=1, h=8, w=16, fx=1.0, md=0.1, cos=0.9, partials=p[9])
        a.update(kw)
        return ops.LIB.um_icp_reduce(*p[:7], a["n"], a["h"], a["w"], a["fx"], 1.0, 0.0, 0.0, a["md"], a["cos"], p[7],
                                     a["partials"], None)

    assert reduce(n=0) == -22 and b"bad frames" in err()
    assert reduce(fx=float("inf")) == -22 and b"fx" in err()
    assert reduce(md=0.0) == -22 and b"max_distance" in err() and reduce(cos=1.5) == -22
    assert reduce(partials=ctypes.c_void_p(9 * 4096 + 4)) == -22 and b"aligned" in err()
    assert reduce(partials=p[0]) == -22 and b"overlap" in err()
    assert ops.LIB.um_icp_solve(p[0], 0, 1, p[1], 36.0, 1e-2, 1, p[2], None) == -22 and b"bad partials" in err()
    assert ops.LIB.um_icp_solve(p[0], 1, 1, p[1], 36.0, 0.0, 1, p[2], None) == -22 and b"min_pivot" in err()
    assert ops.LIB.um_icp_solve(p[0], 1, 1, p[1], -1.0, 1e-2, 1, p[2], None) == -22 and b"min_inliers" in err()
    assert ops.LIB.um_icp_solve(p[0], 1, 1, p[1], 36.0, 1e-2, 1, p[0], None) == -22 and b"overlap" in err()
    acc = [p[0], 1, 1, p[1], 0.3, None, None, p[2], p[3], p[4], p[5], p[6], p[7], None]
    bad = list(acc)
    bad[6] = p[8]
    assert ops.LIB.um_icp_accept(*bad) == -22 and b"correction" in err()
    bad = list(acc)
    bad[4] = 1.5
    assert ops.LIB.um_icp_accept(*bad) == -22 and b"min_inlier_fraction" in err()
    bad = list(acc)
    bad[9] = p[8]
    bad[10] = ctypes.c_void_p(8 * 4096 + 4)
    assert ops.LIB.um_icp_accept(*bad) == -22 and b"aligned" in err()
    bad = list(acc)
    bad[12] = p[3]
    assert ops.LIB.um_icp_accept(*bad) == -22 and b"overlap" in err()
