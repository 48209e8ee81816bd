"""TSDF fusion without a GPU: the float64 statement (tests/refops_fusion.py) on analytic scenes seen from rotated cameras and on
hand-made single-voxel cases, `covering_box`, the world-to-camera helper, the PLY writer, and argument checks."""
import ctypes

import numpy as np
import pytest
import torch

import refops_fusion as RF
from unimatch_b200 import ops
from unimatch_b200.fusion import MAX_VOXELS, TSDFVolume, covering_box, fuse_depths, write_ply
from unimatch_b200.inference import DepthFusionRunner, _relative_poses, _world_to_camera

H, W = 24, 32


def _fuse64(scene, K, poses, origin, vs, dims, trunc=None, h=H, w=W):
    trunc = 4 * vs if trunc is None else trunc
    depths = np.stack([RF.render(scene, K, P, h, w) for P in poses])
    frames = np.full((len(poses), h, w, 3), 128, np.uint8)
    w2c = np.stack([np.linalg.inv(P)[:3] for P in poses])
    vol = RF.integrate(RF.empty_volume(dims), origin, vs, trunc, depths, frames, w2c, K)
    return vol, RF.extract(vol, origin, vs)


def test_constant_depth_plane_points_lie_on_the_plane():
    """Cameras rolled about their optical axis (world +z) and moved parallel to the plane z = 1 see the constant depth
    1.5, so every voxel's TSDF is exactly linear in z and the zero crossings lie on the plane."""
    scene, K, poses = RF.constant_plane_clip()
    assert all(np.ptp(RF.render(scene, K, P, H, W)) == 0 for P in poses)
    vs = 0.02
    origin, dims = (-0.3, -0.3, 0.903), (30, 30, 10)
    vol, (pts, cols) = _fuse64(scene, K, poses, origin, vs, dims)
    assert len(pts) == 30 * 30                  # one z-edge crossing per column, no x / y crossing
    assert np.abs(pts[:, 2] - 1.0).max() <= 1e-6 * vs
    assert (cols == 128).all()
    assert (vol["weight"] == len(poses)).sum() > 0


def _tolerance(scene, K, poses, vs, lo, hi, h, w):
    """Bound on the distance of an extracted point to the surface.

    Frame k's projective difference sdf_k(p) = d_k(nearest pixel) - z_k(p) of a voxel p near the surface is
    a_k dist(p) + e_k(p): a_k = cos(beta) / cos(phi) (ray to optical axis, ray to normal) is the factor by which a z-depth
    difference along the ray exceeds the Euclidean distance, and |e_k| <= E, the largest change of the depth within half a
    pixel of a pixel centre (RF.footprint_error).  The fused TSDF, away from the truncation (|sdf| <= a_max vs + E < trunc on
    every crossing edge, checked below), is mean_k(a_k) dist + mean_k(e_k) at each end of an edge, so where its linear
    interpolation vanishes, |dist| <= E / a_min from the e terms, plus at most vs (a_max - a_min) / (4 a_min) where the two
    ends average different frames' a_k (d0 d1 (a0 - a1) / (a0 d0 - a1 d1) with d0 d1 < 0 and |d0| + |d1| <= vs), plus
    the sagitta vs^2 / (8 R) of a sphere of radius R over one edge.  10 % covers the second-order terms (the projective
    factor changes by about vs / depth across an edge)."""
    E, a_lo, a_hi = RF.footprint_error(scene, K, poses, h, w, lo, hi)
    sag = vs * vs / (8 * scene[2]) if scene[0] == "sphere" else 0.0
    assert a_hi * vs + E < 4 * vs
    return 1.1 * (E / a_lo + vs * (a_hi - a_lo) / (4 * a_lo) + sag)


@pytest.mark.parametrize("clip", ["tilted_plane", "sphere"])
def test_rotated_cameras_points_lie_within_the_footprint_bound(clip):
    scene, K, poses = getattr(RF, clip + "_clip")()
    vs = 0.01
    origin, dims = covering_scene(scene)
    vol, (pts, _) = _fuse64(scene, K, poses, origin, vs, dims, h=48, w=64)
    lo = np.array(origin) - 4 * vs
    hi = np.array(origin) + np.array(dims) * vs + 4 * vs
    tol = _tolerance(scene, K, poses, vs, lo, hi, 48, 64)
    assert len(pts) > 1000
    err = RF.distance(scene, pts)
    assert err.max() <= tol, (err.max(), tol)
    assert tol < vs


def covering_scene(scene):
    """A 1 cm volume around the part of the scene the clips see"""
    if scene[0] == "plane":
        return (-0.35, -0.3, 1.05), (70, 60, 75)
    return (-0.3, -0.25, 1.0), (60, 50, 40)


# ---- hand-made single voxels --------------------------------------------------------------------------------------------
K1 = [[2.0, 0, 1.0], [0, 2.0, 1.0], [0, 0, 1]]               # 3 x 3 frames; the optical axis meets pixel (1, 1)
VS, TR = 0.125, 0.5                                           # exact in binary: the voxel centre is exactly (0, 0, z)


def _one(z, depths, rgb=None, w2c=None, trunc=TR):
    """Fuses 3 x 3 frames, each of constant depth depths[t], into the one voxel centred at (0, 0, z)"""
    n = len(depths)
    d = np.stack([np.full((3, 3), v, np.float64) for v in depths])
    fr = np.zeros((n, 3, 3, 3), np.uint8) if rgb is None else np.stack([np.broadcast_to(np.uint8(c), (3, 3, 3)) for c in rgb])
    w2c = np.stack([np.eye(4)[:3]] * n) if w2c is None else w2c
    vol = RF.integrate(RF.empty_volume((1, 1, 1)), (-VS / 2, -VS / 2, z - VS / 2), VS, trunc, d, fr, w2c, K1)
    return vol["tsdf"].item(), vol["weight"].item(), vol["color"][:, 0, 0, 0]


def test_single_voxel_truncation_and_cut():
    f, wt, _ = _one(1.0, [3.0])                                                 # sdf 2 > trunc: truncated to 1
    assert (f, wt) == (1.0, 1.0)
    f, wt, _ = _one(1.0, [1.25])
    assert (f, wt) == (0.5, 1.0)
    f, wt, _ = _one(1.0, [1.0 - TR])                                            # sdf = -trunc: kept
    assert (f, wt) == (-1.0, 1.0)
    assert _one(1.0, [1.0 - TR - 1e-6])[1] == 0                                 # behind the surface by more than trunc


@pytest.mark.parametrize("d", [0.0, -1.0, float("nan"), float("inf"), float("-inf")])
def test_single_voxel_invalid_depths_are_skipped(d):
    assert _one(1.0, [d])[1] == 0


def test_single_voxel_behind_the_camera_or_outside_the_frame():
    assert _one(-1.0, [1.0])[1] == 0                                            # c.z < 0
    assert _one(0.0, [1.0])[1] == 0                                             # c.z = 0
    shift = np.stack([np.hstack([np.eye(3), [[1.0], [0], [0]]])])               # moves the voxel to u = 1 + 2 * 1 = 3
    assert _one(1.0, [1.2], w2c=shift)[1] == 0
    half = np.stack([np.hstack([np.eye(3), [[0.74], [0], [0]]])])               # u = 2.48 -> pixel 2: inside
    assert _one(1.0, [1.2], w2c=half)[1] == 1
    # half-way points round up: u = 2.5 -> pixel 3 (outside), u = -0.5 -> pixel 0 (inside)
    assert _one(1.0, [1.2], w2c=shift * [1, 1, 1, 0.75])[1] == 0
    assert _one(1.0, [1.2], w2c=shift * [1, 1, 1, -0.75])[1] == 1


def test_single_voxel_weight_counting_and_colour_mean():
    f, wt, c = _one(1.0, [1.125, 0.0, 1.25, 1.375], rgb=[[30, 60, 90], [255, 255, 255], [60, 60, 60], [90, 0, 30]])
    assert wt == 3
    assert f == pytest.approx((0.25 + 0.5 + 0.75) / 3)
    np.testing.assert_allclose(c, [60, 40, 60])


def test_extraction_edges_order_and_colour():
    vol = RF.empty_volume((2, 2, 1))
    vol["tsdf"][0] = [[-0.5, 0.5], [0.25, 0.75]]
    vol["weight"][0] = [[1, 1], [1, 0]]
    vol["color"][:, 0, 0, 0] = [0, 100, 255]
    vol["color"][:, 0, 0, 1] = [100, 100, 0]
    vol["color"][:, 0, 1, 0] = [200, 0, 255]
    pts, cols = RF.extract(vol, (0, 0, 0), 0.1)
    # voxel (0,0): +x edge to 0.5 at s = 0.5, +y edge to 0.25 at s = 2/3; voxel (1,0)'s +y neighbour has weight 0
    np.testing.assert_allclose(pts, [[0.1, 0.05, 0.05], [0.05, 0.05 + 0.1 * 2 / 3, 0.05]])
    np.testing.assert_array_equal(cols, [[50, 100, 128], [133, 33, 255]])


# ---- volume geometry, poses, files ------------------------------------------------------------------------------------
def test_covering_box_bounds():
    K = [[50.0, 0, 16], [0, 50.0, 12], [0, 0, 1]]
    origin, dims, trunc = covering_box(np.array(K), [np.eye(4)], (24, 32), 2.0, 0.05)
    assert trunc == pytest.approx(0.2)
    np.testing.assert_allclose(origin, [-16 / 50 * 2 - 0.2, -12 / 50 * 2 - 0.2, -0.2])
    extent = np.array([2 * 0.64 + 0.4, 2 * 0.48 + 0.4, 2.4])
    assert (np.array(dims) * 0.05 >= extent - 1e-12).all() and (np.array(dims) * 0.05 <= extent + 0.05 + 1e-6).all()
    _, _, poses = RF.tilted_plane_clip()
    origin, dims, trunc = covering_box(np.array(K), poses, (24, 32), 1.5, 0.02, trunc=0.1)
    lo, hi = np.array(origin), np.array(origin) + np.array(dims) * 0.02
    pts = []
    for P in poses.astype(np.float32).astype(np.float64):          # the poses as the box reads them
        for x, y in ((0, 0), (32, 0), (0, 24), (32, 24)):
            pts.append(P[:3, :3] @ np.array([(x - 16) / 50 * 1.5, (y - 12) / 50 * 1.5, 1.5]) + P[:3, 3])
        pts.append(P[:3, 3])
    pts = np.array(pts)
    np.testing.assert_allclose(pts.min(0), lo + 0.1, atol=1e-12)   # the low corner is the frusta's, padded by trunc
    assert (pts.max(0) <= hi - 0.1 + 1e-12).all() and (pts.max(0) > hi - 0.1 - 0.02).all()


def test_world_to_camera_is_numpy_float32_inverse():
    _, _, poses = RF.sphere_clip()
    p32 = [p.astype(np.float32) for p in poses]
    got = _world_to_camera(p32)
    assert got.dtype == np.float32 and got.shape == (len(p32), 3, 4) and got.flags["C_CONTIGUOUS"]
    for g, p in zip(got, p32):
        np.testing.assert_array_equal(g, np.linalg.inv(p)[:3])
    # the runner's relative poses are built from the same inverse
    rel = _relative_poses(p32[:2], False)[0]
    np.testing.assert_array_equal(rel, (np.linalg.inv(p32[1]) @ p32[0]).astype(np.float32))


def test_ply_round_trip(tmp_path):
    g = np.random.default_rng(3)
    pts = g.standard_normal((17, 3)).astype(np.float32)
    cols = g.integers(0, 256, (17, 3)).astype(np.uint8)
    path = tmp_path / "cloud.ply"
    write_ply(str(path), torch.from_numpy(pts), cols)
    data = path.read_bytes()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    header = data[:end].decode("ascii").splitlines()
    assert header == ["ply", "format binary_little_endian 1.0", "element vertex 17", "property float x",
                      "property float y", "property float z", "property uchar red", "property uchar green",
                      "property uchar blue", "end_header"]
    body = np.frombuffer(data[end:], dtype=[("xyz", "<f4", 3), ("rgb", "u1", 3)])
    assert len(body) == 17
    np.testing.assert_array_equal(body["xyz"], pts)
    np.testing.assert_array_equal(body["rgb"], cols)
    write_ply(str(path), np.zeros((0, 3), np.float32), np.zeros((0, 3), np.uint8))
    assert path.read_bytes().endswith(b"element vertex 0\nproperty float x\nproperty float y\nproperty float z\n"
                                      b"property uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n")


# ---- argument checks ------------------------------------------------------------------------------------------------
def test_volume_arguments_are_checked():
    with pytest.raises(ValueError, match="2\\^31"):
        TSDFVolume((0, 0, 0), 0.01, (2048, 2048, 512))
    assert 2047 * 2048 * 512 <= MAX_VOXELS
    with pytest.raises(ValueError, match="dims"):
        TSDFVolume((0, 0, 0), 0.01, (4, 0, 4))
    with pytest.raises(ValueError, match="voxel_size"):
        TSDFVolume((0, 0, 0), 0.0, (4, 4, 4))
    with pytest.raises(ValueError, match="trunc"):
        TSDFVolume((0, 0, 0), 0.01, (4, 4, 4), trunc=-1.0)
    with pytest.raises(ValueError, match="origin"):
        TSDFVolume((0, float("nan"), 0), 0.01, (4, 4, 4))
    with pytest.raises(ValueError, match="CUDA"):
        TSDFVolume((0, 0, 0), 0.01, (4, 4, 4), device="cpu")
    with pytest.raises(ValueError, match="max_depth"):
        covering_box(np.eye(3), [np.eye(4)], (4, 4), 0.0, 0.01)


def test_fuse_depths_arguments_are_checked():
    vol = object.__new__(TSDFVolume)
    vol.device = torch.device("cuda", 0)
    d, f = torch.zeros((2, 4, 4)), torch.zeros((2, 4, 4, 3), dtype=torch.uint8)
    with pytest.raises(ValueError, match="TSDFVolume"):
        fuse_depths(object(), d, f, np.eye(3), [np.eye(4)] * 2)
    with pytest.raises(ValueError, match="device float32"):
        fuse_depths(vol, d, f, np.eye(3), [np.eye(4)] * 2)          # host depths
    with pytest.raises(ValueError, match="device float32"):
        fuse_depths(vol, torch.zeros((4, 4)), f, np.eye(3), [np.eye(4)] * 2)


def test_runner_refuses_bidirectional_depth_and_other_volumes():
    vol = object.__new__(TSDFVolume)
    vol.device = torch.device("cuda", 0)
    with pytest.raises(ValueError, match="pred_bidir_depth.*twice"):
        DepthFusionRunner(None, (8, 8), 1, "cuda:0", np.eye(3), vol, pred_bidir_depth=True)
    with pytest.raises(ValueError, match="TSDFVolume"):
        DepthFusionRunner(None, (8, 8), 1, "cuda:0", np.eye(3), object())
    with pytest.raises(ValueError, match="device"):
        DepthFusionRunner(None, (8, 8), 1, "cuda:1", np.eye(3), vol)


def test_c_entries_check_arguments_without_a_gpu():
    one = ctypes.c_void_p(256)
    origin = (ctypes.c_float * 3)(0, 0, 0)
    rc = ops.LIB.um_tsdf_integrate(None, None, None, 4, 4, 4, origin, 0.1, 0.4, None, None, None, 1, 4, 4, 1, 1, 1, 1, None,
                                   None)
    assert rc == -22 and b"um_tsdf_integrate" in ops.LIB.um_last_error()
    rc = ops.LIB.um_tsdf_surface_count(one, one, 2048, 2048, 512, one, None)
    assert rc == -22 and b"2^31 - 1" in ops.LIB.um_last_error()
    rc = ops.LIB.um_tsdf_surface_points(one, one, one, 4, 4, 4, origin, -1.0, one, 0, None, None, None)
    assert rc == -22 and b"voxel_size" in ops.LIB.um_last_error()
