"""The TSDF ray cast without a GPU: the float64 statement (tests/refops_render.py) on volumes fused from the exact depths of
analytic scenes, rendered at their input poses and at held-out poses between them, against a depth bound derived from the
fusion's footprint; a plane at grazing incidence; hand-made 2 x 2 x 2 volumes; float32 against float64; argument checks."""
import ctypes
import math

import numpy as np
import pytest
import torch

import refops_fusion as RF
import refops_mesh as RM
import refops_render as RR
from test_fusion_cpu import _fuse64, covering_scene
from unimatch_b200 import ops
from unimatch_b200.fusion import TSDFVolume
from unimatch_b200.inference import _camera_to_world

H, W = 48, 64


def _between(poses):
    """Held-out poses half-way between consecutive ones: the mean centre, and the rotation nearest the mean rotation"""
    out = []
    for P, Q in zip(poses[:-1], poses[1:]):
        u, _, vt = np.linalg.svd(P[:3, :3] + Q[:3, :3])
        out.append(RF.pose(u @ vt, (P[:3, 3] + Q[:3, 3]) / 2))
    return np.stack(out)


def _render64(vol, origin, vs, trunc, poses, K, h=H, w=W, near=0.0, far=np.inf):
    return RR.raycast(vol, origin, vs, trunc, np.stack([P[:3] for P in poses]), K, h, w, near, far)


def _max_ray_length(K, h, w):
    """Largest |d| over the pixel-centre rays, d the direction with camera z-component 1"""
    return float(np.linalg.norm(RF.rays(K, h, w), axis=-1).max())


def _depth_bound(scene, K, fuse_poses, Kr, render_poses, vs, lo, hi, h, w, scale):
    """Bound on the depth error of a hit, for a volume fused from the exact depths of fuse_poses at scale x (h, w) pixels
    and rendered at render_poses with intrinsics Kr at h x w.

    As in test_fusion_cpu._tolerance, trunc * F at a voxel near the surface is the mean over the frames that saw it of
    a_k dist + e_k, with a_k in [a_lo, a_hi] (fusing cameras) and |e_k| <= E (RF.footprint_error), provided |sdf| < trunc
    there.  Trilinear interpolation instead of edge interpolation: the sample's value is sum_i w_i (a_i dist_i + e_i) over
    the cell's corners; with dist_i = dist + delta_i and sum_i w_i delta_i = 0 (trilinear weights reproduce linear
    functions), where it vanishes |dist| <= (E + |sum_i w_i (a_i - a_mid) delta_i|) / a_lo, and
    sum_i w_i |delta_i| <= vs / 2 per axis weighted by |n_a|, at most sqrt(3) vs / 2, so the a_k term is
    sqrt(3) vs (a_hi - a_lo) / (4 a_lo); a sphere of radius R adds trilinear interpolation's error vs^2 / 8 times the
    Hessian's trace 2 / r, r >= R - 3 vs near the surface.  Along a rendering ray a distance error moves the z-depth by
    b = cos(beta) / cos(phi) <= b_hi (rendering rays).  Fine-step refinement: the bracketing samples are at most vs / 2
    apart in t and both the secant's root and a zero of the interpolated field lie between them, which adds vs / 2.
    10 % covers second-order terms, 1e-9 voxel sizes the statement's float64 rounding."""
    E, a_lo, a_hi = RF.footprint_error(scene, K, fuse_poses, h * scale, w * scale, lo, hi)
    _, _, b_hi = RF.footprint_error(scene, Kr, render_poses, h, w, lo, hi)
    sag = vs * vs / (4 * (scene[2] - 3 * vs)) if scene[0] == "sphere" else 0.0
    zero = (E + math.sqrt(3) * vs * (a_hi - a_lo) / 4) / a_lo + sag
    return 1.1 * (b_hi * zero + vs / 2) + 1e-9 * vs


def _interior(scene, K, P, h, w, planes, origin, vs, margin=2):
    """Pixels whose exact surface point lies where every voxel within `margin` cells of it is inside the grid and
    observed, and the exact depths"""
    d = RF.render(scene, K, P, h, w)
    x = P[:3, 3] + (RF.rays(K, h, w) @ P[:3, :3].T) * d[..., None]
    g = np.floor((x - np.asarray(origin)) / vs - 0.5).astype(np.int64)
    Z, Y, X = planes["weight"].shape
    ok = d > 0
    for dz in range(-margin, margin + 2):
        for dy in range(-margin, margin + 2):
            for dx in range(-margin, margin + 2):
                i, j, k = g[..., 0] + dx, g[..., 1] + dy, g[..., 2] + dz
                inside = (i >= 0) & (i < X) & (j >= 0) & (j < Y) & (k >= 0) & (k < Z)
                seen = np.zeros(d.shape, bool)
                seen[inside] = planes["weight"][k[inside], j[inside], i[inside]] > 0
                ok &= seen
    return ok, d


NORMAL_DEGREES = 12.0      # the fused field's gradient, away from frustum edges, follows the surface normal this closely


@pytest.mark.parametrize("clip", ["constant_plane", "tilted_plane", "sphere"])
def test_fused_clips_render_within_the_derived_bound(clip):
    """Fused at 8 x the clip's resolution (for the rotated clips), which keeps the nearest-pixel footprint error E well
    below a voxel, and rendered at the clip's own resolution"""
    vs, trunc = 0.01, 0.04
    if clip == "constant_plane":
        h, w, scale = 24, 32, 1
        origin, dims = (-0.6, -0.6, 0.903), (120, 120, 20)
    else:
        h, w, scale = H, W, 8
    scene, K, poses = getattr(RF, clip + "_clip")(h=h * scale, w=w * scale)
    Kr = getattr(RF, clip + "_clip")(h=h, w=w)[1]
    if clip != "constant_plane":
        origin, dims = covering_scene(scene)
    vol, _ = _fuse64(scene, K, poses, origin, vs, dims, trunc, h=h * scale, w=w * scale)
    lo = np.array(origin) - trunc
    hi = np.array(origin) + np.array(dims) * vs + trunc
    for render_poses in (poses, _between(poses)):
        tol = _depth_bound(scene, K, poses, Kr, render_poses, vs, lo, hi, h, w, scale)
        assert tol < vs
        depth, color, normal = _render64(vol, origin, vs, trunc, render_poses, Kr, h, w)
        n_interior = 0
        for v, P in enumerate(render_poses):
            inner, exact = _interior(scene, Kr, P, h, w, vol, origin, vs)
            n_interior += inner.sum()
            assert (depth[v][inner] > 0).all()                           # every interior pixel is a hit
            hit = depth[v] > 0
            assert not (hit & (exact == 0)).any()
            assert np.abs(depth[v] - exact)[hit].max() <= tol
            r = RF.rays(Kr, h, w) @ P[:3, :3].T
            nrm = RF.normal_at(scene, P[:3, 3] + r * exact[..., None])
            nrm = nrm * -np.sign((nrm * r).sum(-1, keepdims=True))          # towards the camera: free space
            cos = (normal[v] * nrm).sum(-1)[inner]
            assert cos.min() >= math.cos(math.radians(NORMAL_DEGREES)), math.degrees(math.acos(cos.min()))
            assert (color[v][hit] == 128).all()
        assert n_interior > 0.1 * len(render_poses) * h * w


def test_grazing_plane_misses_no_crossing():
    """The plane z = 1, free space below it (an exact truncated SDF), seen from below at up to about 80 degrees
    incidence: every ray meeting it inside the observed slab is a hit, at the exact depth (trilinear interpolation and the
    secant are exact on a linear field), and coarse steps cross the free space."""
    vs, trunc = 0.02, 0.08
    origin, dims = (-1.0, -1.0, 0.8), (150, 100, 20)
    planes = RM.sdf_volume(lambda x: 1.0 - x[..., 2], origin, vs, dims, trunc)
    K = [[40.0, 0, 16.0], [0, 40.0, 12.0], [0, 0, 1]]
    P = RF.pose(RF.rot("y", math.radians(80)), [-1.2, 0.0, 0.95 - 2.2 * math.cos(math.radians(80))])
    scene = ("plane", [0.0, 0.0, 1.0], 1.0)
    depth, _, normal, n = RR.raycast(planes, origin, vs, trunc, P[None, :3], K, 24, 32, counts=True)
    inner, exact = _interior(scene, K, P, 24, 32, planes, origin, vs)
    assert inner.sum() > 100
    r = RF.rays(K, 24, 32) @ P[:3, :3].T
    cos_inc = np.abs(r[..., 2]) / np.linalg.norm(r, axis=-1)
    assert math.degrees(math.acos(cos_inc[inner].min())) > 75                 # grazing
    assert (depth[0][inner] > 0).all()
    np.testing.assert_allclose(depth[0][inner], exact[inner], atol=1e-9)
    np.testing.assert_allclose(normal[0][inner], np.broadcast_to([0, 0, -1.0], normal[0][inner].shape), atol=1e-9)
    t_lo = RR.rays(P[None, :3], K, 24, 32, origin, vs, dims)[2].reshape(24, 32)
    fine_steps = (exact - t_lo) / (vs / 2)
    assert n[0][inner].mean() < 0.8 * fine_steps[inner].mean()


# ---- hand-made 2 x 2 x 2 volumes ---------------------------------------------------------------------------------------
K1 = [[1.0, 0, 0.0], [0, 1.0, 0.0], [0, 0, 1]]          # 1 x 1 frames: pixel (0, 0) looks along the optical axis
LOOK_UP = RF.pose(np.eye(3), [1.0, 1.0, -1.0])           # at the box's x, y centre, looking along +z
LOOK_DOWN = RF.pose(RF.rot("x", np.pi), [1.0, 1.0, 3.0])


def _two(F=(0.75, -0.25), weight=None, dims=(2, 2, 2)):
    """A volume of unit voxels at the origin whose TSDF runs along z through the values F per z layer; colour (0, 100,
    200) in the first layer, (200, 100, 0) in the last"""
    X, Y, Z = dims
    vol = RF.empty_volume(dims)
    vol["tsdf"][:] = np.asarray(F, float)[:Z, None, None]
    vol["weight"][:] = 1.0 if weight is None else weight
    vol["color"][:, 0] = np.array([0, 100, 200.0])[:, None, None]
    vol["color"][:, -1] = np.array([200, 100, 0.0])[:, None, None]
    return vol


def _cast(vol, P, near=0.0, far=np.inf, dtype=np.float64, trunc=2.0):
    d, c, n = RR.raycast(vol, (0, 0, 0), 1.0, trunc, P[None, :3], K1, 1, 1, near, far, dtype)
    return d[0, 0, 0], c[0, 0, 0], n[0, 0, 0]


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_hand_made_hit(dtype):
    """F = 0.75 - g_z on the ray g = (0.5, 0.5, t - 1.5), which is parallel to x and y: samples at t = 1.5, 2.0 (fine
    steps of 0.5), 2.5 with F = 0.75, 0.25, -0.25, so s = 0.5 and the depth is 2.25 (the surface at z = 1.25 seen from
    z = -1); the colour at g_z = 0.5 and 1 is (100, 100, 100) and (200, 100, 0); every voxel's z gradient is -1."""
    d, c, n = _cast(_two(), LOOK_UP, dtype=dtype)
    assert d == 2.25
    assert c.tolist() == [150, 100, 50]
    assert n.tolist() == [0.0, 0.0, -1.0]


def test_back_face_is_a_miss():
    d, c, n = _cast(_two(), LOOK_DOWN)                   # from z = 3 the field goes from negative to positive
    assert d == 0 and not c.any() and not n.any()
    d, _, _ = _cast(_two(F=(-0.25, 0.75)), LOOK_DOWN)    # the mirrored field is a front face from there
    assert d == 2.25


def test_unknown_voxel_breaks_the_chain():
    F = (0.75, 0.5, 0.25, -0.25, -0.5)
    dims = (2, 2, 5)
    assert _cast(_two(F, dims=dims), LOOK_UP)[0] == pytest.approx(1.5 + 2.5)   # the crossing at g_z = 2.5
    weight = np.ones((5, 2, 2))
    weight[2, 1, 0] = 0                                  # cells 1 and 2 are unknown: positive, unknown, negative
    assert _cast(_two(F, weight=weight, dims=dims), LOOK_UP)[0] == 0
    weight = np.ones((2, 2, 2))
    weight[1, 0, 1] = 0
    assert _cast(_two(weight=weight), LOOK_UP)[0] == 0   # the only cell is unknown


def test_near_and_far_cut_the_crossing():
    vol = _two()
    assert _cast(vol, LOOK_UP, near=2.3)[0] == 0         # starts behind the surface
    assert _cast(vol, LOOK_UP, far=2.2)[0] == 0          # ends in front of it
    assert _cast(vol, LOOK_UP, near=2.1, far=2.4)[0] == pytest.approx(2.25)
    assert _cast(vol, LOOK_UP, near=2.25)[0] == 2.25     # F == 0 at the first sample counts as outside: s = 0


def test_rays_that_miss_the_box_and_flat_volumes():
    vol = _two()
    assert _cast(vol, RF.pose(np.eye(3), [3.0, 1.0, -1.0]))[0] == 0         # parallel to z, beside the box
    assert _cast(vol, RF.pose(RF.rot("x", np.pi), [1.0, 1.0, -1.0]))[0] == 0  # looking away from it
    for dims in ((1, 2, 2), (2, 1, 2), (2, 2, 1)):
        assert _cast(_two(dims=dims), LOOK_UP)[0] == 0


def test_rays_slab_range():
    gd, go, t_lo, t_hi, ok = RR.rays(LOOK_UP[None, :3], K1, 1, 1, (0, 0, 0), 1.0, (2, 2, 2))
    assert ok.all() and gd[:, 0].tolist() == [0, 0, 1] and go[:, 0].tolist() == [0.5, 0.5, -1.5]
    assert (t_lo[0], t_hi[0]) == (1.5, 2.5)


def test_float32_statement_is_close_to_float64():
    scene, K, poses = RF.sphere_clip()
    vs = 0.01
    origin, dims = covering_scene(scene)
    vol, _ = _fuse64(scene, K, poses, origin, vs, dims, h=H, w=W)
    vol32 = {k: v.astype(np.float32) for k, v in vol.items()}
    c2w = _camera_to_world(poses)
    d64, c64, n64 = RR.raycast(vol32, origin, vs, 4 * vs, c2w, K, H, W)
    d32, c32, n32 = RR.raycast(vol32, origin, vs, 4 * vs, c2w, K, H, W, dtype=np.float32)
    assert d32.dtype == np.float32 and (d32 > 0).mean() > 0.5
    assert ((d32 > 0) == (d64 > 0)).mean() > 0.999
    both = (d32 > 0) & (d64 > 0)
    assert np.abs(d32 - d64)[both].max() <= 1e-5
    assert np.abs(n32 - n64)[both].max() <= 1e-4
    assert np.abs(c32.astype(int) - c64.astype(int))[both].max() <= 1


def test_camera_to_world_rows():
    _, _, poses = RF.tilted_plane_clip()
    rows = _camera_to_world([p for p in poses])
    assert rows.dtype == np.float32 and rows.shape == (len(poses), 3, 4) and rows.flags["C_CONTIGUOUS"]
    np.testing.assert_array_equal(rows, poses.astype(np.float32)[:, :3])


# ---- argument checks ------------------------------------------------------------------------------------------------
def test_render_arguments_are_checked():
    vol = object.__new__(TSDFVolume)
    vol.device = torch.device("cuda", 0)
    K = np.array([[10.0, 0, 4], [0, 10.0, 4], [0, 0, 1]])
    with pytest.raises(ValueError, match="intrinsics"):
        vol.render(np.eye(4), [np.eye(4)], (8, 8))
    with pytest.raises(ValueError, match="fx"):
        vol.render(np.diag([0.0, 1.0, 1.0]), [np.eye(4)], (8, 8))
    with pytest.raises(ValueError, match="pose"):
        vol.render(K, [np.eye(3)], (8, 8))
    with pytest.raises(ValueError, match="finite"):
        vol.render(K, [np.full((4, 4), np.nan)], (8, 8))
    with pytest.raises(ValueError, match="frame_size"):
        vol.render(K, [np.eye(4)], (0, 8))
    with pytest.raises(ValueError, match="near"):
        vol.render(K, [np.eye(4)], (8, 8), near=-1.0)
    with pytest.raises(ValueError, match="near"):
        vol.render(K, [np.eye(4)], (8, 8), near=2.0, far=1.0)
    with pytest.raises(ValueError, match="near"):
        vol.render(K, [np.eye(4)], (8, 8), far=float("nan"))


def test_c_entry_checks_arguments_without_a_gpu():
    one = ctypes.c_void_p(256)
    origin = (ctypes.c_float * 3)(0, 0, 0)

    def call(**kw):
        a = dict(tsdf=one, weight=ctypes.c_void_p(1024), color=ctypes.c_void_p(2048), X=2, Y=2, Z=2, vs=0.1, trunc=0.4,
                 c2w=ctypes.c_void_p(4096), n=1, h=4, w=4, fx=1.0, fy=1.0, cx=0.0, cy=0.0, near=0.0, far=float("inf"),
                 depth=ctypes.c_void_p(8192), rgb=ctypes.c_void_p(8192 + 64), normal=ctypes.c_void_p(8192 + 128))
        a.update(kw)
        rc = ops.LIB.um_tsdf_raycast(a["tsdf"], a["weight"], a["color"], a["X"], a["Y"], a["Z"], origin, a["vs"], a["trunc"],
                                     a["c2w"], a["n"], a["h"], a["w"], a["fx"], a["fy"], a["cx"], a["cy"], a["near"],
                                     a["far"], a["depth"], a["rgb"], a["normal"], None)
        return rc, ops.LIB.um_last_error()

    assert call(tsdf=None) == (-22, b"um_tsdf_raycast: no pointer may be NULL")
    assert b"2^31 - 1" in call(X=2048, Y=2048, Z=512)[1]
    assert b"trunc" in call(trunc=0.0)[1]
    assert b"views" in call(n=0)[1] and b"views" in call(n=65536)[1]
    assert b"fx" in call(fx=0.0)[1] and b"fx" in call(cy=float("nan"))[1]
    assert b"near" in call(near=-1.0)[1] and b"near" in call(near=1.0, far=1.0)[1] and b"near" in call(far=float("nan"))[1]
    assert b"aligned" in call(c2w=ctypes.c_void_p(4098))[1]
    assert b"overlap" in call(rgb=ctypes.c_void_p(8192))[1]
