"""TSDF fusion on the device: `um_tsdf_integrate` and the surface extraction bit for bit against the float32 statement
(tests/refops_fusion.py), frame splitting and `n_valid`, the analytic scenes through the kernels, and `DepthFusionRunner`
against `fuse_depths` on its own outputs (graph replay and eager, short last steps, warm-up, pieces of a clip) and against
`infer_depth_sequence` + `fuse_depths`."""
import numpy as np
import pytest
import torch

import refops_fusion as RF
from test_fusion_cpu import _tolerance, covering_scene
from unimatch_b200.fusion import TSDFVolume, fuse_depths
from unimatch_b200.inference import DepthFusionRunner, _world_to_camera, infer_depth_sequence
from unimatch_b200.synthetic import synthetic_model, synthetic_posed_sequence, workload_call

pytestmark = pytest.mark.gpu
_OPS = torch.ops.unimatch_sm100
_DEPTH_RANGE = ("min_depth", "max_depth", "num_depth_candidates")


def _random_clip(n, h, w, seed):
    """Random depths in [1.5, 4] m with invalid entries (0, negative, NaN, +-inf), random uint8 frames and cameras near the
    origin looking along +z, rotated by up to 0.3 rad about each axis (float32 camera-to-world poses)."""
    g = np.random.default_rng(seed)
    d = g.uniform(1.5, 4.0, (n, h, w))
    bad = g.random((n, h, w))
    for lo, v in ((0.0, 0.0), (0.01, -1.0), (0.02, np.nan), (0.03, np.inf), (0.04, -np.inf)):
        d[(bad >= lo) & (bad < lo + 0.01)] = v
    frames = g.integers(0, 256, (n, h, w, 3), dtype=np.uint8)
    poses = []
    for _ in range(n):
        R = RF.rot("z", g.uniform(-0.3, 0.3)) @ RF.rot("y", g.uniform(-0.3, 0.3)) @ RF.rot("x", g.uniform(-0.3, 0.3))
        poses.append(RF.pose(R, g.uniform(-0.3, 0.3, 3) - [0, 0, 1.0]).astype(np.float32))
    return d.astype(np.float32), frames, poses


# an odd-sized volume (not a multiple of the 256-voxel block) whose centres are exact binary fractions
ORIGIN, VS, DIMS = (-2.25, -1.5, 0.5), 0.125, (37, 23, 19)
K = np.array([[30.0, 0, 28.0], [0, 30.0, 20.0], [0, 0, 1]], np.float32)


def _volume(dims=DIMS, origin=ORIGIN, vs=VS):
    return TSDFVolume(origin, vs, dims, device="cuda")


def _planes(vol):
    return {"tsdf": vol.tsdf.cpu().numpy(), "weight": vol.weight.cpu().numpy(), "color": vol.color.cpu().numpy()}


def _assert_same(a, b):
    for k in ("tsdf", "weight", "color"):
        assert np.array_equal(a[k], b[k], equal_nan=True), k


def test_integrate_bit_for_bit_and_extraction():
    d, frames, poses = _random_clip(6, 40, 56, seed=1)
    vol = _volume()
    fuse_depths(vol, torch.from_numpy(d).cuda(), torch.from_numpy(frames).cuda(), K, poses)
    ref = RF.integrate(RF.empty_volume(DIMS, np.float32), vol.origin, vol.voxel_size, vol.trunc, d, frames,
                       _world_to_camera(poses), K, dtype=np.float32)
    got = _planes(vol)
    _assert_same(got, ref)
    assert 0.2 < (got["weight"] > 0).mean() < 1.0
    pts, cols = vol.extract_points()
    rp, rc = RF.extract(ref, vol.origin, vol.voxel_size, dtype=np.float32)
    assert len(rp) > 1000
    assert np.array_equal(pts.cpu().numpy(), rp) and np.array_equal(cols.cpu().numpy(), rc)
    pts2, cols2 = vol.extract_points()
    assert torch.equal(pts, pts2) and torch.equal(cols, cols2)


def test_integrate_half_way_pixels():
    """Voxel centres x, y in odd multiples of 1/16 at z = 2 and fx = 8, cx = cy = 0.25 project to u = 4x + 0.25, many
    exactly on a pixel half-way point, where floor(u + 0.5) takes the pixel above."""
    Kh = np.array([[8.0, 0, 0.25], [0, 8.0, 0.25], [0, 0, 1]], np.float32)
    origin, dims = (-0.5, -0.5, 1.9375), (8, 8, 1)                # centres -0.4375 .. 0.4375, z = 2.0
    g = np.random.default_rng(4)
    d = g.uniform(1.9, 2.1, (1, 4, 4)).astype(np.float32)
    frames = g.integers(0, 256, (1, 4, 4, 3), dtype=np.uint8)
    poses = [np.eye(4, dtype=np.float32)]
    vol = _volume(dims, origin, 0.125)
    fuse_depths(vol, torch.from_numpy(d).cuda(), torch.from_numpy(frames).cuda(), Kh, poses)
    ref = RF.integrate(RF.empty_volume(dims, np.float32), origin, 0.125, vol.trunc, d, frames, _world_to_camera(poses), Kh,
                       dtype=np.float32)
    _assert_same(_planes(vol), ref)
    u = 4 * (np.arange(8) * 0.125 - 0.4375) + 0.25                # exact: -1.5, -1.0, ..., 2.0
    assert (np.mod(u, 1) == 0.5).sum() == 4
    # u = -0.5 reads pixel 0, u = 3.5 would read pixel 4 (outside): the weights show which voxels were read
    assert (ref["weight"][0] > 0).sum() == int(((u >= -0.5) & (u < 3.5)).sum()) ** 2


def test_frame_splitting_and_n_valid():
    d, frames, poses = _random_clip(7, 40, 56, seed=2)
    dd, ff = torch.from_numpy(d).cuda(), torch.from_numpy(frames).cuda()
    whole = _volume()
    fuse_depths(whole, dd, ff, K, poses)
    for cuts in ((1,), (3, 6)):
        vol = _volume()
        for a, b in zip((0,) + cuts, cuts + (7,)):
            fuse_depths(vol, dd[a:b], ff[a:b], K, poses[a:b])
        _assert_same(_planes(vol), _planes(whole))
    part, first4 = _volume(), _volume()
    w2c = torch.from_numpy(_world_to_camera(poses)).cuda()
    part._integrate(dd, ff, w2c, torch.tensor([4], dtype=torch.int32, device="cuda"), K)
    fuse_depths(first4, dd[:4], ff[:4], K, poses[:4])
    _assert_same(_planes(part), _planes(first4))
    none = _volume()
    none._integrate(dd, ff, w2c, torch.tensor([0], dtype=torch.int32, device="cuda"), K)
    assert not none.weight.any() and not none.tsdf.any() and not none.color.any()
    assert len(none.extract_points()[0]) == 0


@pytest.mark.parametrize("clip", ["constant_plane", "tilted_plane", "sphere"])
def test_analytic_scenes_through_the_kernels(clip):
    scene, Kc, poses = getattr(RF, clip + "_clip")()
    if clip == "constant_plane":
        h, w = 24, 32
        # binary-exact geometry: every float32 operation on the way to the crossing is exact, so the points are
        # on the plane to the CPU bound (1e-6 voxel sizes)
        vs, origin, dims = 1 / 32, (-0.3125, -0.3125, 0.875), (20, 20, 8)
    else:
        h, w = 48, 64
        vs = 0.01
        origin, dims = covering_scene(scene)
    depths = np.stack([RF.render(scene, Kc, P, h, w) for P in poses]).astype(np.float32)
    frames = np.full((len(poses), h, w, 3), 77, np.uint8)
    vol = _volume(dims, origin, vs)
    fuse_depths(vol, torch.from_numpy(depths).cuda(), torch.from_numpy(frames).cuda(), np.array(Kc, np.float32),
                [p.astype(np.float32) for p in poses])
    pts, cols = vol.extract_points()
    pts = pts.cpu().numpy().astype(np.float64)
    assert (cols == 77).all()
    if clip == "constant_plane":
        assert len(pts) == 20 * 20
        assert np.abs(pts[:, 2] - 1.0).max() <= 1e-6 * vs
    else:
        lo = np.array(origin) - 4 * vs
        hi = np.array(origin) + np.array(dims) * vs + 4 * vs
        assert len(pts) > 1000
        assert RF.distance(scene, pts).max() <= _tolerance(scene, Kc, poses, vs, lo, hi, h, w)


# ---- the runner ---------------------------------------------------------------------------------------------------------
def _model():
    m, call = synthetic_model("gmdepth-scale1-regrefine1"), workload_call("gmdepth-scale1-regrefine1")
    return m, {k: v for k, v in call.items() if k not in _DEPTH_RANGE + ("task",)}


def _clip(T=8, h=64, w=96):
    frames, Kc, poses = synthetic_posed_sequence(T, h, w, seed=31)
    return frames, Kc, poses, list(zip(frames.numpy(), poses.numpy()))


def _runner_volume(Kc, poses, h, w):
    return TSDFVolume.covering(Kc, poses.numpy(), (h, w), 3.0, 0.05, device="cuda")


@pytest.mark.parametrize("batch,use_graph", [(1, True), (3, True), (3, False)])
def test_runner_equals_fuse_depths_on_its_outputs(batch, use_graph):
    """8 frames, 7 pairs: at batch 3 the last step has 1 real pair and 2 padding pairs, which must not be fused."""
    m, kw = _model()
    frames, Kc, poses, items = _clip()
    vol = _runner_volume(Kc, poses, 64, 96)
    runner = DepthFusionRunner(m, (64, 96), batch, "cuda", Kc, vol, use_graph=use_graph, **kw)
    assert list(runner.run(items[:1])) == []                     # captures the graphs (warm-up on reset inputs)
    assert not vol.weight.any() and not vol.tsdf.any() and not vol.color.any()
    res = [r["depth"].clone() for r in runner.run(items)]
    assert len(res) == 7
    ref = _runner_volume(Kc, poses, 64, 96)
    fuse_depths(ref, torch.stack(res).cuda(), frames[:-1].cuda(), Kc, poses.numpy()[:-1])
    _assert_same(_planes(vol), _planes(ref))
    assert (ref.weight > 0).float().mean() > 0.01


def test_runner_pieces_and_no_downloads():
    """Two run() calls feed one volume: each piece's last frame is not fused; with return_depth=False the runner yields
    empty dicts."""
    m, kw = _model()
    frames, Kc, poses, items = _clip()
    whole = _runner_volume(Kc, poses, 64, 96)
    r1 = DepthFusionRunner(m, (64, 96), 2, "cuda", Kc, whole, **kw)
    depths = [r["depth"].clone() for r in r1.run(items)]
    pieces = _runner_volume(Kc, poses, 64, 96)
    r2 = DepthFusionRunner(m, (64, 96), 2, "cuda", Kc, pieces, return_depth=False, **kw)
    out = list(r2.run(items[:4])) + list(r2.run(items[4:]))
    assert out == [{}] * 6
    ref = _runner_volume(Kc, poses, 64, 96)
    keep = [0, 1, 2, 4, 5, 6]                                      # frame 3 ends the first piece
    fuse_depths(ref, torch.stack(depths)[keep].cuda(), frames[keep].cuda(), Kc, poses.numpy()[keep])
    tol = 1e-4 * max(d.abs().max().item() for d in depths) / pieces.trunc
    # the pieces re-encode frame 4 on its own, so their depths match the whole run's up to summation order
    w_same = torch.eq(pieces.weight, ref.weight)
    assert w_same.float().mean() > 0.999
    assert (pieces.tsdf - ref.tsdf)[w_same].abs().max().item() <= tol + 1e-6


def test_runner_agrees_with_infer_depth_sequence_and_fuse_depths():
    """Within the depths' agreement: the encoder's summation order depends on how many frames are encoded together (see
    UniMatch.encode_frames), so the depths agree to 1e-4 of the largest depth, as tests/test_depth_sequence_gpu.py states;
    a TSDF value moves by at most its depth change over trunc.  A voxel near a frustum, pixel or -trunc boundary may be
    updated by one side only, so the weights may differ on a few voxels."""
    m, kw = _model()
    frames, Kc, poses, items = _clip()
    vol = _runner_volume(Kc, poses, 64, 96)
    list(DepthFusionRunner(m, (64, 96), 3, "cuda", Kc, vol, return_depth=False, **kw).run(items))
    d = infer_depth_sequence(m, frames.cuda(), Kc, poses, **kw)["depth"]
    ref = _runner_volume(Kc, poses, 64, 96)
    fuse_depths(ref, d, frames[:-1].cuda(), Kc, poses.numpy()[:-1])
    w_same = torch.eq(vol.weight, ref.weight)
    assert w_same.float().mean() > 0.999
    tol = 1e-4 * d.abs().max().item() / vol.trunc
    assert (vol.tsdf - ref.tsdf)[w_same].abs().max().item() <= tol + 1e-6
