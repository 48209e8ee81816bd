"""ICP tracking on the device: the pyramid and live normals bit for bit against the float32 statement (tests/refops_icp.py),
one association pass's block sums bit for bit, `TSDFVolume.track` against the statement on fused random clips, the corner
clip and a room, graph replay, and `DepthFusionRunner(track=True)`: graph against eager, against an eager loop of the
tracking ops plus integration, the synthetic plane sequence, a short last step and several `run()` calls."""
import math

import numpy as np
import pytest
import torch

import refops_fusion as RF
import refops_icp as RI
from test_fusion_gpu import DIMS, K, ORIGIN, VS, _clip, _model, _planes, _random_clip, _runner_volume
from unimatch_b200.fusion import TSDFVolume, _ICP, fuse_depths
from unimatch_b200.inference import DepthFusionRunner

pytestmark = pytest.mark.gpu
_OPS = torch.ops.unimatch_sm100
POSE_TOL = 1e-6      # the solve's fp64 cos / sin are CUDA's on the device and libm's in numpy: the estimates agree to the
                     # last bits of fp64 after each step, not bit for bit, so the tracked poses are compared to 1e-6


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32 if a.dtype == np.float32 else np.uint64)


def _check_track(vol, depths, Kc, poses, min_tracked=0, **kw):
    """track() against the float32 statement on the downloaded planes"""
    d = torch.from_numpy(np.asarray(depths, np.float32)).cuda()
    out = vol.track(d, Kc, poses, **kw)
    n_levels = kw.get("levels", 3)
    ref = RI.track(_planes(vol), vol.origin, vol.voxel_size, vol.trunc, np.asarray(depths, np.float32), np.asarray(Kc),
                   np.stack(poses).astype(np.float32), n_levels=n_levels, iterations=kw.get("iterations", (4, 5, 10)))
    assert np.array_equal(out["tracked"].numpy(), ref["tracked"])
    assert np.array_equal(out["inliers"].numpy(), ref["inliers"])
    assert np.abs(out["pose"].numpy().astype(np.float64) - ref["pose"]).max() <= POSE_TOL
    assert np.abs(out["rmse"].numpy() - ref["rmse"]).max() <= POSE_TOL
    assert ref["tracked"].sum() >= min_tracked
    untracked = ~ref["tracked"]
    assert np.array_equal(out["pose"].numpy()[untracked], np.stack(poses).astype(np.float32)[untracked])
    return out, ref


def test_pyramid_and_live_normals_bit_for_bit():
    d, _, _ = _random_clip(3, 41, 58, seed=5)
    dd = torch.from_numpy(d).cuda()
    trunc = 0.3
    down = _OPS.icp_downsample(dd, trunc)
    ref = RI.downsample(d, np.float32(trunc))
    assert down.shape == (3, 20, 29) and np.array_equal(_bits(down.cpu().numpy()), _bits(ref))
    smooth = np.random.default_rng(2).uniform(1.5, 1.6, (2, 40, 56)).astype(np.float32)
    smooth[0, 5, 7] = 0.0
    for depth in (d, smooth, ref):
        lv = (31.0, 29.5, 27.75, 20.25)
        n = _OPS.icp_normals(torch.from_numpy(np.ascontiguousarray(depth)).cuda(), *lv).cpu().numpy()
        rn = RI.normals(depth, *lv)
        assert np.array_equal(_bits(n), _bits(rn)) and (rn != 0).any()


def _fused_random(seed, n=6, h=40, w=56):
    d, frames, poses = _random_clip(n, h, w, seed=seed)
    vol = TSDFVolume(ORIGIN, VS, DIMS, device="cuda")
    fuse_depths(vol, torch.from_numpy(d).cuda(), torch.from_numpy(frames).cuda(), K, poses)
    return vol, d, poses


def _fused_corner():
    scenes, Kc, poses = RI.corner_clip()
    h, w = 48, 64
    depths = np.stack([RI.render_union(scenes, Kc, P, h, w) for P in poses]).astype(np.float32)
    vol = TSDFVolume((-0.6, -0.45, 1.3), 0.02, (70, 53, 58), device="cuda")
    frames = np.full((len(poses), h, w, 3), 128, np.uint8)
    Kf = np.array(Kc, np.float32)
    fuse_depths(vol, torch.from_numpy(depths).cuda(), torch.from_numpy(frames).cuda(), Kf, [p.astype(np.float32) for p in poses])
    return vol, depths, Kf, poses


@pytest.mark.parametrize("scene", ["random", "corner"])
def test_one_association_pass_bit_for_bit(scene):
    """init, the level-0 model map and one um_icp_reduce from perturbed poses: every block partial bit for bit, and so
    the inlier count exactly (random depths have few inliers, the corner clip many)"""
    if scene == "random":
        (vol, d, poses), Kc = _fused_random(1), K
    else:
        vol, d, Kc, poses = _fused_corner()
    g = np.random.default_rng(3)
    start = np.stack([RI.perturb(P, g) for P in poses]).astype(np.float32)
    n, h, w = d.shape
    icp = _ICP(vol, torch.from_numpy(Kc), n, h, w, 3, (4, 5, 10), 0.1, 20.0, 0.3, "test")
    dd = torch.from_numpy(d).cuda()
    pyr, nrm = icp.prepare(dd)
    poses64 = torch.from_numpy(start.astype(np.float64)).cuda()
    nv = torch.tensor([n], dtype=torch.int32, device="cuda")
    _OPS.icp_init(poses64, None, nv, icp.state, icp.c2w, icp.w2c)
    fx, fy, cx, cy = icp.levels[0][:4]
    md, _, mn = _OPS.tsdf_raycast(vol.tsdf, vol.weight, vol.color, vol.origin, vol.voxel_size, vol.trunc, icp.c2w, h, w,
                                  fx, fy, cx, cy, 0.0, math.inf)
    _OPS.icp_reduce(pyr[0], nrm[0], md, mn, icp.state, icp.c2w, icp.w2c, fx, fy, cx, cy, icp.max_distance,
                    icp.cos_max_angle, nv, icp.partials)
    st, c2w, w2c = RI.init(start.astype(np.float64))
    assert np.array_equal(_bits(icp.c2w.cpu().numpy()), _bits(c2w)) and np.array_equal(_bits(icp.w2c.cpu().numpy()), _bits(w2c))
    rd, rn = RI.model_maps(_planes(vol), vol.origin, vol.voxel_size, vol.trunc, c2w, RI.levels(Kc, h, w, 1)[0])
    terms = RI.pixel_terms(d, RI.normals(d, fx, fy, cx, cy), rd, rn, st["T"], c2w, w2c, fx, fy, cx, cy,
                           np.float32(icp.max_distance), np.float32(icp.cos_max_angle))
    ref = RI.block_partials(terms)
    got = icp.partials[:ref.size].view(ref.shape).cpu().numpy()
    assert np.array_equal(_bits(got), _bits(ref))
    S = RI.sums(ref)
    assert (S[:, 28] <= S[:, 29]).all() and (S[:, 29] > 0).all()
    if scene == "corner":
        assert (S[:, 28] > 0.3 * S[:, 29]).all()


@pytest.mark.parametrize("seed", [1, 4])
def test_track_fused_random_clips(seed):
    vol, d, poses = _fused_random(seed)
    g = np.random.default_rng(seed)
    start = [RI.perturb(P, g).astype(np.float32) for P in poses]
    _check_track(vol, d, K, start)
    out = vol.track(torch.from_numpy(d).cuda(), K, start)
    again = vol.track(torch.from_numpy(d).cuda(), K, start)
    assert all(torch.equal(out[k], again[k]) for k in out)


def test_track_corner_clip():
    vol, depths, Kf, poses = _fused_corner()
    g = np.random.default_rng(0)
    start = [RI.perturb(P, g).astype(np.float32) for P in poses]
    out, _ = _check_track(vol, depths, Kf, start, min_tracked=len(poses))
    for P, T in zip(poses, out["pose"].numpy()):
        assert RI.pose_error(P, T)[0] <= 0.01


def test_track_room():
    """mesh_bench's room at 2 cm, seen from render_bench's cameras at 60 x 80: live depths are render() at the true
    poses, tracking starts 2 cm and 2 degrees away"""
    from tools.mesh_bench import build_volume
    from tools.render_bench import cameras
    vol = build_volume((120, 90, 100), 0.02, torch.device("cuda"))
    extent = [n * vol.voxel_size for n in vol.dims]
    Kc, poses = cameras(extent, 4, 60, 80)
    depths = vol.render(Kc, poses, (60, 80))["depth"].cpu().numpy()
    g = np.random.default_rng(9)
    start = [RI.perturb(P, g).astype(np.float32) for P in poses]
    _check_track(vol, depths, Kc, start, min_tracked=3)


def test_empty_volume_and_no_frames():
    vol = TSDFVolume(ORIGIN, VS, DIMS, device="cuda")
    d, _, poses = _random_clip(2, 40, 56, seed=6)
    out, _ = _check_track(vol, d, K, poses)
    assert not out["tracked"].any() and not out["inliers"].any()
    none = vol.track(torch.zeros((0, 40, 56), device="cuda"), K, [])
    assert none["pose"].shape == (0, 4, 4) and none["tracked"].shape == (0,)


def test_graph_replay_equals_the_eager_call():
    vol, d, poses = _fused_random(2, n=3)
    n, h, w = d.shape
    icp = _ICP(vol, torch.from_numpy(K), n, h, w, 3, (4, 5, 10), 0.1, 20.0, 0.3, "test")
    dd = torch.from_numpy(d).cuda()
    poses64 = torch.zeros((n, 4, 4), dtype=torch.float64, device="cuda")
    nv = torch.tensor([n], dtype=torch.int32, device="cuda")
    outs = (torch.empty((n, 4, 4), device="cuda"), torch.empty((n,), dtype=torch.uint8, device="cuda"),
            torch.empty((n,), dtype=torch.int64, device="cuda"), torch.empty((n,), device="cuda"))
    poses64.copy_(torch.from_numpy(np.stack(poses).astype(np.float64)))
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        icp.track(*icp.prepare(dd), poses64, nv, outs)
    torch.cuda.current_stream().wait_stream(stream)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        icp.track(*icp.prepare(dd), poses64, nv, outs)
    g = np.random.default_rng(5)
    for trial in range(2):
        start = [RI.perturb(P, g).astype(np.float32) for P in poses]
        poses64.copy_(torch.from_numpy(np.stack(start).astype(np.float64)))
        graph.replay()
        ref = vol.track(dd, K, start)
        assert torch.equal(outs[0].cpu(), ref["pose"]) and torch.equal(outs[1].cpu().bool(), ref["tracked"])
        assert torch.equal(outs[2].cpu(), ref["inliers"]) and torch.equal(outs[3].cpu(), ref["rmse"])


def _drift_clip(n, h, w, seed=7):
    """The corner clip with given poses that carry an accumulated random walk of 0.8 cm and 0.8 degrees per frame (as
    tests/test_icp_cpu.py's drifting clip): (scenes, K float32, true poses float64, given poses float32)"""
    scenes, Kc, poses = RI.corner_clip(n=n, h=h, w=w, seed=seed)
    g = np.random.default_rng(2)
    drift, given = np.eye(4), []
    for P in poses:
        given.append(drift @ P)
        drift = RI.perturb(np.eye(4), g, 0.008, 0.8) @ drift
    return scenes, np.array(Kc, np.float32), poses, np.stack(given).astype(np.float32)


def _corner_volume():
    return TSDFVolume((-0.6, -0.45, 1.3), 0.02, (70, 53, 58), device="cuda")


def test_correction_carried_frame_by_frame():
    """The drifting corner clip, tracked and fused one frame at a time on the device with the carried correction C, as
    the runner does: every frame after the first is tracked; the pose, inliers and tracked flag agree with the statement
    run from the device's own volume and C (poses to 1e-6); the world-to-camera rows of the tracked fp64 estimate are
    its rigid inverse and C is T P^-1, bit for bit; the volume is the float32 integration at those rows bit for bit."""
    h, w = 48, 64
    scenes, Kf, poses, given = _drift_clip(6, h, w)
    depths = np.stack([RI.render_union(scenes, Kf, P, h, w) for P in poses]).astype(np.float32)
    frames = np.full((1, h, w, 3), 128, np.uint8)
    vol = _corner_volume()
    icp = _ICP(vol, torch.from_numpy(Kf), 1, h, w, 3, (4, 5, 10), 0.1, 20.0, 0.3, "test")
    C = torch.eye(4, dtype=torch.float64, device="cuda")
    one = torch.ones((1,), dtype=torch.int32, device="cuda")
    for t in range(len(poses)):
        planes, C_before = _planes(vol), C.cpu().numpy()
        ref = RI.track(planes, vol.origin, vol.voxel_size, vol.trunc, depths[t:t + 1], Kf, given[t:t + 1],
                       correction=C_before)
        outs = (torch.empty((1, 4, 4), device="cuda"), torch.empty((1,), dtype=torch.uint8, device="cuda"),
                torch.empty((1,), dtype=torch.int64, device="cuda"), torch.empty((1,), device="cuda"))
        d = torch.from_numpy(depths[t:t + 1]).cuda()
        P64 = torch.from_numpy(given[t:t + 1].astype(np.float64)).cuda()
        icp.track(*icp.prepare(d), P64, one, outs, correction=C)
        vol._integrate(d, torch.from_numpy(frames).cuda(), icp.w2c_out, one, torch.from_numpy(Kf))
        tracked = bool(outs[1][0])
        assert tracked == bool(ref["tracked"][0]) == (t > 0)
        assert int(outs[2][0]) == int(ref["inliers"][0])
        assert np.abs(outs[0][0].cpu().numpy().astype(np.float64) - ref["pose"][0]).max() <= POSE_TOL
        T = icp.state[0, :12].view(3, 4).cpu().numpy()
        assert np.array_equal(_bits(icp.w2c_out[0].cpu().numpy()), _bits(RI.rigid_inverse_rows(T)))
        C_after = RI.correction_after(T, given[t]) if tracked else C_before
        assert np.array_equal(_bits(C.cpu().numpy()), _bits(C_after))
        fused = RF.integrate({k: v.copy() for k, v in planes.items()}, vol.origin, vol.voxel_size, vol.trunc,
                             depths[t:t + 1], frames, RI.rigid_inverse_rows(T)[None], Kf, dtype=np.float32)
        got = _planes(vol)
        for k in ("tsdf", "weight", "color"):
            assert np.array_equal(got[k], fused[k]), k
        assert RI.pose_error(poses[t], T)[0] <= vol.voxel_size
    assert np.abs(C.cpu().numpy() - np.eye(4)).max() > 1e-3                  # the drift was corrected


# ---- the runner ---------------------------------------------------------------------------------------------------------
def _run(batch, use_graph, pieces, track=True, return_depth=True, scene="plane"):
    """The runner over the synthetic plane clip, or (scene="corner") over the drifting corner clip at 64 x 96: its
    frames carry their index in pixel (0, 0) and the runner's depth of pair (t, t+1) is replaced by the exact rendered
    depth of frame t, looked up on the device inside the step, so the frames after the first are tracked."""
    m, kw = _model()
    if scene == "plane":
        frames, Kc, poses, items = _clip()
        vol = _runner_volume(Kc, poses, 64, 96)
    else:
        scenes, Kc, true, given = _drift_clip(8, 64, 96)
        frames = torch.zeros((8, 64, 96, 3), dtype=torch.uint8)
        frames[:, 0, 0, 0] = torch.arange(8, dtype=torch.uint8)
        poses = torch.from_numpy(given)
        items = list(zip(frames.numpy(), given))
        vol = _corner_volume()
    runner = DepthFusionRunner(m, (64, 96), batch, "cuda", Kc, vol, use_graph=use_graph, track=track,
                               return_depth=return_depth, **kw)
    if scene == "corner":
        assert runner.size == runner.ori                                      # the depth is not resized
        table = torch.from_numpy(np.stack([RI.render_union(scenes, Kc, P, 64, 96) for P in true]).astype(np.float32)).cuda()

        def scene_depth(slot, first, second):
            idx = torch.cat((runner.carry_frame, runner.dev_in[slot][:-1]))[:, 0, 0, 0].long()
            return table[idx]
        runner._depth = scene_depth
    res = []
    for a, b in pieces:
        res += [{k: v.clone() for k, v in r.items()} for r in runner.run(items[a:b])]
    return runner, vol, res, (frames, Kc, poses)


def _assert_volumes_equal(a, b):
    for k in ("tsdf", "weight", "color"):
        assert torch.equal(getattr(a, k), getattr(b, k)), k


def _eager_loop(pieces, res, frames, Kc, poses, volume):
    """The tracking ops and integration frame by frame on the runner's own depths, the correction carried the same way
    (pieces fuse all but each piece's last frame); returns the correction"""
    keep = [t for a, b in pieces for t in range(a, b - 1)]
    assert len(keep) == len(res)
    Kt = torch.as_tensor(Kc).float()
    icp = _ICP(volume, Kt, 1, 64, 96, 3, (4, 5, 10), 0.1, 20.0, 0.3, "test")
    C = torch.eye(4, dtype=torch.float64, device="cuda")
    one = torch.ones((1,), dtype=torch.int32, device="cuda")
    for t, r in zip(keep, res):
        depth = r["depth"][None].cuda().contiguous()
        outs = (torch.empty((1, 4, 4), device="cuda"), torch.empty((1,), dtype=torch.uint8, device="cuda"),
                torch.empty((1,), dtype=torch.int64, device="cuda"), torch.empty((1,), device="cuda"))
        P = torch.from_numpy(poses.numpy()[t:t + 1].astype(np.float64)).cuda()
        icp.track(*icp.prepare(depth), P, one, outs, correction=C)
        volume._integrate(depth, frames[t:t + 1].cuda(), icp.w2c_out, one, Kt)
        assert torch.equal(outs[0][0].cpu(), r["pose"]) and bool(outs[1][0]) == bool(r["tracked"])
    return C


@pytest.mark.parametrize("scene", ["plane", "corner"])
def test_runner_graph_equals_eager_and_the_eager_loop(scene):
    """batch 3 over 8 frames (a short last step), fed as one run() and as two: the graph and the eager runner give the
    same volume, poses and correction bit for bit, and so does an eager loop of the tracking ops and integration.  On
    the corner clip every fused frame after the first is tracked, so a correction other than the identity is carried
    across steps, the short last step and the two run() calls, and the fused poses are within a voxel of the truth."""
    for pieces in (((0, 8),), ((0, 5), (5, 8))):
        ra, va, res_a, (frames, Kc, poses) = _run(3, True, pieces, scene=scene)
        rb, vb, res_b, _ = _run(3, False, pieces, scene=scene)
        _assert_volumes_equal(va, vb)
        assert torch.equal(ra.pose_correction, rb.pose_correction)
        assert all(torch.equal(x["pose"], y["pose"]) and torch.equal(x["tracked"], y["tracked"]) for x, y in zip(res_a, res_b))
        ref = _runner_volume(Kc, poses, 64, 96) if scene == "plane" else _corner_volume()
        C = _eager_loop(pieces, res_a, frames, Kc, poses, ref)
        _assert_volumes_equal(va, ref)
        assert torch.equal(C, ra.pose_correction)
        if scene == "corner":
            keep = [t for a, b in pieces for t in range(a, b - 1)]
            assert [bool(r["tracked"]) for r in res_a] == [t != 0 for t in keep]
            assert (ra.pose_correction - torch.eye(4, dtype=torch.float64, device="cuda")).abs().max() > 1e-3
            _, _, true, _ = _drift_clip(8, 64, 96)
            for t, r in zip(keep, res_a):
                assert RI.pose_error(true[t], r["pose"].numpy())[0] <= va.voxel_size


def test_runner_on_the_synthetic_plane_tracks_nothing():
    """The synthetic sequence is a fronto-parallel plane: the first frame meets an empty volume and every later one a
    plane, which leaves three unknowns free, so no frame is tracked and every pose is the given one exactly.  The
    volume then differs from track=False's only through the world-to-camera rows: the device's rigid inverse of the
    fp64 pose against np.linalg.inv in float32, a few float32 ulps per entry.  A voxel that reads the same pixel moves by
    at most that change of its camera depth over trunc (below 1e-5 m over trunc: the entries are rotations of magnitude
    <= 1 and translations below a metre, the voxels within 10 m).  A voxel whose nearest pixel flips at a pixel boundary
    reads a neighbouring depth instead; at most 0.1 % of the voxels are allowed to."""
    rt, vt, res, (frames, Kc, poses) = _run(3, True, ((0, 8),), return_depth=False)
    rp, vp, _, _ = _run(3, True, ((0, 8),), track=False, return_depth=False)
    assert all(set(r) == {"pose", "tracked"} for r in res)
    assert not any(bool(r["tracked"]) for r in res)
    assert all(torch.equal(r["pose"], poses[t]) for t, r in enumerate(res))
    assert torch.equal(rt.pose_correction, torch.eye(4, dtype=torch.float64, device="cuda"))
    same = torch.eq(vt.weight, vp.weight)
    close = (vt.tsdf - vp.tsdf).abs() <= 1e-5 / vt.trunc + 1e-6
    assert (same & close).float().mean() > 0.999
