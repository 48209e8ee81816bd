"""The multi-view consistency filter on the device: `um_depth_consistency` and `depth_points` bit for bit against the
float32 statement (tests/refops_consistency.py) on random clips, the analytic clips, odd tables and sizes, and
`DepthFusionRunner(consistency_views=k)` against `fuse_depths` of `filter_depths` on the runner's own depths (graph and
eager, batch 1 and 3, a short last step, pieces, `reset_scene()`), against a host loop of filter, `track` and
`fuse_depths`, and `consistency_views=0` against the runner without the option."""
import numpy as np
import pytest
import torch

import refops_consistency as RC
import refops_icp as RI
from test_fusion_gpu import _clip, _model, _random_clip, _runner_volume
from test_icp_gpu import POSE_TOL, _corner_volume, _drift_clip
from unimatch_b200.fusion import TSDFVolume, _ICP, depth_points, filter_depths, fuse_depths, sequence_sources
from unimatch_b200.inference import DepthFusionRunner, _camera_to_world, _world_to_camera

pytestmark = pytest.mark.gpu
_OPS = torch.ops.unimatch_sm100


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _check_filter(d, Kc, poses, sources, **kw):
    """filter_depths against the float32 statement, twice (the same bits from run to run)"""
    dd = torch.from_numpy(np.ascontiguousarray(d, np.float32)).cuda()
    out = filter_depths(dd, Kc, poses, sources, **kw)
    again = filter_depths(dd, Kc, poses, sources, **kw)
    n = len(poses)
    ps = [np.asarray(p, np.float32) for p in poses]
    views, depth = RC.consistency(d, _camera_to_world(ps), _world_to_camera(ps), np.asarray(Kc, np.float32), range(n),
                                  sources, kw.get("max_pixel", 1.0), kw.get("max_relative", 0.01), kw.get("min_views", 2))
    assert np.array_equal(out["views"].cpu().numpy(), views)
    assert np.array_equal(_bits(out["depth"].cpu().numpy()), _bits(depth))
    assert torch.equal(out["views"], again["views"]) and torch.equal(out["depth"], again["depth"])
    return out, views


@pytest.mark.parametrize("seed", [0, 1])
def test_random_clips_bit_for_bit(seed):
    """Random depths with invalid entries, cameras 0.3 rad apart: many sources fail, and some pass on the smooth parts"""
    d, _, poses = _random_clip(6, 37, 53, seed=seed)
    g = np.random.default_rng(seed)
    d = np.where(g.random(d.shape) < 0.5, np.float32(2.5), d).astype(np.float32)       # flat patches that can agree
    Kc = np.array([[30.0, 0, 26.5], [0, 30.0, 18.0], [0, 0, 1]], np.float32)
    _check_filter(d, Kc, poses, sequence_sources(6, 2, 2), min_views=1)
    _check_filter(d, Kc, poses, sequence_sources(6, 3, 1), max_pixel=2.5, max_relative=0.2, min_views=2)


@pytest.mark.parametrize("name", ["sphere", "tilted", "corner"])
def test_analytic_clips_bit_for_bit(name):
    D, Kc, P, _ = RC.clip_depths(name)
    out, views = _check_filter(D, Kc, list(P), sequence_sources(5, 2, 2))
    assert views.max() == 4 and (out["depth"] > 0).float().mean() > 0.5
    frames = np.random.default_rng(4).integers(0, 256, D.shape + (3,), dtype=np.uint8)
    _check_points(out["depth"].cpu().numpy(), frames, Kc, list(P))


def test_odd_tables_and_sizes():
    d, _, poses = _random_clip(5, 20, 30, seed=3)
    d = np.where(np.random.default_rng(3).random(d.shape) < 0.6, np.float32(2.0), d).astype(np.float32)
    Kc = np.array([[25.0, 0, 15.0], [0, 25.0, 10.0], [0, 0, 1]], np.float32)
    table = np.array([[-1, 1, 1, 2], [0, -1, 0, 3], [4, 4, -1, -1], [-1, -1, -1, -1], [3, 2, 1, 0]], np.int32)
    _check_filter(d, Kc, poses, table, min_views=1)                                   # -1 and duplicate sources
    _check_filter(d, Kc, poses, table, min_views=4)
    _check_filter(d, Kc, poses, sequence_sources(5, 1, 0), min_views=1)               # S = 1
    wide = np.array([[(t + 1 + j) % 5 for j in range(255)] for t in range(5)], np.int32)
    wide[wide == np.arange(5)[:, None]] = -1
    _check_filter(d, Kc, poses, wide, min_views=3)                                     # S = 255
    one = np.full((3, 1, 1), 2.0, np.float32)                                          # 1-pixel frames
    K1 = np.array([[1.0, 0, 0.0], [0, 1.0, 0.0], [0, 0, 1]], np.float32)
    _check_filter(one, K1, [np.eye(4, dtype=np.float32)] * 3, sequence_sources(3, 1, 1), min_views=1)


def test_out_of_range_entries_read_nothing_on_the_device():
    """The entry itself treats out-of-range references and sources as absent (filter_depths refuses them first)"""
    d, _, poses = _random_clip(4, 16, 24, seed=6)
    Kc = np.array([[20.0, 0, 12.0], [0, 20.0, 8.0], [0, 0, 1]], np.float32)
    dev = torch.from_numpy(d).cuda()
    c2w, w2c = (torch.from_numpy(f(poses)).cuda() for f in (_camera_to_world, _world_to_camera))
    refs = torch.tensor([0, 7, -3, 2], dtype=torch.int32, device="cuda")
    src = torch.tensor([[1, 9, -5], [0, 1, 2], [0, 1, 2], [1000, 3, -1]], dtype=torch.int32, device="cuda")
    views, out = _OPS.depth_consistency(dev, c2w, w2c, refs, src, 20.0, 20.0, 12.0, 8.0, 1.0, 0.01, 1)
    rv, rd = RC.consistency(d, _camera_to_world(poses), _world_to_camera(poses), Kc, [0, 7, -3, 2],
                            [[1, 9, -5], [0, 1, 2], [0, 1, 2], [1000, 3, -1]], min_views=1)
    assert np.array_equal(views.cpu().numpy(), rv) and np.array_equal(_bits(out.cpu().numpy()), _bits(rd))
    assert not views[1:3].any() and not out[1:3].any()


def _check_points(d, frames, Kc, poses):
    pts, cols = depth_points(torch.from_numpy(np.ascontiguousarray(d)).cuda(), torch.from_numpy(frames).cuda(), Kc, poses)
    rp, rc = RC.points(d, frames, _camera_to_world(poses), Kc)
    assert np.array_equal(_bits(pts.cpu().numpy()), _bits(rp)) and np.array_equal(cols.cpu().numpy(), rc)
    return pts


def test_depth_points_bit_for_bit():
    d, frames, poses = _random_clip(5, 33, 47, seed=8)
    Kc = np.array([[30.0, 0, 23.5], [0, 30.0, 16.5], [0, 0, 1]], np.float32)
    pts = _check_points(d, frames, Kc, poses)
    assert 0 < pts.shape[0] < d.size
    p2, _ = depth_points(torch.from_numpy(d).cuda(), torch.from_numpy(frames).cuda(), Kc, poses)
    assert torch.equal(pts, p2)
    empty = np.zeros((2, 9, 7), np.float32)
    assert depth_points(torch.from_numpy(empty).cuda(), torch.zeros((2, 9, 7, 3), dtype=torch.uint8, device="cuda"), Kc,
                        poses[:2])[0].shape == (0, 3)


# ---- the runner ---------------------------------------------------------------------------------------------------------
def _run(batch, use_graph, pieces, k, m=2, track=False, scene="plane", reset_after=None):
    """The runner over the synthetic plane clip, or (scene="corner") the drifting corner clip whose depths are the
    exact rendered ones (as tests/test_icp_gpu.py feeds them).  Returns (runner, volume, results, clip)."""
    m_, kw = _model()
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
    runner = DepthFusionRunner(m_, (64, 96), batch, "cuda", Kc, vol, use_graph=use_graph, track=track,
                               consistency_views=k, consistency_min_views=m, **kw)
    if scene == "corner":
        table = torch.from_numpy(np.stack([RI.render_union(scenes, Kc, P, 64, 96) for P in true]).astype(np.float32)).cuda()

        def scene_depth(slot, first, second):
            idx = torch.cat((runner.carry_frame, runner.dev_in[slot][:-1]))[:, 0, 0, 0].long()
            return table[idx]
        runner._depth = scene_depth
    res = []
    for i, (a, b) in enumerate(pieces):
        if reset_after is not None and i == reset_after:
            runner.reset_scene()
            res = []
        res += [{key: v.clone() for key, v in r.items()} for r in runner.run(items[a:b])]
    return runner, vol, res, (frames, Kc, poses)


def _fused(pieces, reset_after=None):
    keep = [t for i, (a, b) in enumerate(pieces) if reset_after is None or i >= reset_after for t in range(a, b - 1)]
    return keep


def _reference(res, keep, frames, Kc, poses, k, m, volume):
    D = torch.stack([r["depth"] for r in res]).cuda()
    P = poses.numpy()[keep]
    f = filter_depths(D, Kc, list(P), sequence_sources(len(keep), k, 0), min_views=m)
    fuse_depths(volume, f["depth"], frames[keep].cuda(), Kc, list(P))
    return f


def _assert_volumes_equal(a, b):
    for key in ("tsdf", "weight", "color"):
        assert torch.equal(getattr(a, key), getattr(b, key)), key


@pytest.mark.parametrize("k,batch,use_graph", [(2, 1, True), (2, 3, True), (4, 3, True), (4, 3, False), (4, 1, False)])
def test_runner_equals_fuse_depths_of_filter_depths(k, batch, use_graph):
    """8 frames, 7 fused: at batch 3 the last step has 1 real pair; fed whole, then in two pieces"""
    for pieces in (((0, 8),), ((0, 5), (5, 8))):
        runner, vol, res, (frames, Kc, poses) = _run(batch, use_graph, pieces, k, m=2 if k == 2 else 3)
        keep = _fused(pieces)
        assert len(res) == len(keep)
        ref = _runner_volume(Kc, poses, 64, 96)
        f = _reference(res, keep, frames, Kc, poses, k, runner.consistency_min_views, ref)
        _assert_volumes_equal(vol, ref)
        assert torch.equal(torch.stack([r["views"] for r in res]), f["views"].cpu())
        assert (ref.weight > 0).any()


def test_runner_reset_scene():
    """reset_scene() between two pieces: the second piece is a new scene (empty volume and ring)"""
    pieces = ((0, 4), (4, 8))
    runner, vol, res, (frames, Kc, poses) = _run(3, True, pieces, 2, reset_after=1)
    keep = _fused(pieces, reset_after=1)
    ref = _runner_volume(Kc, poses, 64, 96)
    _reference(res, keep, frames, Kc, poses, 2, 2, ref)
    _assert_volumes_equal(vol, ref)
    assert not res[0]["views"].any()                              # the new scene's first frame has no earlier frame


def test_runner_without_consistency_is_unchanged():
    _, va, ra, _ = _run(3, True, ((0, 8),), 0)
    m_, kw = _model()
    frames, Kc, poses, items = _clip()
    vb = _runner_volume(Kc, poses, 64, 96)
    rb = [{key: v.clone() for key, v in r.items()} for r in DepthFusionRunner(m_, (64, 96), 3, "cuda", Kc, vb, **kw).run(items)]
    _assert_volumes_equal(va, vb)
    assert all(set(x) == {"depth"} and torch.equal(x["depth"], y["depth"]) for x, y in zip(ra, rb))


def test_runner_with_tracking_matches_a_host_loop():
    """track=True on the drifting corner clip: the filtered depth is tracked and fused; a host loop of filter_depths,
    the tracking ops and integration frame by frame gives the same poses within the track-runner test's tolerance and
    the same volume"""
    pieces = ((0, 5), (5, 8))
    runner, vol, res, (frames, Kc, poses) = _run(3, True, pieces, 2, m=1, track=True, scene="corner")
    keep = _fused(pieces)
    D = torch.stack([r["depth"] for r in res]).cuda()
    P = poses.numpy()[keep]
    f = filter_depths(D, Kc, list(P), sequence_sources(len(keep), 2, 0), min_views=1)
    assert torch.equal(f["views"].cpu(), torch.stack([r["views"] for r in res]))
    ref = _corner_volume()
    Kt = torch.as_tensor(Kc).float()
    icp = _ICP(ref, Kt, 1, 64, 96, 3, (4, 5, 10), 0.1, 20.0, 0.3, "test")
    C = torch.eye(4, dtype=torch.float64, device="cuda")
    one = torch.ones((1,), dtype=torch.int32, device="cuda")
    for i, (t, r) in enumerate(zip(keep, res)):
        depth = f["depth"][i:i + 1].contiguous()
        outs = (torch.empty((1, 4, 4), device="cuda"), torch.empty((1,), dtype=torch.uint8, device="cuda"),
                torch.empty((1,), dtype=torch.int64, device="cuda"), torch.empty((1,), device="cuda"))
        Pt = torch.from_numpy(poses.numpy()[t:t + 1].astype(np.float64)).cuda()
        icp.track(*icp.prepare(depth), Pt, one, outs, correction=C)
        ref._integrate(depth, frames[t:t + 1].cuda(), icp.w2c_out, one, Kt)
        assert (outs[0][0].cpu() - r["pose"]).abs().max().item() <= POSE_TOL
        assert bool(outs[1][0]) == bool(r["tracked"])
    assert sum(bool(r["tracked"]) for r in res) >= 4
    _assert_volumes_equal(vol, ref)
