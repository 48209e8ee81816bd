"""The point-cloud kernels on the device against the statement (tests/refops_recon.py): `nearest_neighbors` bit for bit
on every CPU case, `voxel_down_sample` bit for bit, the metrics' counts exactly and means to 1e-12, run-to-run
identity, 10^6 x 10^6 against float64 cKDTree, and a fused `TSDFVolume` scored against the surface its cameras saw."""
import math

import numpy as np
import pytest
import torch
from scipy import ndimage
from scipy.spatial import cKDTree

import refops_fusion as RF
import refops_recon as RR
from test_recon_eval_cpu import CASES, _sphere, case
from test_render_cpu import _depth_bound
from test_fusion_cpu import covering_scene
from unimatch_b200.evaluation import reconstruction_metrics
from unimatch_b200.fusion import TSDFVolume, fuse_depths, nearest_neighbors, voxel_down_sample

pytestmark = pytest.mark.gpu
KEYS = ("acc", "comp", "chamfer", "prec", "recall", "fscore")


@pytest.mark.parametrize("name", sorted(CASES))
def test_nearest_equals_brute_force(name):
    points, queries = case(name)
    d, i = nearest_neighbors(torch.from_numpy(queries).cuda(), points)
    assert d.is_cuda and d.dtype == torch.float32 and i.dtype == torch.int64
    ref_d, ref_i = RR.brute_nearest(queries, points)
    assert np.array_equal(d.cpu().numpy().view(np.uint32), ref_d.view(np.uint32))
    assert np.array_equal(i.cpu().numpy(), ref_i)


def test_nearest_random_sizes_and_run_to_run():
    g = np.random.default_rng(5)
    for n, q in ((1, 1), (255, 257), (3001, 1023), (20000, 5000)):
        points = np.concatenate([_sphere(n, n), g.uniform(-2, 3, (max(1, n // 100), 3)).astype(np.float32)])
        queries = g.uniform(-2, 3, (q, 3)).astype(np.float32)
        d, i = nearest_neighbors(queries, points)
        ref_d, ref_i = RR.brute_nearest(queries, points)
        assert np.array_equal(d.cpu().numpy().view(np.uint32), ref_d.view(np.uint32))
        assert np.array_equal(i.cpu().numpy(), ref_i)
        d2, i2 = nearest_neighbors(queries, points)
        assert torch.equal(d.view(torch.int32), d2.view(torch.int32)) and torch.equal(i, i2)


def test_nearest_empty_and_refusals():
    d, i = nearest_neighbors(np.zeros((0, 3), np.float32), np.ones((3, 3), np.float32))
    assert d.shape == (0,) and i.shape == (0,) and d.is_cuda
    with pytest.raises(ValueError, match="no points"):
        nearest_neighbors(np.ones((3, 3), np.float32), np.zeros((0, 3), np.float32))
    bad = np.ones((3, 3), np.float32)
    bad[1, 2] = np.nan
    with pytest.raises(ValueError, match="finite"):
        nearest_neighbors(bad, np.ones((3, 3), np.float32))
    bad[1, 2] = np.inf
    with pytest.raises(ValueError, match="finite"):
        nearest_neighbors(np.ones((3, 3), np.float32), bad)


@pytest.mark.parametrize("v", [0.02, 0.1, 0.37])
def test_voxel_down_sample_equals_statement(v):
    g = np.random.default_rng(int(v * 100))
    pts = np.concatenate([_sphere(5003, 9), g.uniform(-1, 2, (300, 3)).astype(np.float32)])
    out = voxel_down_sample(pts, v)
    ref = RR.down_sample(pts, v)
    assert out.is_cuda and np.array_equal(out.cpu().numpy().view(np.uint32), ref.view(np.uint32))
    assert torch.equal(out, voxel_down_sample(torch.from_numpy(pts).cuda(), v))


def test_voxel_down_sample_refusals():
    assert voxel_down_sample(np.zeros((0, 3), np.float32), 0.1).shape == (0, 3)
    with pytest.raises(ValueError, match="2\\^21"):
        voxel_down_sample(np.array([[0, 0, 0], [3e3, 0, 0]], np.float32), 1e-3)
    with pytest.raises(ValueError, match="finite"):
        voxel_down_sample(np.array([[0, 0, 0], [np.nan, 0, 0]], np.float32), 0.1)


@pytest.mark.parametrize("down", [None, 0.02, 0.05])
def test_metrics_match_statement(down):
    g = np.random.default_rng(11)
    gt = _sphere(4000, 3)
    pred = np.concatenate([gt[::3] + g.normal(0, 0.02, (1334, 3)), g.uniform(-1, 2, (40, 3))]).astype(np.float32)
    m = reconstruction_metrics(torch.from_numpy(pred).cuda(), gt, down_sample=down)
    ref = RR.metrics(pred, gt, 0.05, down)
    assert (m["n_pred"], m["n_gt"]) == (ref["n_pred"], ref["n_gt"])
    assert m["prec"] == ref["prec"] and m["recall"] == ref["recall"] and m["fscore"] == ref["fscore"]
    for k in ("acc", "comp", "chamfer"):
        assert m[k] == pytest.approx(ref[k], rel=1e-12)
    assert reconstruction_metrics(torch.from_numpy(pred).cuda(), gt, down_sample=down) == m     # run to run


def test_metrics_empty_and_refusals():
    one = np.ones((5, 3), np.float32)
    for pred, gt, n in ((np.zeros((0, 3), np.float32), one, (0, 1)), (one, np.zeros((0, 3), np.float32), (1, 0))):
        m = reconstruction_metrics(pred, gt)
        assert all(math.isnan(m[k]) for k in KEYS) and (m["n_pred"], m["n_gt"]) == n
    bad = one.copy()
    bad[2, 0] = np.inf
    with pytest.raises(ValueError, match="finite"):
        reconstruction_metrics(bad, one)
    with pytest.raises(ValueError, match="2\\^21"):
        reconstruction_metrics(np.array([[0, 0, 0], [5e3, 0, 0]], np.float32), one, down_sample=1e-3)


def test_million_points_against_float64_kdtree():
    g = np.random.default_rng(12)
    points = g.uniform(0, 3, (1_000_000, 3)).astype(np.float32)
    queries = g.uniform(-0.1, 3.1, (1_000_000, 3)).astype(np.float32)
    d = nearest_neighbors(queries, points)[0].cpu().numpy()
    ref = cKDTree(points.astype(np.float64)).query(queries.astype(np.float64), workers=-1)[0]
    assert np.allclose(d, ref, rtol=1e-6, atol=0)


def _back_projected(scene, K, poses, h, w):
    """The exact depth pixels of the clip's cameras, back-projected: the surface those cameras saw"""
    out = []
    for P in poses:
        d = RF.render(scene, K, P, h, w)
        x = P[:3, 3] + (RF.rays(K, h, w) @ P[:3, :3].T) * d[..., None]
        out.append(x[d > 0])
    return np.concatenate(out).astype(np.float32)


@pytest.mark.parametrize("clip", ["sphere", "tilted_plane"])
def test_fused_volume_scored_against_its_surface(clip):
    """Fused at 8 x the clip's resolution, as the render tests fuse it.  Each extracted point lies within the render
    tests' derived bound of the surface, so acc stays below it plus the GT's sample spacing, and comp below it plus
    a cube diagonal (a surface point's cube has a crossing edge, whose point is within the diagonal); precision at 5 cm
    is 1, and recall is 1 on the GT points at least 5 cm inside the border of the region the volume observed (the
    weight > 0 set, eroded across the viewing direction)."""
    vs, trunc, h, w, scale = 0.01, 0.04, 48, 64, 8
    scene, K, poses = getattr(RF, clip + "_clip")(h=h * scale, w=w * scale)
    Kr = getattr(RF, clip + "_clip")(h=h, w=w)[1]
    origin, dims = covering_scene(scene)
    vol = TSDFVolume(origin, vs, dims, trunc=trunc, device="cuda")
    depths = torch.from_numpy(np.stack([RF.render(scene, K, P, h * scale, w * scale) for P in poses])).float().cuda()
    frames = torch.zeros(depths.shape + (3,), dtype=torch.uint8, device="cuda")
    fuse_depths(vol, depths, frames, np.asarray(K, np.float32), [P.astype(np.float32) for P in poses])
    pred = vol.extract_points()[0]
    gt = _back_projected(scene, K, poses, h * scale, w * scale)
    lo, hi = np.array(origin) - trunc, np.array(origin) + vs * np.array(dims) + trunc
    tol = _depth_bound(scene, K, poses, Kr, poses, vs, lo, hi, h, w, scale)
    spacing = float(cKDTree(gt).query(gt[::97], k=2)[0][:, 1].max())
    m = reconstruction_metrics(pred, gt, down_sample=None)
    assert m["n_pred"] > 1000 and m["acc"] < tol + spacing and m["comp"] < tol + math.sqrt(3) * vs, (m, tol, spacing)
    assert m["prec"] == 1.0
    seen = (vol.weight > 0).cpu().numpy()                                   # [Z, Y, X]
    # eroded across the viewing direction only (x and y: the clips look along +z); along z the observed region ends a
    # truncation distance behind the surface, which is not a border of what the cameras saw
    inner = ndimage.binary_erosion(seen, np.ones((1, 3, 3), bool), iterations=int(math.ceil(0.05 / vs)) + 1)
    k = np.floor((gt - np.asarray(vol.origin)) / vs).astype(np.int64)
    ok = ((k >= 0) & (k < np.asarray(dims))).all(1)
    keep = np.zeros(len(gt), bool)
    keep[ok] = inner[k[ok, 2], k[ok, 1], k[ok, 0]]
    assert keep.sum() > 1000
    d_gt = nearest_neighbors(gt[keep], pred)[0]
    assert bool((d_gt < np.float32(0.05)).all())
