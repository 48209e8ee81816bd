"""The point-cloud statement (tests/refops_recon.py) on the host: the kernel's ring search over any cell table equals the
brute-force float32 scan bit for bit; the metrics match an independent float64 Atlas formula on cKDTree; down-sampling
matches hand-computed cells; `read_ply` reads `write_ply`'s files and ScanNet's layout; argument checks."""
import math

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

import refops_recon as RR
from unimatch_b200.evaluation import reconstruction_metrics
from unimatch_b200.fusion import _boxes, down_sample_grid, nn_grid, read_ply, write_ply


def _sphere(n, seed, r=0.5):
    g = np.random.default_rng(seed)
    v = g.normal(size=(n, 3))
    return (r * v / np.linalg.norm(v, axis=1, keepdims=True) + [0.2, -0.1, 1.3]).astype(np.float32)


def _cases():
    g = np.random.default_rng(7)
    lattice = np.stack(np.meshgrid(*[np.arange(5.0)] * 3, indexing="ij"), -1).reshape(-1, 3).astype(np.float32)
    dup = g.uniform(-1, 1, (60, 3)).astype(np.float32)
    plane = g.uniform(-1, 1, (150, 3)).astype(np.float32)
    plane[:, 2] = 0.25
    return {
        "uniform": (g.uniform(-1, 1, (157, 3)), g.uniform(-1.2, 1.2, (91, 3))),
        "surface": (_sphere(203, 1), _sphere(77, 2, r=0.52)),
        "lattice_ties": (lattice, (np.stack(np.meshgrid(*[np.arange(-0.5, 5.0, 0.5)] * 3, indexing="ij"), -1)
                                   .reshape(-1, 3)[::7])),
        "duplicates": (np.concatenate([dup, dup[::-1], dup[:10]]), np.concatenate([dup[:20], g.uniform(-1, 1, (20, 3))])),
        "far_queries": (g.uniform(-1, 1, (64, 3)), np.array([[3000.0, 0, 0], [-2500.0, 1200.0, 0], [0, 0, -4000.0],
                                                             [1e4, -1e4, 1e4], [0.5, 2000.0, 0.5]])),
        "single_point": (np.array([[0.3, -0.2, 0.9]]), g.uniform(-1, 1, (33, 3))),
        "one_cell": (g.uniform(0, 1e-3, (40, 3)), g.uniform(-1e-3, 2e-3, (30, 3))),
        "coplanar": (plane, np.concatenate([g.uniform(-1, 1, (40, 3)), plane[:10]])),
    }


CASES = _cases()


def case(name):
    p, q = CASES[name]
    return np.asarray(p, np.float32), np.asarray(q, np.float32)


def _grids(points):
    lo, hi = points.min(0), points.max(0)
    yield nn_grid(lo, hi, len(points))
    ext = float((hi - lo).max()) or 1.0
    for cells in (1, 3, 17):                                           # coarse to fine, the same box
        c = ext / cells
        yield lo.tolist(), c, tuple(max(1, math.ceil(float(e) / c)) for e in hi - lo)


@pytest.mark.parametrize("name", sorted(CASES))
def test_grid_search_equals_brute_force(name):
    points, queries = case(name)
    ref_d, ref_i = RR.brute_nearest(queries, points)
    for origin, cell, dims in _grids(points):
        d, i = RR.grid_nearest(queries, points, origin, cell, dims)
        assert np.array_equal(d.view(np.uint32), ref_d.view(np.uint32)), (name, cell)
        assert np.array_equal(i, ref_i), (name, cell)


def test_ties_go_to_the_least_index():
    points = np.array([[1, 0, 0], [0, 1, 0], [-1, 0, 0], [1, 0, 0]], np.float32)
    d, i = RR.brute_nearest(np.zeros((1, 3), np.float32), points)
    assert d[0] == 1 and i[0] == 0
    d, i = RR.grid_nearest(np.zeros((1, 3), np.float32), points, [-1.0, 0.0, 0.0], 0.5, (4, 2, 1))
    assert d[0] == 1 and i[0] == 0


def _atlas64(pred, gt, t):
    """Atlas's eval_mesh as a float64 formula on cKDTree (no down-sampling)"""
    d_pred = cKDTree(gt.astype(np.float64)).query(pred.astype(np.float64))[0]
    d_gt = cKDTree(pred.astype(np.float64)).query(gt.astype(np.float64))[0]
    return d_pred, d_gt


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_metrics_match_float64_atlas(seed):
    g = np.random.default_rng(seed)
    gt = _sphere(900, seed)
    pred = np.concatenate([gt[::2] + g.normal(0, 0.02, (450, 3)), g.uniform(-1, 2, (20, 3))]).astype(np.float32)
    t = 0.05
    m = RR.metrics(pred, gt, t, None)
    d_pred, d_gt = _atlas64(pred, gt, t)
    for key, d in (("acc", d_pred), ("comp", d_gt)):
        assert m[key] == pytest.approx(d.mean(), rel=1e-6)
    for key, d in (("prec", d_pred), ("recall", d_gt)):
        near = np.abs(d - t) <= 1e-6 * t                              # counts may differ only there
        lo, hi = np.count_nonzero((d < t) & ~near), np.count_nonzero((d < t) | near)
        assert lo / len(d) <= m[key] <= hi / len(d)
    p, r = m["prec"], m["recall"]
    assert m["fscore"] == pytest.approx(2 * p * r / (p + r)) and m["chamfer"] == pytest.approx((m["acc"] + m["comp"]) / 2)
    assert (m["n_pred"], m["n_gt"]) == (len(pred), len(gt))


def test_metrics_edge_cases():
    far = np.array([[10.0, 0, 0]], np.float32)
    m = RR.metrics(far, np.zeros((1, 3), np.float32), 0.05, None)
    assert m["prec"] == m["recall"] == 0 and m["fscore"] == 0.0               # Atlas gives NaN there
    m = RR.metrics(np.zeros((0, 3)), far, 0.05, None)
    assert all(math.isnan(m[k]) for k in ("acc", "comp", "chamfer", "prec", "recall", "fscore"))
    assert (m["n_pred"], m["n_gt"]) == (0, 1)


def test_down_sample_hand_computed():
    # v = 1, min = (0, 0, 0): the grid starts at -0.5, so cell k holds [k - 0.5, k + 0.5)
    pts = np.array([[0.0, 0, 0], [0.4, 0, 0], [0.6, 0, 0], [1.4, 0, 0], [0.2, 1.0, 0], [0.1, 0.2, 0.3]], np.float32)
    origin, v, dims = RR.down_sample_grid(pts, 1.0)
    assert origin == [-0.5, -0.5, -0.5] and dims == (2, 2, 1)
    out = RR.down_sample(pts, 1.0)
    expect = np.array([[(0.0 + 0.4 + 0.1) / 3, 0.2 / 3, 0.3 / 3], [(0.6 + 1.4) / 2, 0, 0], [0.2, 1.0, 0]])
    assert np.array_equal(out, expect.astype(np.float32))               # ordered by key, x fastest
    assert down_sample_grid((pts.min(0), pts.max(0)), 1.0, "t") == ([-0.5, -0.5, -0.5], 1.0, [2, 2, 1])


def test_down_sample_refuses_large_grids():
    pts = np.array([[0, 0, 0], [3e3, 0, 0]], np.float32)
    with pytest.raises(ValueError):
        RR.down_sample_grid(pts, 1e-3)
    with pytest.raises(ValueError, match="2\\^21"):
        down_sample_grid((pts.min(0), pts.max(0)), 1e-3, "voxel_down_sample")


def test_nn_grid_caps_the_table():
    lo, cell, dims = nn_grid([0, 0, 0], [1, 2, 0], 1000)
    assert math.prod(dims) <= 2000 and dims[2] == 1 and cell > 0
    lo, cell, dims = nn_grid([0, 0, 0], [1e4, 1, 1], 10)               # a far floater: larger cells, not more
    assert math.prod(dims) <= 20 and max(dims) <= 2 ** 21
    assert nn_grid([1, 1, 1], [1, 1, 1], 5) == ([1.0, 1.0, 1.0], 1.0, (1, 1, 1))


def _mesh(seed=3):
    g = np.random.default_rng(seed)
    pts = g.normal(size=(30, 3)).astype(np.float32)
    col = g.integers(0, 256, (30, 3), dtype=np.uint8)
    nrm = g.normal(size=(30, 3)).astype(np.float32)
    faces = g.integers(0, 30, (12, 3)).astype(np.int32)
    return pts, col, nrm, faces


@pytest.mark.parametrize("with_normals", [False, True])
@pytest.mark.parametrize("with_faces", [False, True])
def test_read_ply_round_trips_write_ply(tmp_path, with_normals, with_faces):
    pts, col, nrm, faces = _mesh()
    path = str(tmp_path / "m.ply")
    write_ply(path, pts, col, nrm if with_normals else None, faces if with_faces else None)
    out = read_ply(path)
    assert np.array_equal(out["points"], pts) and np.array_equal(out["colors"], col)
    assert ("normals" in out) == with_normals and ("faces" in out) == with_faces
    if with_normals:
        assert np.array_equal(out["normals"], nrm)
    if with_faces:
        assert out["faces"].dtype == np.int32 and np.array_equal(out["faces"], faces)


def _scannet_bytes(pts, col, faces, fmt="binary_little_endian", count=3):
    head = ("ply\nformat %s 1.0\ncomment VCGLIB generated\nelement vertex %d\nproperty float x\nproperty float y\n"
            "property float z\nproperty uchar red\nproperty uchar green\nproperty uchar blue\nproperty uchar alpha\n"
            "element face %d\nproperty list uchar int vertex_indices\nend_header\n" % (fmt, len(pts), len(faces)))
    end = "<" if fmt == "binary_little_endian" else ">"
    v = np.empty(len(pts), [("p", end + "f4", 3), ("c", "u1", 4)])
    v["p"], v["c"] = pts, np.concatenate([col, np.full((len(pts), 1), 255, np.uint8)], 1)
    f = np.empty(len(faces), [("n", "u1"), ("v", end + "i4", count)])
    f["n"], f["v"] = count, faces[:, :1].repeat(count, 1) if count != 3 else faces
    return head.encode() + v.tobytes() + f.tobytes()


def test_read_ply_scannet_layout_and_refusals(tmp_path):
    pts, col, _, faces = _mesh(4)
    path = tmp_path / "scene0000_00_vh_clean_2.ply"
    path.write_bytes(_scannet_bytes(pts, col, faces))
    out = read_ply(str(path))
    assert np.array_equal(out["points"], pts) and np.array_equal(out["colors"], col)
    assert np.array_equal(out["faces"], faces) and "normals" not in out
    for data, match in ((_scannet_bytes(pts, col, faces, "binary_big_endian"), "binary_little_endian"),
                        (_scannet_bytes(pts, col, faces, count=4), "triangle"),
                        (b"ply\nformat ascii 1.0\nelement vertex 1\nproperty float x\nproperty float y\n"
                         b"property float z\nend_header\n0 0 0\n", "binary_little_endian")):
        path.write_bytes(data)
        with pytest.raises(ValueError, match=match):
            read_ply(str(path))


def test_argument_checks():
    pts = np.zeros((4, 3), np.float32)
    with pytest.raises(ValueError, match="\\[N,3\\]"):
        reconstruction_metrics(np.zeros((4, 2), np.float32), pts)
    with pytest.raises(ValueError, match="float32"):
        reconstruction_metrics(pts.astype(np.float64), pts)
    for bad in (0.0, -0.1, math.inf, math.nan, 1e-50):
        with pytest.raises(ValueError, match="threshold"):
            reconstruction_metrics(pts, pts, threshold=bad)
    for bad in (0.0, -0.02, math.nan):
        with pytest.raises(ValueError, match="voxel size"):
            reconstruction_metrics(pts, pts, down_sample=bad)
    with pytest.raises(ValueError, match="finite"):                   # the bounding-box read catches NaN and inf
        _boxes([torch.zeros((0, 3)), torch.tensor([[0.0, 1.0, 2.0], [math.nan, 0.0, 0.0]])], "t")
    with pytest.raises(ValueError, match="finite"):
        _boxes([torch.tensor([[0.0, math.inf, 2.0]])], "t")
    assert _boxes([torch.zeros((0, 3)), torch.tensor([[0.0, 1.0, 2.0], [3.0, -1.0, 2.0]])], "t") == \
        [None, ([0.0, -1.0, 2.0], [3.0, 1.0, 2.0])]
