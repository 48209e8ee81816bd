"""The TSDF mesh on the device: `TSDFVolume.extract_mesh` against the statement (tests/refops_mesh.py) -- faces
exactly, normals bit for bit, points and colours equal to `extract_points()` bit for bit -- on fused random clips,
uploaded analytic fields, an empty volume, a surface without faces and volumes one voxel thick; run-to-run identity; a
`DepthFusionRunner` volume."""
import numpy as np
import pytest
import torch

import refops_fusion as RF
import refops_mesh as RM
from test_fusion_gpu import DIMS, K, ORIGIN, VS, _model, _planes, _random_clip, _runner_volume, _clip
from unimatch_b200 import ops
from unimatch_b200.fusion import TSDFVolume, fuse_depths
from unimatch_b200.inference import DepthFusionRunner

pytestmark = pytest.mark.gpu


def _upload(vol, planes):
    for k in ("tsdf", "weight", "color"):
        getattr(vol, k).copy_(torch.from_numpy(np.asarray(planes[k], np.float32)))
    return vol


def _check_mesh(vol, min_faces=1):
    """extract_mesh against extract_points and the float32 statement on the downloaded planes; returns the mesh"""
    pts, cols, nrm, tris = vol.extract_mesh()
    assert pts.dtype == torch.float32 and cols.dtype == torch.uint8 and nrm.dtype == torch.float32
    assert tris.dtype == torch.int32 and tris.shape[1:] == (3,) and tris.device == vol.device
    p0, c0 = vol.extract_points()
    assert torch.equal(pts, p0) and torch.equal(cols, c0)
    planes = _planes(vol)
    rp, rc, rn, rt = RM.mesh(planes, vol.origin, vol.voxel_size, np.float32)
    assert np.array_equal(pts.cpu().numpy(), rp) and np.array_equal(cols.cpu().numpy(), rc)
    assert np.array_equal(nrm.cpu().numpy().view(np.uint32), rn.view(np.uint32))
    assert np.array_equal(tris.cpu().numpy(), rt)
    assert len(rt) >= min_faces
    return pts, cols, nrm, tris


@pytest.mark.parametrize("seed", [1, 3])
def test_fused_random_clip(seed):
    d, frames, poses = _random_clip(6, 40, 56, seed=seed)
    vol = TSDFVolume(ORIGIN, VS, DIMS, device="cuda")                  # odd dims, not a multiple of 256 voxels
    fuse_depths(vol, torch.from_numpy(d).cuda(), torch.from_numpy(frames).cuda(), K, poses)
    mesh = _check_mesh(vol, min_faces=1000)
    again = vol.extract_mesh()
    assert all(torch.equal(a, b) for a, b in zip(mesh, again))
    assert RM.unmatched_edges(mesh[3].cpu().numpy())                  # unobserved voxels leave boundaries


@pytest.mark.parametrize("name,field", [
    ("sphere", RM.sphere((0.013, -0.021, 0.017), 0.61)),
    ("torus", RM.torus((0.011, -0.013, 0.007), 0.55, 0.21)),
])
def test_uploaded_analytic_fields(name, field):
    vs = 1 / 32
    origin, dims = (-1.0, -1.0, -0.75), (64, 61, 47)
    planes = RM.sdf_volume(field, origin, vs, dims, 4 * vs)
    planes["color"] = np.random.default_rng(2).uniform(0, 255, planes["color"].shape)
    vol = _upload(TSDFVolume(origin, vs, dims, device="cuda"), planes)
    _, _, nrm, tris = _check_mesh(vol, min_faces=1000)
    assert RM.is_closed_manifold(tris.cpu().numpy())
    assert RM.euler_characteristic(tris.cpu().numpy()) == (2 if name == "sphere" else 0)
    assert torch.allclose(nrm.norm(dim=1), torch.ones(1, device="cuda"), atol=1e-6)


def test_empty_volume_launches_only_the_counts():
    vol = TSDFVolume(ORIGIN, VS, DIMS, device="cuda")
    before = ops.launch_count()
    pts, cols, nrm, tris = vol.extract_mesh()
    assert ops.launch_count() - before == 4                            # two count passes and their scans
    assert pts.shape == cols.shape == nrm.shape == (0, 3) and tris.shape == (0, 3)


def test_points_without_faces():
    """Crossings along one observed row of voxels, but no cube with all 8 corners observed"""
    planes = RF.empty_volume((9, 4, 5))
    planes["tsdf"][2, 1] = np.linspace(-1, 1, 9)
    planes["weight"][2, 1] = 1
    planes["color"][:, 2, 1] = 200
    vol = _upload(TSDFVolume((0, 0, 0), 0.1, (9, 4, 5), device="cuda"), planes)
    pts, _, nrm, tris = _check_mesh(vol, min_faces=0)
    assert len(pts) == 1 and len(tris) == 0
    assert nrm.cpu().tolist() == [[1.0, 0.0, 0.0]]                     # along the row's gradient


@pytest.mark.parametrize("dims", [(1, 9, 7), (8, 1, 7), (8, 9, 1), (1, 1, 300)])
def test_a_dimension_of_one(dims):
    g = np.random.default_rng(7)
    X, Y, Z = dims
    planes = {"tsdf": g.uniform(-1, 1, (Z, Y, X)), "weight": (g.random((Z, Y, X)) > 0.1).astype(np.float64),
              "color": g.uniform(0, 255, (3, Z, Y, X))}
    vol = _upload(TSDFVolume((0.5, -0.25, 1.0), 0.05, dims, device="cuda"), planes)
    pts, _, _, tris = _check_mesh(vol, min_faces=0)
    assert len(pts) > 0 and len(tris) == 0


def test_runner_volume():
    m, kw = _model()
    frames, Kc, poses, items = _clip()
    vol = _runner_volume(Kc, poses, 64, 96)
    runner = DepthFusionRunner(m, (64, 96), 3, "cuda", Kc, vol, return_depth=False, **kw)
    list(runner.run(items))
    _check_mesh(runner.volume, min_faces=100)
