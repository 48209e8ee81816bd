"""The TSDF mesh without a GPU: the committed case table against its generator and the rule it states, the statement
(tests/refops_mesh.py) on exact signed distance fields (closed 2-manifolds of the right Euler characteristic, distances
and normals within bounds derived from the voxel size) and on random fields (every configuration, no cracks, boundaries
only at unobserved voxels), the PLY writer with normals and faces, and the C entries' argument checks."""
import ctypes

import numpy as np
import pytest
import torch

import refops_fusion as RF
import refops_mesh as RM
from unimatch_b200 import ops
from unimatch_b200.csrc import um_mc_table as MC
from unimatch_b200.fusion import write_ply


def test_committed_table_is_the_generators():
    with open(MC.HEADER) as f:
        assert f.read() == MC.render()


def test_triangles_per_configuration():
    assert np.bincount(RM.NTRI, minlength=6).tolist() == [2, 16, 50, 80, 76, 32]
    for cfg in range(256):
        neg = [(cfg >> c) & 1 for c in range(8)]
        cut = {e for e in range(12) if neg[MC.edge_corners(e)[0]] != neg[MC.edge_corners(e)[1]]}
        used = {e for t in RM.TRIANGLES[cfg] for e in t}
        assert used == cut, cfg                              # only crossing edges, and every one of them
        assert all(len(set(t)) == 3 for t in RM.TRIANGLES[cfg])


def test_face_segments_depend_only_on_the_face():
    """Two configurations with the same four signs on a face draw the same segments there, so the cubes sharing that
    face (which see the same four values) meet without cracks; seen from the other side they run the other way."""
    for f in MC.faces():
        axis, side, corners, edges = f
        mask = sum(1 << c for c in corners)
        by_signs = {}
        for cfg in range(256):
            segs = sorted(MC.face_segments(cfg, *f))
            prev = by_signs.setdefault(cfg & mask, segs)
            assert segs == prev, (f, cfg)
        if side == 0:
            continue
        # the neighbour across this face has these corners on its side-0 face, with the same signs
        other = [g for g in MC.faces() if g[0] == axis and g[1] == 0][0]
        for signs, segs in by_signs.items():
            cfg = sum(1 << (c ^ (1 << axis)) for c in corners if signs >> c & 1)
            twin = {e: [g for g in other[3]
                        if g >> 2 == e >> 2 and MC.edge_corners(g)[0] == MC.edge_corners(e)[0] ^ (1 << axis)][0]
                    for e in edges}
            assert sorted(MC.face_segments(cfg, *other)) == sorted((twin[b], twin[a]) for a, b in segs), (axis, signs)


@pytest.mark.parametrize("name,fields,euler", [
    ("sphere", [RM.sphere((0.013, -0.021, 0.017), 0.61)], 2),
    ("two_spheres", [RM.sphere((-0.52, 0.011, 0.023), 0.33), RM.sphere((0.47, -0.017, -0.031), 0.29)], 4),
    ("torus", [RM.torus((0.011, -0.013, 0.007), 0.55, 0.21)], 0),
])
def test_analytic_meshes_are_closed_manifolds(name, fields, euler):
    vs, trunc = 1 / 32, 4 / 32
    origin, dims = (-1.0, -1.0, -1.0), (64, 64, 64)
    vol = RM.sdf_volume(lambda x: np.min([f(x) for f in fields], 0), origin, vs, dims, trunc)
    pts, _, _, tris = RM.mesh(vol, origin, vs)
    assert len(tris) > 1000
    assert RM.is_closed_manifold(tris)                       # each undirected edge in two faces, opposite directions
    assert RM.euler_characteristic(tris) == euler
    assert len(np.unique(tris)) == len(pts)                  # every point is in a face: all cubes are observed here


def _random_field(shape, seed, unobserved=0.0):
    g = np.random.default_rng(seed)
    Z, Y, X = shape
    F = g.uniform(-1, 1, shape)
    F[[0, -1]], F[:, [0, -1]], F[:, :, [0, -1]] = 1.0, 1.0, 1.0   # a positive one-voxel border
    W = (g.random(shape) >= unobserved).astype(np.float64)
    return {"tsdf": F, "weight": W, "color": g.uniform(0, 255, (3,) + shape)}


def test_random_fields_cover_every_configuration_and_stay_closed():
    """Closed: every edge is in as many faces in one direction as in the other.  Where an ambiguous face's positive
    corners are joined across the face, both cubes may fan a diagonal between the same two of its crossings, so an edge
    can be in two faces each way (the sheets touch along it); smooth fields at the voxel size do not do that (above)."""
    vol = _random_field((22, 21, 23), seed=5)
    cfg, complete = RM.cube_cases(vol)
    assert complete.all() and set(np.unique(cfg)) == set(range(256))
    tris = RM.faces(vol)
    assert len(tris) == RM.NTRI[cfg].sum()
    assert RM.unmatched_edges(tris) == []


def test_boundaries_only_next_to_unobserved_voxels():
    vol = _random_field((19, 17, 21), seed=6, unobserved=0.03)
    hit = RM.crossings(vol)
    owner = np.argwhere(hit)                                 # vertex -> (k, j, i, axis), in vertex order
    _, complete = RM.cube_cases(vol)
    Z, Y, X = vol["tsdf"].shape

    def incomplete_next_to(v):
        k, j, i, a = owner[v]
        for d1 in (0, 1):
            for d2 in (0, 1):
                d = [0, 0, 0]                                # cube offsets on the other two axes: -1 or 0
                o = [b for b in range(3) if b != a]
                d[o[0]], d[o[1]] = -d1, -d2
                ci, cj, ck = i + d[0], j + d[1], k + d[2]
                if not (0 <= ci < X - 1 and 0 <= cj < Y - 1 and 0 <= ck < Z - 1) or not complete[ck, cj, ci]:
                    return True
        return False

    tris = RM.faces(vol)
    bad = RM.unmatched_edges(tris)
    assert len(bad) > 10
    assert all(incomplete_next_to(a) and incomplete_next_to(b) for a, b in bad)
    unused = np.setdiff1d(np.arange(len(owner)), tris)
    assert len(unused) > 0 and all(incomplete_next_to(v) for v in unused)


def test_sphere_geometry_within_voxel_bounds():
    """On the sphere of radius R at voxel size vs (F linear in the distance within trunc, which covers every crossing
    edge and its gradient stencil): a vertex is the zero of the chord of the convex distance along its edge, at most
    vs^2 / (8 (R - vs)) from the surface; each voxel's central difference is within (vs / (R - vs))^2 of the gradient's
    direction, and a vertex normal lies between its two voxels' gradients, whose directions differ by at most
    vs / (R - vs), as does the true normal along the edge; each face's normal agrees with its vertices'."""
    R, vs, trunc = 0.61, 1 / 32, 4 / 32
    centre = np.array([0.013, -0.021, 0.017])
    origin, dims = (-1.0, -1.0, -1.0), (64, 64, 64)
    vol = RM.sdf_volume(RM.sphere(centre, R), origin, vs, dims, trunc)
    pts, _, nrm, tris = RM.mesh(vol, origin, vs)
    dist = RF.distance(("sphere", centre, R), pts)
    assert dist.max() <= vs * vs / (8 * (R - vs)) + 1e-12
    true = RF.normal_at(("sphere", centre, R), pts)
    assert np.allclose(np.linalg.norm(nrm, axis=-1), 1)
    e = vs / (R - vs)
    angle = np.arccos(np.clip((nrm * true).sum(-1), -1, 1))
    assert angle.max() <= e + e * e, (angle.max(), e)
    p = pts[tris]
    geo = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    assert ((geo[:, None, :] * nrm[tris]).sum(-1) > 0).all()


def test_float32_normals_follow_the_float64_statement():
    vol = _random_field((9, 8, 11), seed=8, unobserved=0.1)
    n32, n64 = RM.normals(vol, np.float32), RM.normals(vol, np.float64)
    assert n32.dtype == np.float32 and len(n32) == len(RF.extract(vol, (0, 0, 0), 0.1)[0])
    np.testing.assert_allclose(n32, n64, atol=1e-5)


def test_ply_round_trip_with_normals_and_faces(tmp_path):
    g = np.random.default_rng(3)
    pts = g.standard_normal((17, 3)).astype(np.float32)
    cols = g.integers(0, 256, (17, 3)).astype(np.uint8)
    nrm = g.standard_normal((17, 3)).astype(np.float32)
    tris = g.integers(0, 17, (9, 3)).astype(np.int32)
    path = tmp_path / "mesh.ply"
    write_ply(str(path), torch.from_numpy(pts), cols, normals=torch.from_numpy(nrm), faces=torch.from_numpy(tris))
    data = path.read_bytes()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    assert data[:end].decode("ascii").splitlines() == [
        "ply", "format binary_little_endian 1.0", "element vertex 17", "property float x", "property float y",
        "property float z", "property float nx", "property float ny", "property float nz", "property uchar red",
        "property uchar green", "property uchar blue", "element face 9", "property list uchar int vertex_indices",
        "end_header"]
    vert = np.frombuffer(data[end:end + 17 * 27], dtype=[("xyz", "<f4", 3), ("n", "<f4", 3), ("rgb", "u1", 3)])
    np.testing.assert_array_equal(vert["xyz"], pts)
    np.testing.assert_array_equal(vert["n"], nrm)
    np.testing.assert_array_equal(vert["rgb"], cols)
    face = np.frombuffer(data[end + 17 * 27:], dtype=[("n", "u1"), ("v", "<i4", 3)])
    assert (face["n"] == 3).all()
    np.testing.assert_array_equal(face["v"], tris)
    # without normals and faces the file is the point cloud's
    write_ply(str(path), pts, cols)
    plain = path.read_bytes()
    assert b"nx" not in plain and b"face" not in plain and len(plain) - plain.index(b"end_header\n") - 11 == 17 * 15
    with pytest.raises(ValueError, match="faces"):
        write_ply(str(path), pts, cols, faces=np.array([[0, 1, 17]]))
    with pytest.raises(ValueError, match="normals"):
        write_ply(str(path), pts, cols, normals=nrm[:3])


def test_c_entries_check_arguments_without_a_gpu():
    one = ctypes.c_void_p(256)
    origin = (ctypes.c_float * 3)(0, 0, 0)
    lib = ops.LIB
    assert lib.um_tsdf_mesh_count(None, one, 4, 4, 4, one, None) == -22 and b"NULL" in lib.um_last_error()
    assert lib.um_tsdf_mesh_count(one, one, 2048, 2048, 512, one, None) == -22 and b"2^31 - 1" in lib.um_last_error()
    assert lib.um_tsdf_mesh_count(ctypes.c_void_p(258), one, 4, 4, 4, one, None) == -22
    assert b"aligned" in lib.um_last_error()
    # offsets of 8 * 2 bytes at 256 overlap the tsdf plane at 260
    assert lib.um_tsdf_mesh_count(ctypes.c_void_p(260), ctypes.c_void_p(1 << 20), 4, 4, 4, one, None) == -22
    assert b"overlap" in lib.um_last_error()

    def mesh(**kw):
        a = dict(tsdf=1 << 20, weight=2 << 20, color=3 << 20, X=4, Y=4, Z=4, vs=0.1, po=4 << 20, P=10, fo=5 << 20, T=4,
                 first=6 << 20, points=7 << 20, colors=8 << 20, normals=9 << 20, faces=10 << 20)
        a.update(kw)
        p = [ctypes.c_void_p(a[k]) if a[k] else None for k in ("tsdf", "weight", "color")]
        rc = lib.um_tsdf_mesh(*p, a["X"], a["Y"], a["Z"], origin, a["vs"],
                              ctypes.c_void_p(a["po"]) if a["po"] else None, a["P"], ctypes.c_void_p(a["fo"]), a["T"],
                              *(ctypes.c_void_p(a[k]) if a[k] else None
                                for k in ("first", "points", "colors", "normals", "faces")), None)
        return rc, lib.um_last_error()

    for kw, msg in (({"po": 0}, b"no input"), ({"normals": 0}, b"normals must not be NULL"),
                    ({"faces": 0}, b"faces must not be NULL"), ({"Y": 0}, b"bad volume"), ({"vs": 0.0}, b"voxel_size"),
                    ({"P": 3 * 64 + 1}, b"bad point count"), ({"P": -1}, b"bad point count"),
                    ({"T": 5 * 64 + 1}, b"bad face count"), ({"P": 0}, b"bad face count"),
                    ({"normals": (9 << 20) + 2}, b"aligned"), ({"po": (4 << 20) + 4}, b"aligned"),
                    ({"faces": (2 << 20) + 16}, b"overlap"), ({"first": (7 << 20) + 64}, b"overlap")):
        rc, err = mesh(**kw)
        assert rc == -22 and msg in err, (kw, err)
    big = 1 << 31
    rc, err = mesh(X=2048, Y=2048, Z=511, P=big, T=0)
    assert rc == -22 and b"bad point count" in err
    rc, err = mesh(X=2048, Y=2048, Z=511, P=1000, T=big)
    assert rc == -22 and b"bad face count" in err
    assert mesh(P=0, T=0, first=0, points=0, colors=0, normals=0, faces=0)[0] == 0    # nothing to write: no launch

