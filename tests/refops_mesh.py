"""Executable statement of the TSDF mesh (`um_tsdf_mesh_count` / `um_tsdf_mesh`, include/unimatch_sm100.h;
`TSDFVolume.extract_mesh`), in numpy: the faces from the case table of unimatch_b200/csrc/um_mc_table.py, the vertices
and colours of `refops_fusion.extract`, and the normals in float64 and, with `dtype=np.float32`, in the kernels' order of
operations (each fma correctly rounded through `oracle.submission_io.fma32`), bit for bit.  Also exact signed distance
fields of spheres and tori as volumes, and the mesh's topology (edges, Euler characteristic)."""
import numpy as np

import refops_fusion as RF
from oracle.submission_io import fma32
from unimatch_b200.csrc.um_mc_table import MAX_TRIANGLES, edge_corners, triangles

TRIANGLES = [triangles(c) for c in range(256)]
NTRI = np.array([len(t) for t in TRIANGLES])
TABLE = np.zeros((256, MAX_TRIANGLES, 3), np.int64)                  # [cfg, triangle, vertex] edge ids
for _c, _t in enumerate(TRIANGLES):
    if _t:
        TABLE[_c, :len(_t)] = _t
CORNER_OFFSETS = np.array([[(c >> a) & 1 for a in range(3)] for c in range(8)])           # corner -> (dx, dy, dz)
# edge -> (dx, dy, dz, axis): the offset of the voxel that owns it within the cube, and its axis
EDGE_OWNER = np.array([[(edge_corners(e)[0] >> a) & 1 for a in range(3)] + [e >> 2] for e in range(12)])


def _planes(vol, dtype=np.float64):
    return np.asarray(vol["tsdf"], dtype), np.asarray(vol["weight"], dtype)


def crossings(vol):
    """hit [Z, Y, X, 3]: voxel v's edge along axis a emits a point (the predicate of `refops_fusion.extract`)"""
    F, Wt = _planes(vol)
    hit = np.zeros(F.shape + (3,), bool)
    for a in range(3):
        ax = 2 - a
        lo, hi = [slice(None)] * 3, [slice(None)] * 3
        lo[ax], hi[ax] = slice(0, -1), slice(1, None)
        F0, F1, W0, W1 = F[tuple(lo)], F[tuple(hi)], Wt[tuple(lo)], Wt[tuple(hi)]
        hit[tuple(lo) + (a,)] = (W0 > 0) & (W1 > 0) & ((F0 < 0) != (F1 < 0))
    return hit


def cube_cases(vol):
    """(cfg, complete) per cube [Z-1, Y-1, X-1]: the configuration bits (F < 0 per corner) and whether all 8 corners are
    observed"""
    F, Wt = _planes(vol)
    Z, Y, X = F.shape
    cfg = np.zeros((max(Z - 1, 0), max(Y - 1, 0), max(X - 1, 0)), np.int64)
    complete = np.ones(cfg.shape, bool)
    for c, (dx, dy, dz) in enumerate(CORNER_OFFSETS):
        sl = (slice(dz, dz + Z - 1), slice(dy, dy + Y - 1), slice(dx, dx + X - 1))
        cfg |= (F[sl] < 0).astype(np.int64) << c
        complete &= Wt[sl] > 0
    return cfg, complete


def faces(vol):
    """int32 [T, 3] vertex indices into `refops_fusion.extract`'s points, by cube linear index, then table order"""
    hit = crossings(vol)
    index = (np.cumsum(hit.reshape(-1)) - 1).reshape(hit.shape)     # vertex index per (voxel, axis) where hit
    cfg, complete = cube_cases(vol)
    n = np.where(complete, NTRI[cfg], 0)
    k, j, i = np.nonzero(n)                                          # C order = cube linear index order
    edges = TABLE[cfg[k, j, i]]                                      # [m, 5, 3]
    own = EDGE_OWNER[edges]                                          # [m, 5, 3, 4]
    at = (k[:, None, None] + own[..., 2], j[:, None, None] + own[..., 1], i[:, None, None] + own[..., 0], own[..., 3])
    used = np.arange(MAX_TRIANGLES)[None, :] < n[k, j, i][:, None]
    assert hit[at][used].all()
    idx = index[at]
    return idx[used].astype(np.int32).reshape(-1, 3)


def _fma(a, b, c, dtype):
    return fma32(a, b, c) if dtype == np.float32 else a * b + c


def gradients(vol, dtype=np.float64):
    """g [Z, Y, X, 3]: per voxel and axis, the central difference over the neighbours inside the grid and observed, the
    one-sided difference when only one is, else 0"""
    F, Wt = _planes(vol, dtype)
    g = np.zeros(F.shape + (3,), dtype)
    with np.errstate(invalid="ignore", over="ignore"):
        for a in range(3):
            ax = 2 - a
            Fm, Fp = np.zeros_like(F), np.zeros_like(F)
            lo, hi = np.zeros(F.shape, bool), np.zeros(F.shape, bool)
            a0, a1 = [slice(None)] * 3, [slice(None)] * 3
            a0[ax], a1[ax] = slice(0, -1), slice(1, None)
            a0, a1 = tuple(a0), tuple(a1)
            Fm[a1], lo[a1] = F[a0], Wt[a0] > 0                      # v- of voxel v is v - e_a
            Fp[a0], hi[a0] = F[a1], Wt[a1] > 0
            g[..., a] = np.where(lo & hi, (Fp - Fm) * dtype(0.5), np.where(hi, Fp - F, np.where(lo, F - Fm, dtype(0))))
    return g


def normals(vol, dtype=np.float64):
    """[P, 3] unit normals of the vertices, in `refops_fusion.extract`'s order"""
    F, _ = _planes(vol, dtype)
    hit = crossings(vol)
    g = gradients(vol, dtype)
    per_axis = []
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        for a in range(3):
            ax = 2 - a
            a0, a1 = [slice(None)] * 3, [slice(None)] * 3
            a0[ax], a1[ax] = slice(0, -1), slice(1, None)
            a0, a1 = tuple(a0), tuple(a1)
            s = np.zeros(F.shape, dtype)
            s[a0] = np.where(hit[a0 + (a,)], F[a0] / (F[a0] - F[a1]), 0)
            g0, g1 = g, np.zeros_like(g)
            g1[a0] = g[a1]
            n = _fma(s[..., None], g1 - g0, g0, dtype).astype(dtype)
            l2 = _fma(n[..., 1], n[..., 1], n[..., 0] * n[..., 0], dtype).astype(dtype)
            l2 = _fma(n[..., 2], n[..., 2], l2, dtype).astype(dtype)
            length = np.sqrt(l2)[..., None]
            per_axis.append(np.where(length == 0, dtype(0), n / length).astype(dtype))
    return np.stack(per_axis, -2).reshape(-1, 3, 3)[hit.reshape(-1, 3)]


def mesh(vol, origin, voxel_size, dtype=np.float64):
    """(points, colors, normals, faces) of `TSDFVolume.extract_mesh` on the volume's planes"""
    pts, cols = RF.extract(vol, origin, voxel_size, dtype)
    return pts, cols, normals(vol, dtype), faces(vol)


# ---- analytic fields and topology ------------------------------------------------------------------------------------
def sdf_volume(sdf, origin, voxel_size, dims, trunc):
    """The volume of an exact signed distance field sdf(x [..., 3]) -> [...], truncated as integration truncates it:
    F = min(1, sdf / trunc), observed (weight 1) wherever sdf >= -trunc, grey colour"""
    px, py, pz = RF.centres(origin, voxel_size, dims)
    d = sdf(np.stack([px, py, pz], -1))
    Z, Y, X = d.shape
    return {"tsdf": np.where(d >= -trunc, np.minimum(1.0, d / trunc), 0.0), "weight": (d >= -trunc).astype(np.float64),
            "color": np.full((3, Z, Y, X), 128.0)}


def sphere(centre, radius):
    return lambda x: np.linalg.norm(x - np.asarray(centre), axis=-1) - radius


def torus(centre, major, minor):
    """A torus about the z axis through `centre`"""
    def f(x):
        d = x - np.asarray(centre)
        return np.hypot(np.hypot(d[..., 0], d[..., 1]) - major, d[..., 2]) - minor
    return f


def edge_counts(tris):
    """{(a, b): number of faces with the directed edge a -> b}"""
    tris = np.asarray(tris, np.int64)
    directed = np.concatenate([tris[:, [0, 1]], tris[:, [1, 2]], tris[:, [2, 0]]])
    keys, counts = np.unique(directed, axis=0, return_counts=True)
    return {(int(a), int(b)): int(c) for (a, b), c in zip(keys, counts)}


def unmatched_edges(tris):
    """Directed edges a -> b in more faces than b -> a: the mesh's boundary (none: the mesh is closed)"""
    ec = edge_counts(tris)
    return [e for e, c in ec.items() if c > ec.get((e[1], e[0]), 0)]


def is_closed_manifold(tris):
    """Every undirected edge in exactly two faces, once in each direction"""
    ec = edge_counts(tris)
    return all(c == 1 and ec.get((e[1], e[0]), 0) == 1 for e, c in ec.items())


def euler_characteristic(tris):
    tris = np.asarray(tris, np.int64)
    edges = np.unique(np.sort(np.concatenate([tris[:, [0, 1]], tris[:, [1, 2]], tris[:, [2, 0]]]), 1), axis=0)
    return len(np.unique(tris)) - len(edges) + len(tris)
