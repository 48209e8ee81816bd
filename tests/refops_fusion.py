"""Executable statement of TSDF fusion (`um_tsdf_integrate`, `um_tsdf_surface_count` / `um_tsdf_surface_points`,
include/unimatch_sm100.h; `fuse_depths`, `TSDFVolume` and `DepthFusionRunner` in unimatch_b200), in numpy, and exact
float64 depth maps of analytic scenes seen from rotated cameras.

`dtype=np.float64` is the statement the analytic tests compare with.  `dtype=np.float32` evaluates it in the kernels' order
of operations (each fma correctly rounded through `oracle.submission_io.fma32`, every other operation an IEEE float32
operation), so it is what the kernels compute bit for bit.
"""
import numpy as np

from oracle.submission_io import fma32


def _fma(a, b, c, dtype):
    return fma32(a, b, c) if dtype == np.float32 else a * b + c


def centres(origin, voxel_size, dims, dtype=np.float64):
    """Voxel centres per axis: fma(idx + 0.5, voxel_size, origin) -> (px, py, pz), each [Z, Y, X]"""
    ax = [_fma(np.arange(n).astype(dtype) + dtype(0.5), dtype(voxel_size), dtype(o), dtype).astype(dtype)
          for n, o in zip(dims, origin)]
    pz, py, px = np.meshgrid(ax[2], ax[1], ax[0], indexing="ij")
    return px, py, pz


def empty_volume(dims, dtype=np.float64):
    X, Y, Z = dims
    return {"tsdf": np.zeros((Z, Y, X), dtype), "weight": np.zeros((Z, Y, X), dtype), "color": np.zeros((3, Z, Y, X), dtype)}


def integrate(vol, origin, voxel_size, trunc, depths, frames, w2c, K, dtype=np.float64, n_valid=None):
    """Fuses frames 0 .. n_valid - 1 of depths [n, h, w], uint8 frames [n, h, w, 3] and world-to-camera rows w2c
    [n, 3, 4] into `vol` (a dict of tsdf / weight [Z, Y, X] and color [3, Z, Y, X]); returns the new volume."""
    depths, w2c = np.asarray(depths, dtype), np.asarray(w2c, dtype)
    frames = np.asarray(frames)
    n, h, w = depths.shape
    n = n if n_valid is None else min(max(int(n_valid), 0), n)
    Z, Y, X = vol["tsdf"].shape
    px, py, pz = centres(origin, voxel_size, (X, Y, Z), dtype)
    fx, fy, cx, cy = (dtype(v) for v in (K[0][0], K[1][1], K[0][2], K[1][2]))
    trunc = dtype(trunc)
    F, Wt = vol["tsdf"].astype(dtype), vol["weight"].astype(dtype)
    C = vol["color"].astype(dtype)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        for t in range(n):
            M = w2c[t]
            c = [_fma(M[r, 2], pz, _fma(M[r, 1], py, _fma(M[r, 0], px, M[r, 3], dtype), dtype), dtype) for r in range(3)]
            ok = c[2] > 0
            u = _fma(fx, c[0] / c[2], cx, dtype)
            v = _fma(fy, c[1] / c[2], cy, dtype)
            xf, yf = np.floor(u + dtype(0.5)), np.floor(v + dtype(0.5))
            ok &= (xf >= 0) & (xf < w) & (yf >= 0) & (yf < h)
            xi, yi = np.where(ok, xf, 0).astype(np.int64), np.where(ok, yf, 0).astype(np.int64)
            d = depths[t][yi, xi]
            ok &= np.isfinite(d) & (d > 0)
            sdf = d - c[2]
            ok &= ~(sdf < -trunc)
            f = np.minimum(dtype(1), sdf / trunc)
            w1 = Wt + dtype(1)
            F = np.where(ok, _fma(F, Wt, f, dtype) / w1, F).astype(dtype)
            rgb = frames[t][yi, xi].astype(dtype)
            for ch in range(3):
                C[ch] = np.where(ok, _fma(C[ch], Wt, rgb[..., ch], dtype) / w1, C[ch])
            Wt = np.where(ok, w1, Wt).astype(dtype)
    return {"tsdf": F, "weight": Wt, "color": C}


def extract(vol, origin, voxel_size, dtype=np.float64):
    """The zero-crossing points (float [P, 3]) and colours (uint8 [P, 3]) of the volume, ordered by voxel linear index,
    then edge axis x, y, z."""
    F, Wt, C = (np.asarray(vol[k], dtype) for k in ("tsdf", "weight", "color"))
    Z, Y, X = F.shape
    p0 = centres(origin, voxel_size, (X, Y, Z), dtype)
    vs = dtype(voxel_size)
    per_axis = []                      # per axis: (hit [Z, Y, X], point [Z, Y, X, 3], colour [Z, Y, X, 3])
    for a in range(3):
        sl0 = [slice(None)] * 3
        sl1 = [slice(None)] * 3
        ax = 2 - a                     # array axis of world axis a
        sl0[ax], sl1[ax] = slice(0, -1), slice(1, None)
        hit = np.zeros(F.shape, bool)
        s = np.zeros(F.shape, dtype)
        F0, F1, W0, W1 = F[tuple(sl0)], F[tuple(sl1)], Wt[tuple(sl0)], Wt[tuple(sl1)]
        h = (W0 > 0) & (W1 > 0) & ((F0 < 0) != (F1 < 0))
        hit[tuple(sl0)] = h
        with np.errstate(invalid="ignore", divide="ignore"):
            s[tuple(sl0)] = np.where(h, F0 / (F0 - F1), 0)
        pt = np.stack([(_fma(s, vs, p0[q], dtype) if q == a else p0[q]).astype(dtype) for q in range(3)], -1)
        col = np.zeros(F.shape + (3,), np.uint8)
        for ch in range(3):
            c0 = C[ch]
            c1 = np.zeros_like(c0)
            c1[tuple(sl0)] = c0[tuple(sl1)]
            q = np.rint(_fma(s, c1 - c0, c0, dtype))
            col[..., ch] = np.clip(q, 0, 255).astype(np.uint8)
        per_axis.append((hit, pt, col))
    hits = np.stack([p[0] for p in per_axis], -1).reshape(-1, 3)          # [voxel, axis]
    pts = np.stack([p[1] for p in per_axis], -2).reshape(-1, 3, 3)
    cols = np.stack([p[2] for p in per_axis], -2).reshape(-1, 3, 3)
    return pts[hits], cols[hits]


# ---- analytic scenes ------------------------------------------------------------------------------------------------
def rot(axis, angle):
    """Rotation matrix about axis 'x', 'y' or 'z'"""
    c, s = np.cos(angle), np.sin(angle)
    i, j = {"x": (1, 2), "y": (2, 0), "z": (0, 1)}[axis]
    R = np.eye(3)
    R[i, i], R[i, j], R[j, i], R[j, j] = c, -s, s, c
    return R


def pose(R, centre):
    """Camera-to-world [4, 4] (float64) of a camera at `centre` with rotation R (columns: camera axes in the world)"""
    P = np.eye(4)
    P[:3, :3], P[:3, 3] = R, centre
    return P


def rays(K, h, w, du=0.0, dv=0.0):
    """Camera-frame ray directions with z = 1 through pixel centres (x + du, y + dv): [h, w, 3] float64"""
    ys, xs = np.meshgrid(np.arange(h) + dv, np.arange(w) + du, indexing="ij")
    return np.stack([(xs - K[0][2]) / K[0][0], (ys - K[1][2]) / K[1][1], np.ones_like(xs)], -1)


def render(scene, K, P, h, w, du=0.0, dv=0.0):
    """Exact float64 z-depth [h, w] of `scene` along the pixel-centre rays of camera P (0 where a ray misses it).
    scene: ('plane', n, c) for {x: n.x = c}, or ('sphere', centre, radius) (the near intersection)."""
    r = rays(K, h, w, du, dv) @ P[:3, :3].T              # world directions, camera z-component 1
    C = P[:3, 3]
    if scene[0] == "plane":
        n, c = np.asarray(scene[1], float), float(scene[2])
        with np.errstate(divide="ignore", invalid="ignore"):
            t = (c - n @ C) / (r @ n)
    else:
        s, R = np.asarray(scene[1], float), float(scene[2])
        oc = C - s
        a, b, cc = (r * r).sum(-1), 2 * (r @ oc), oc @ oc - R * R
        disc = b * b - 4 * a * cc
        with np.errstate(invalid="ignore"):
            t = (-b - np.sqrt(disc)) / (2 * a)
    return np.where(np.isfinite(t) & (t > 0), t, 0.0)    # t is the z-depth: the camera-frame ray has z = 1


def normal_at(scene, x):
    """Unit surface normal at world points x [..., 3]"""
    if scene[0] == "plane":
        n = np.asarray(scene[1], float)
        return np.broadcast_to(n / np.linalg.norm(n), x.shape)
    d = x - np.asarray(scene[1], float)
    return d / np.linalg.norm(d, axis=-1, keepdims=True)


def distance(scene, x):
    """Unsigned Euclidean distance of world points x [..., 3] to the surface"""
    if scene[0] == "plane":
        n = np.asarray(scene[1], float)
        return np.abs(x @ n - scene[2]) / np.linalg.norm(n)
    return np.abs(np.linalg.norm(x - np.asarray(scene[1], float), axis=-1) - scene[2])


def constant_plane_clip(n=5, h=24, w=32, z0=1.0, cam_z=-0.5, seed=0):
    """The plane z = z0 seen by cameras whose optical axis is world +z, rolled about it by random angles and translated
    parallel to the plane: every depth map is the constant z0 - cam_z.  Returns (scene, K, poses [n, 4, 4] float64)."""
    g = np.random.default_rng(seed)
    K = [[0.8 * w, 0, w / 2], [0, 0.8 * w, h / 2], [0, 0, 1]]
    poses = [pose(rot("z", g.uniform(-np.pi, np.pi)), [g.uniform(-0.1, 0.1), g.uniform(-0.1, 0.1), cam_z]) for _ in range(n)]
    return ("plane", [0.0, 0.0, 1.0], z0), K, np.stack(poses)


def tilted_plane_clip(n=5, h=48, w=64, seed=1):
    """A plane tilted by 25 degrees about x and 15 about y, 1.4 m in front of cameras rotated by up to 8 degrees about each
    axis around a common look direction: every pixel sees the plane."""
    g = np.random.default_rng(seed)
    K = [[2.0 * w, 0, w / 2], [0, 2.0 * w, h / 2], [0, 0, 1]]
    nrm = rot("y", np.radians(15)) @ rot("x", np.radians(25)) @ np.array([0.0, 0.0, -1.0])
    poses = []
    for _ in range(n):
        R = rot("z", g.uniform(-0.14, 0.14)) @ rot("y", g.uniform(-0.14, 0.14)) @ rot("x", g.uniform(-0.14, 0.14))
        poses.append(pose(R, g.uniform(-0.08, 0.08, 3)))
    c = nrm @ np.array([0.0, 0.0, 1.4])
    return ("plane", nrm.tolist(), float(c)), K, np.stack(poses)


def sphere_clip(n=5, h=48, w=64, seed=2):
    """A sphere of radius 1 centred 2.2 m in front of cameras rotated by up to 6 degrees about each axis: the sphere
    fills every frame (no silhouette; every ray is within 24 degrees of the centre direction)."""
    g = np.random.default_rng(seed)
    K = [[2.0 * w, 0, w / 2], [0, 2.0 * w, h / 2], [0, 0, 1]]
    poses = []
    for _ in range(n):
        R = rot("z", g.uniform(-0.1, 0.1)) @ rot("y", g.uniform(-0.1, 0.1)) @ rot("x", g.uniform(-0.1, 0.1))
        poses.append(pose(R, g.uniform(-0.05, 0.05, 3)))
    return ("sphere", [0.0, 0.0, 2.2], 1.0), K, np.stack(poses)


def footprint_error(scene, K, poses, h, w, lo, hi):
    """Over the pixels of all frames whose surface point lies in the box [lo, hi] (the part of the scene a volume there
    can fuse), E: the largest change of the exact depth between a pixel centre and the corners of its pixel square
    (the nearest-pixel lookup reads a depth at most half a pixel from the voxel's own ray in each direction; the depth is
    smooth, so its extreme over the square sits at a corner up to second-order terms), and the range (a_min, a_max) of
    the projective scale a = cos(beta) / cos(phi) by which the z-depth difference d - z near the surface exceeds the
    Euclidean distance (beta: ray to optical axis, phi: ray to the surface normal)."""
    E, a_lo, a_hi = 0.0, np.inf, 0.0
    for P in poses:
        d = render(scene, K, P, h, w)
        r = rays(K, h, w) @ P[:3, :3].T
        x = P[:3, 3] + r * d[..., None]
        inside = (d > 0) & (x >= np.asarray(lo)).all(-1) & (x <= np.asarray(hi)).all(-1)
        if not inside.any():
            continue
        for du in (-0.5, 0.5):
            for dv in (-0.5, 0.5):
                E = max(E, float(np.abs(render(scene, K, P, h, w, du, dv) - d)[inside].max()))
        ru = r / np.linalg.norm(r, axis=-1, keepdims=True)
        cos_beta = ru @ P[:3, 2]
        cos_phi = np.abs((ru * normal_at(scene, x)).sum(-1))
        a = (cos_beta / cos_phi)[inside]
        a_lo, a_hi = min(a_lo, float(a.min())), max(a_hi, float(a.max()))
    return E, a_lo, a_hi
