"""Executable statement of the mesh rasteriser (`um_mesh_bin_count` / `um_mesh_bin` / `um_mesh_ranges` /
`um_mesh_raster`, include/unimatch_sm100.h; `render_mesh`), of `visible_points` (`um_visible_points`) and of
`depth_metrics` (`um_depth_metrics`), in numpy: brute force over all faces per pixel, with each face's fp64 pixel
rectangle applied (or, with `rect=False`, dropped).

`dtype=np.float32` evaluates the rasteriser in the kernel's order of operations (each fma correctly rounded through
`oracle.submission_io.fma32`, every other operation an IEEE float32 operation), so it is what the kernel computes bit for
bit.  `dtype=np.float64` is the same statement in float64, which the accuracy tests compare with.  Also the test meshes:
icospheres, a room box, and helpers for cameras.
"""
import numpy as np

from oracle.submission_io import fma32

TILE = 16


def _fma(a, b, c, dtype):
    return fma32(a, b, c) if dtype == np.float32 else np.asarray(a * b + c, dtype)


def camera_vertices(points, M, dtype=np.float32):
    """V [P, 3]: the points through the world-to-camera rows M [3, 4], in um_tsdf_integrate's order"""
    p = np.asarray(points, dtype)
    M = np.asarray(M, dtype)
    return np.stack([_fma(M[r, 2], p[:, 2], _fma(M[r, 1], p[:, 1], _fma(M[r, 0], p[:, 0], M[r, 3], dtype), dtype), dtype)
                     for r in range(3)], -1).astype(dtype)


def _cross(a, b, dtype):
    return np.stack([(a[..., 1] * b[..., 2]).astype(dtype) - (a[..., 2] * b[..., 1]).astype(dtype),
                     (a[..., 2] * b[..., 0]).astype(dtype) - (a[..., 0] * b[..., 2]).astype(dtype),
                     (a[..., 0] * b[..., 1]).astype(dtype) - (a[..., 1] * b[..., 0]).astype(dtype)], -1).astype(dtype)


def face_terms(points, faces, M, dtype=np.float32):
    """(K [T, 3 edges, 3], det [T]): the signed canonical cross products of edges AB, BC, CA and det = A . K_BC"""
    V = camera_vertices(points, M, dtype)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    Ks = []
    with np.errstate(over="ignore", invalid="ignore"):
        for a, b in ((0, 1), (1, 2), (2, 0)):
            i, j = f[:, a], f[:, b]
            lo, hi = np.minimum(i, j), np.maximum(i, j)
            sign = np.where(i <= j, dtype(1), dtype(-1)).astype(dtype)
            Ks.append((_cross(V[lo], V[hi], dtype) * sign[:, None]).astype(dtype))
        K = np.stack(Ks, 1)
        A = V[f[:, 0]]
        det = _fma(A[:, 2], K[:, 1, 2], _fma(A[:, 1], K[:, 1, 1], (A[:, 0] * K[:, 1, 0]).astype(dtype), dtype), dtype)
    return K, det.astype(dtype)


def rectangles(points, faces, M, K, h, w, near, far=np.inf):
    """(x0, x1, y0, y1, ok) [T] of each face's fp64 pixel rectangle (ok False: none) through the rows M (fp32 entries)"""
    p = np.asarray(points, np.float32).astype(np.float64)
    M = np.asarray(M, np.float32).astype(np.float64)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    fx, fy, cx, cy = (float(np.float32(v)) for v in (K[0][0], K[1][1], K[0][2], K[1][2]))
    near, far = float(np.float32(near)), float(np.float32(far))
    c = [((M[r, 0] * p[:, 0] + M[r, 1] * p[:, 1]) + M[r, 2] * p[:, 2]) + M[r, 3] for r in range(3)]
    c = np.stack(c, -1)[f]                                                 # [T, 3 vertices, 3]
    z = c[..., 2]
    ok = ~((z < near).all(1) | (z > far).all(1))
    u0 = np.full(len(f), np.inf)
    u1, v0, v1 = -u0, u0.copy(), -u0
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        def extend(sel, x, y, zz):
            nonlocal u0, u1, v0, v1
            u = fx * (x / zz) + cx
            v = fy * (y / zz) + cy
            u0 = np.where(sel, np.fmin(u0, u), u0)
            u1 = np.where(sel, np.fmax(u1, u), u1)
            v0 = np.where(sel, np.fmin(v0, v), v0)
            v1 = np.where(sel, np.fmax(v1, v), v1)

        for k in range(3):
            P, Q = c[:, k], c[:, (k + 1) % 3]
            pin, qin = P[:, 2] >= near, Q[:, 2] >= near
            extend(pin, P[:, 0], P[:, 1], P[:, 2])
            s = (near - P[:, 2]) / (Q[:, 2] - P[:, 2])
            extend(pin != qin, P[:, 0] + s * (Q[:, 0] - P[:, 0]), P[:, 1] + s * (Q[:, 1] - P[:, 1]), near)
        spans = []
        for lo, hi, n in ((u0, u1, w), (v0, v1, h)):
            a, b = np.floor(lo) - 1.0, np.ceil(hi) + 1.0
            ok &= (b >= 0) & (a <= n - 1) & (a <= b)
            spans.append((np.where(ok, np.fmax(a, 0), 0).astype(np.int64), np.where(ok, np.fmin(b, n - 1), -1).astype(np.int64)))
    return spans[0][0], spans[0][1], spans[1][0], spans[1][1], ok


def bin_entries(points, faces, w2c, K, h, w, near, far=np.inf):
    """The number of tile entries of um_mesh_bin_count over the views of w2c [n, 3, 4]"""
    total = 0
    for M in np.asarray(w2c).reshape(-1, 3, 4):
        x0, x1, y0, y1, ok = rectangles(points, faces, M, K, h, w, near, far)
        total += int((((x1 // TILE) - (x0 // TILE) + 1) * ((y1 // TILE) - (y0 // TILE) + 1))[ok].sum())
    return total


def raster(points, faces, w2c, K, h, w, colors=None, near=0.01, far=np.inf, dtype=np.float32, rect=True, chunk=None):
    """(depth [n, h, w], face int32 [n, h, w], rgb uint8 [n, h, w, 3] or None) of the mesh through the world-to-camera
    rows w2c [n, 3, 4] with intrinsics K at h x w: each pixel's least t over all faces, ties to the least face index"""
    w2c = np.asarray(w2c).reshape(-1, 3, 4)
    n = len(w2c)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    T = len(faces)
    fx, fy, cx, cy = (dtype(np.float32(v)) for v in (K[0][0], K[1][1], K[0][2], K[1][2]))
    near32, far32 = dtype(np.float32(near)), dtype(np.float32(far))
    ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    xs, ys = xs.reshape(-1), ys.reshape(-1)
    xc = ((xs.astype(dtype) - cx) / fx).astype(dtype)
    yc = ((ys.astype(dtype) - cy) / fy).astype(dtype)
    depth = np.zeros((n, h * w), dtype)
    face = np.full((n, h * w), -1, np.int32)
    rgb = np.zeros((n, h * w, 3), np.uint8) if colors is not None else None
    chunk = chunk or max(1, 2 ** 21 // max(h * w, 1))
    for v in range(n):
        if T == 0:
            continue
        Kf, det = face_terms(points, faces, w2c[v].astype(dtype) if dtype == np.float64 else w2c[v], dtype)
        x0, x1, y0, y1, ok = rectangles(points, faces, np.asarray(w2c[v], np.float32), K, h, w, near, far)
        best = np.full(h * w, np.inf, dtype)
        bf = np.full(h * w, -1, np.int64)
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            for f0 in range(0, T, chunk):
                sl = slice(f0, min(T, f0 + chunk))
                E = [_fma(Kf[None, sl, e, 0], xc[:, None], _fma(Kf[None, sl, e, 1], yc[:, None], Kf[None, sl, e, 2], dtype),
                          dtype).astype(dtype) for e in range(3)]
                cover = ((E[0] >= 0) & (E[1] >= 0) & (E[2] >= 0)) | ((E[0] <= 0) & (E[1] <= 0) & (E[2] <= 0))
                S = ((E[0] + E[1]).astype(dtype) + E[2]).astype(dtype)
                t = (det[None, sl] / S).astype(dtype)
                hit = cover & (S != 0) & np.isfinite(t) & (t >= near32) & (t <= far32)
                if rect:
                    hit &= ok[None, sl] & (xs[:, None] >= x0[None, sl]) & (xs[:, None] <= x1[None, sl]) \
                        & (ys[:, None] >= y0[None, sl]) & (ys[:, None] <= y1[None, sl])
                tm = np.where(hit, t, np.inf)
                k = tm.argmin(1)                                  # the first least: the least face index
                tk = tm[np.arange(h * w), k]
                better = tk < best
                best = np.where(better, tk, best)
                bf = np.where(better, f0 + k, bf)
        hitpix = bf >= 0
        depth[v] = np.where(hitpix, best, 0)
        face[v] = bf
        if colors is not None and hitpix.any():
            q = np.nonzero(hitpix)[0]
            fq = bf[q]
            with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
                E = [_fma(Kf[fq, e, 0], xc[q], _fma(Kf[fq, e, 1], yc[q], Kf[fq, e, 2], dtype), dtype).astype(dtype)
                     for e in range(3)]
                S = ((E[0] + E[1]).astype(dtype) + E[2]).astype(dtype)
                ba, bb, bc = ((E[1] / S).astype(dtype), (E[2] / S).astype(dtype), (E[0] / S).astype(dtype))
            col = np.asarray(colors, np.uint8).astype(dtype)
            tri = faces[fq]
            for ch in range(3):
                val = _fma(bc, col[tri[:, 2], ch], _fma(bb, col[tri[:, 1], ch], (ba * col[tri[:, 0], ch]).astype(dtype),
                                                        dtype), dtype)
                rgb[v, q, ch] = np.clip(np.rint(val), 0, 255).astype(np.uint8)
    out = (depth.reshape(n, h, w), face.reshape(n, h, w))
    return out + (rgb.reshape(n, h, w, 3) if rgb is not None else None,)


def visible(points, depths, w2c, K, tolerance=0.05):
    """bool [P]: some view sees the point (um_visible_points), in float32"""
    p = np.asarray(points, np.float32)
    depths = np.asarray(depths, np.float32)
    n, h, w = depths.shape
    fx, fy, cx, cy = (np.float32(v) for v in (K[0][0], K[1][1], K[0][2], K[1][2]))
    tol = np.float32(tolerance)
    seen = np.zeros(len(p), bool)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        for t in range(n):
            V = camera_vertices(p, np.asarray(w2c[t], np.float32), np.float32)
            ok = V[:, 2] > 0
            u = fma32(fx, (V[:, 0] / V[:, 2]).astype(np.float32), cx)
            v = fma32(fy, (V[:, 1] / V[:, 2]).astype(np.float32), cy)
            xf, yf = np.floor(u + np.float32(0.5)), np.floor(v + np.float32(0.5))
            ok &= (xf >= 0) & (xf < np.float32(w)) & (yf >= 0) & (yf < np.float32(h))
            xi, yi = np.where(ok, xf, 0).astype(np.int64), np.where(ok, yf, 0).astype(np.int64)
            D = depths[t][yi, xi]
            seen |= ok & np.isfinite(D) & (D > 0) & (V[:, 2] <= (D + tol).astype(np.float32))
    return seen


def depth_sums(pred, gt, max_depth=10.0):
    """The per-frame sums [N, 10] of um_depth_metrics in float64 (libm logs; any summation order)"""
    pred, gt = np.asarray(pred, np.float32), np.asarray(gt, np.float32)
    md = np.float32(max_depth)
    out = np.zeros((len(pred), 10))
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        for i, (p, g) in enumerate(zip(pred.reshape(len(pred), -1), gt.reshape(len(gt), -1))):
            has = np.isfinite(p) & (p > 0)
            m = has & np.isfinite(g) & (g > 0) & (g < md)
            pm, gm = p[m].astype(np.float64), g[m].astype(np.float64)
            d = pm - gm
            ratio = np.maximum((g[m] / p[m]).astype(np.float32), (p[m] / g[m]).astype(np.float32))
            out[i] = [m.sum(), np.abs(d).sum(), (np.abs(d) / gm).sum(), (d * d / gm).sum(), (d * d).sum(),
                      ((np.log(pm) - np.log(gm)) ** 2).sum(), (ratio < np.float32(1.25)).sum(),
                      (ratio < np.float32(1.5625)).sum(), (ratio < np.float32(1.953125)).sum(), has.sum()]
    return out


# ---- test meshes and cameras -------------------------------------------------------------------------------------------
def icosphere(subdivisions=1, radius=1.0, centre=(0.0, 0.0, 0.0), jitter=0.0, seed=0):
    """(points float32 [P, 3], faces int32 [T, 3]): a subdivided icosahedron, counter-clockwise seen from outside, each
    vertex's radius scaled by 1 + uniform(-jitter, jitter); closed"""
    t = (1 + 5 ** 0.5) / 2
    v = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t), (t, 0, -1),
         (t, 0, 1), (-t, 0, -1), (-t, 0, 1)]
    f = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6),
         (7, 1, 8), (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10), (8, 6, 7),
         (9, 8, 1)]
    verts = [np.asarray(p, float) / np.linalg.norm(p) for p in v]
    for _ in range(subdivisions):
        mid, nf = {}, []

        def m(a, b):
            key = (min(a, b), max(a, b))
            if key not in mid:
                p = verts[a] + verts[b]
                verts.append(p / np.linalg.norm(p))
                mid[key] = len(verts) - 1
            return mid[key]
        for a, b, c in f:
            ab, bc, ca = m(a, b), m(b, c), m(c, a)
            nf += [(a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca)]
        f = nf
    g = np.random.default_rng(seed)
    pts = np.asarray(verts) * (radius * (1 + g.uniform(-jitter, jitter, (len(verts), 1))))
    return (pts + np.asarray(centre)).astype(np.float32), np.asarray(f, np.int32)


def room_box(lo=(-1.0, -1.0, -1.0), hi=(1.0, 1.0, 1.0), n=2):
    """(points, faces) of the box [lo, hi] with each face split into n x n squares of two triangles; closed, faces
    counter-clockwise seen from inside"""
    lo, hi = np.asarray(lo, float), np.asarray(hi, float)
    pts, tris, index = [], [], {}

    def vid(q):
        key = tuple(q)
        if key not in index:
            index[key] = len(pts)
            pts.append(lo + (hi - lo) * np.asarray(q, float) / n)
        return index[key]
    for axis in range(3):
        u, v = (axis + 1) % 3, (axis + 2) % 3
        for side in (0, n):
            for i in range(n):
                for j in range(n):
                    q = []
                    for di, dj in ((0, 0), (1, 0), (1, 1), (0, 1)):
                        c = [0, 0, 0]
                        c[axis], c[u], c[v] = side, i + di, j + dj
                        q.append(vid(c))
                    a, b, c, d = q if side == 0 else q[::-1]
                    tris += [(a, b, c), (a, c, d)]
    return np.asarray(pts, np.float32), np.asarray(tris, np.int32)


def look_at(eye, target, up=(0.0, 0.0, 1.0)):
    """Camera-to-world [4, 4] float64 of a camera at eye looking at target (camera y down)"""
    eye, target = np.asarray(eye, float), np.asarray(target, float)
    z = target - eye
    z /= np.linalg.norm(z)
    x = np.cross(z, np.asarray(up, float))
    if np.linalg.norm(x) < 1e-9:
        x = np.cross(z, [1.0, 0.0, 0.0])
    x /= np.linalg.norm(x)
    P = np.eye(4)
    P[:3, 0], P[:3, 1], P[:3, 2], P[:3, 3] = x, np.cross(z, x), z, eye
    return P


def random_rotation(g):
    q = g.normal(size=4)
    q /= np.linalg.norm(q)
    a, b, c, d = q
    return np.array([[a * a + b * b - c * c - d * d, 2 * (b * c - a * d), 2 * (b * d + a * c)],
                     [2 * (b * c + a * d), a * a - b * b + c * c - d * d, 2 * (c * d - a * b)],
                     [2 * (b * d - a * c), 2 * (c * d + a * b), a * a - b * b - c * c + d * d]])


def pose(R, centre):
    P = np.eye(4)
    P[:3, :3], P[:3, 3] = R, centre
    return P
