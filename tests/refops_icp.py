"""Executable statement of ICP tracking against the TSDF volume (`um_icp_*`, include/unimatch_sm100.h;
`TSDFVolume.track` and `DepthFusionRunner(track=True)` in unimatch_b200), in numpy, and analytic scenes made of several
primitives (`render_union`, the corner clip).

`dtype=np.float32` evaluates the per-pixel arithmetic (pyramid, live normals, association and the per-pixel terms) in the
kernels' order of operations (each fma correctly rounded through `oracle.submission_io.fma32`, every other operation an
IEEE float32 operation), so it is what the kernels compute bit for bit; `dtype=np.float64` is the same statement in float64.
The sums (fp64, in the kernels' order), the solve and the pose update are float64 either way.  The model maps are
`refops_render.raycast` at the same dtype.
"""
import math

import numpy as np

import refops_fusion as RF
import refops_render as RR
from oracle.submission_io import fma32

TERMS, STATE = 30, 32
MIN_INLIERS, MIN_PIVOT = 36.0, 1e-2
TX, TY = 16, 8


def _fma(a, b, c, dtype):
    return fma32(a, b, c) if dtype == np.float32 else np.asarray(a * b + c, dtype)


def _valid(d):
    return np.isfinite(d) & (d > 0)


# ---- pyramid and live normals ----------------------------------------------------------------------------------------
def levels(K, h, w, n_levels):
    """[(fx, fy, cx, cy, h, w)] per level, finest first: fx/2, fy/2, (cx - 0.5)/2, (cy - 0.5)/2 in float32"""
    f = np.float32
    fx, fy, cx, cy = f(K[0][0]), f(K[1][1]), f(K[0][2]), f(K[1][2])
    out = [(fx, fy, cx, cy, h, w)]
    for _ in range(n_levels - 1):
        fx, fy, cx, cy = f(fx * f(0.5)), f(fy * f(0.5)), f(f(cx - f(0.5)) * f(0.5)), f(f(cy - f(0.5)) * f(0.5))
        h, w = h // 2, w // 2
        out.append((fx, fy, cx, cy, h, w))
    return out


def downsample(depth, trunc, dtype=np.float32):
    """The next level of depths [n, h, w]: per 2 x 2 block, the mean of its valid depths within trunc of the smallest"""
    d = np.asarray(depth, dtype)
    n, h, w = d.shape
    h2, w2 = h // 2, w // 2
    q = [d[:, dy:2 * h2:2, dx:2 * w2:2] for dy, dx in ((0, 0), (0, 1), (1, 0), (1, 1))]
    ok = [_valid(v) for v in q]
    lo = np.full((n, h2, w2), np.inf, dtype)
    for v, o in zip(q, ok):
        lo = np.where(o, np.fmin(lo, v), lo)
    s, c = np.zeros((n, h2, w2), dtype), np.zeros((n, h2, w2), dtype)
    with np.errstate(invalid="ignore"):
        for v, o in zip(q, ok):
            use = o & ((v - lo).astype(dtype) <= dtype(trunc))
            s = np.where(use, (s + v).astype(dtype), s)
            c = c + use
        return np.where(c > 0, (s / np.maximum(c, 1)).astype(dtype), dtype(0)).astype(dtype)


def _xc(x, c, f, dtype):
    return ((np.asarray(x, dtype) - dtype(c)).astype(dtype) / dtype(f)).astype(dtype)


def vertices(depth, fx, fy, cx, cy, dtype=np.float32):
    """v [n, h, w, 3]: (d (x - cx) / fx, d (y - cy) / fy, d)"""
    d = np.asarray(depth, dtype)
    n, h, w = d.shape
    xs, ys = _xc(np.arange(w), cx, fx, dtype), _xc(np.arange(h), cy, fy, dtype)
    with np.errstate(invalid="ignore", over="ignore"):                  # non-finite depths are invalid pixels
        return np.stack([(d * xs[None, None, :]).astype(dtype), (d * ys[None, :, None]).astype(dtype), d], -1)


def _cross(a, b, dtype):
    return np.stack([(a[..., j] * b[..., k]).astype(dtype) - (a[..., k] * b[..., j]).astype(dtype)
                     for j, k in ((1, 2), (2, 0), (0, 1))], -1).astype(dtype)


def _dot(a, b, dtype):
    """fma(a.z, b.z, fma(a.y, b.y, a.x * b.x))"""
    return _fma(a[..., 2], b[..., 2], _fma(a[..., 1], b[..., 1], (a[..., 0] * b[..., 0]).astype(dtype), dtype), dtype)


def normals(depth, fx, fy, cx, cy, dtype=np.float32):
    """Live normals [n, h, w, 3]: (v(x+1, y) - v) x (v(x, y+1) - v), unit, with n.v <= 0; 0 where invalid"""
    d = np.asarray(depth, dtype)
    v = vertices(d, fx, fy, cx, cy, dtype)
    out = np.zeros(v.shape, dtype)
    ok = _valid(d[:, :-1, :-1]) & _valid(d[:, :-1, 1:]) & _valid(d[:, 1:, :-1])
    v0 = v[:, :-1, :-1]
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        c = _cross((v[:, :-1, 1:] - v0).astype(dtype), (v[:, 1:, :-1] - v0).astype(dtype), dtype)
        length = np.sqrt(_dot(c, c, dtype)).astype(dtype)
        facing = _dot(c, v0, dtype)
        ok &= (length > 0) & np.isfinite(length)
        s = np.where(facing > 0, -length, length)
        out[:, :-1, :-1] = np.where(ok[..., None], (c / s[..., None]).astype(dtype), dtype(0))
    return out


# ---- state, association and the per-pixel terms ----------------------------------------------------------------------
def rigid_inverse_rows(m):
    """fp32 [3, 4] rows of the rigid inverse of fp64 rows m [3, 4]: (R^T, -((R_0i t_0 + R_1i t_1) + R_2i t_2))"""
    out = np.empty((3, 4), np.float32)
    out[:, :3] = m[:, :3].T
    for i in range(3):
        out[i, 3] = np.float32(-((m[0, i] * m[0, 3] + m[1, i] * m[1, 3]) + m[2, i] * m[2, 3]))
    return out


def _times(C, P):
    """Rows [3, 4] of C P for fp64 rows C, P [3, 4] (bottom rows 0 0 0 1): ((C_i0 P_0j + C_i1 P_1j) + C_i2 P_2j) (+ C_i3)"""
    out = np.empty((3, 4))
    for i in range(3):
        for j in range(4):
            v = (C[i, 0] * P[0, j] + C[i, 1] * P[1, j]) + C[i, 2] * P[2, j]
            out[i, j] = v + C[i, 3] if j == 3 else v
    return out


def init(poses, correction=None):
    """State of fp64 poses [n, 4, 4]: {'T', 'ref': fp64 [n, 3, 4], 'degenerate': [n]}, and c2w / w2c fp32 [n, 3, 4]"""
    P = np.asarray(poses, np.float64)[:, :3]
    ref = P.copy() if correction is None else np.stack([_times(np.asarray(correction, np.float64)[:3], p) for p in P])
    c2w = ref.astype(np.float32)
    w2c = np.stack([rigid_inverse_rows(r) for r in ref])
    return {"T": ref.copy(), "ref": ref, "degenerate": np.zeros(len(P), np.int64)}, c2w, w2c


def pixel_terms(depth, live_normal, model_depth, model_normal, T, c2w, w2c, fx, fy, cx, cy, max_distance, cos_max_angle,
                dtype=np.float32):
    """Per live pixel: the terms [n, h, w, 30] (float64 values of the per-pixel products) at the estimates T (fp64 rows
    [n, 3, 4], rounded to dtype), with the reference rows c2w / w2c [n, 3, 4]."""
    d = np.asarray(depth, dtype)
    n, h, w = d.shape
    nl = np.asarray(live_normal, dtype)
    valid = _valid(d) & (nl != 0).any(-1)
    v = vertices(d, fx, fy, cx, cy, dtype)
    Tf = np.asarray(T).astype(dtype)
    M, V = np.asarray(c2w, dtype), np.asarray(w2c, dtype)
    fx, fy, cx, cy = (dtype(x) for x in (fx, fy, cx, cy))
    terms = np.zeros((n, h, w, TERMS))
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        for f in range(n):
            R = Tf[f]
            p = np.stack([_fma(R[a, 2], v[f, ..., 2], _fma(R[a, 1], v[f, ..., 1], _fma(R[a, 0], v[f, ..., 0], R[a, 3], dtype),
                                                          dtype), dtype) for a in range(3)], -1)
            nw = np.stack([_fma(R[a, 2], nl[f, ..., 2], _fma(R[a, 1], nl[f, ..., 1], (R[a, 0] * nl[f, ..., 0]).astype(dtype),
                                                            dtype), dtype) for a in range(3)], -1)
            c = [_fma(V[f, a, 2], p[..., 2], _fma(V[f, a, 1], p[..., 1], _fma(V[f, a, 0], p[..., 0], V[f, a, 3], dtype),
                                                  dtype), dtype) for a in range(3)]
            ok = valid[f] & (c[2] > 0)
            u = _fma(fx, (c[0] / c[2]).astype(dtype), cx, dtype)
            vv = _fma(fy, (c[1] / c[2]).astype(dtype), cy, dtype)
            xf, yf = np.floor((u + dtype(0.5)).astype(dtype)), np.floor((vv + dtype(0.5)).astype(dtype))
            ok &= (xf >= 0) & (xf < w) & (yf >= 0) & (yf < h)
            xi, yi = np.where(ok, xf, 0).astype(np.int64), np.where(ok, yf, 0).astype(np.int64)
            D = np.asarray(model_depth, dtype)[f][yi, xi]
            m = np.asarray(model_normal, dtype)[f][yi, xi]
            ok &= (D > 0) & (m != 0).any(-1)
            xc = ((xi.astype(dtype) - cx).astype(dtype) / fx).astype(dtype)
            yc = ((yi.astype(dtype) - cy).astype(dtype) / fy).astype(dtype)
            e, pc = [], []
            for a in range(3):
                direction = _fma(M[f, a, 0], xc, _fma(M[f, a, 1], yc, M[f, a, 2], dtype), dtype)
                e.append((p[..., a] - _fma(D, direction, M[f, a, 3], dtype)).astype(dtype))
                pc.append((p[..., a] - M[f, a, 3]).astype(dtype))
            e, pc = np.stack(e, -1), np.stack(pc, -1)
            dist = np.sqrt(_dot(e, e, dtype)).astype(dtype)
            ok &= (dist <= dtype(max_distance)) & (_dot(nw, m, dtype) >= dtype(cos_max_angle))
            r = _dot(m, e, dtype)
            a = np.concatenate([_cross(pc, m, dtype), m], -1)
            k = 0
            for i in range(6):
                for j in range(i, 6):
                    terms[f, ..., k] = np.where(ok, (a[..., i] * a[..., j]).astype(dtype), 0)
                    k += 1
            for i in range(6):
                terms[f, ..., 21 + i] = np.where(ok, (a[..., i] * r).astype(dtype), 0)
            terms[f, ..., 27] = np.where(ok, (r * r).astype(dtype), 0)
            terms[f, ..., 28] = ok
            terms[f, ..., 29] = valid[f]
    return terms


def block_partials(terms):
    """[n, nb, 30] fp64 per-block sums of terms [n, h, w, 30] in the kernel's order: 16 x 8 tiles, thread
    ty * 16 + tx, a shfl_down tree (16, 8, 4, 2, 1) per warp, then the 4 warps in order"""
    n, h, w, _ = terms.shape
    gy, gx = -(-h // TY), -(-w // TX)
    t = np.zeros((n, gy * TY, gx * TX, TERMS))
    t[:, :h, :w] = terms
    t = t.reshape(n, gy, TY, gx, TX, TERMS).transpose(0, 1, 3, 2, 4, 5).reshape(n, gy * gx, 4, 32, TERMS)
    o = 16
    while o:
        t = t[..., :o, :] + t[..., o:2 * o, :]
        o //= 2
    t = t[..., 0, :]
    s = t[:, :, 0]
    for q in range(1, 4):
        s = s + t[:, :, q]
    return s


def sums(partials):
    """[n, 30]: the block partials [n, nb, 30] summed as the kernels do, one warp per term: lane l adds blocks l, l + 32,
    ... in order from 0.0, then a shfl_down tree (16, 8, 4, 2, 1) adds the lanes"""
    n, nb, _ = partials.shape
    s = np.zeros((n, 32, TERMS))
    for j in range(0, nb, 32):
        m = min(32, nb - j)
        s[:, :m] = s[:, :m] + partials[:, j:j + m]
    o = 16
    while o:
        s = s[:, :o] + s[:, o:2 * o]
        o //= 2
    return s[:, 0]


def system(S):
    """(A [6, 6], b [6]) of one frame's sums"""
    A = np.zeros((6, 6))
    k = 0
    for i in range(6):
        for j in range(i, 6):
            A[i, j] = A[j, i] = S[k]
            k += 1
    return A, S[21:27].copy()


def _scale(A):
    """Jacobi scaling: 1 / sqrt(A_ii), or 1 where A_ii is not > 0"""
    dg = np.diag(A)
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(dg > 0, 1.0 / np.sqrt(np.where(dg > 0, dg, 1.0)), 1.0)


def scaled_pivots(S):
    """The Cholesky pivots of the Jacobi-scaled system, in the kernel's order (NaN where the scaling fails)"""
    A, _ = system(S)
    sc = _scale(A)
    L = np.zeros((6, 6))
    piv = np.full(6, np.nan)
    for j in range(6):
        d = (A[j, j] * sc[j]) * sc[j]
        for k in range(j):
            d = d - L[j, k] * L[j, k]
        piv[j] = d
        if not d >= MIN_PIVOT:
            break
        L[j, j] = math.sqrt(d)
        for i in range(j + 1, 6):
            e = (A[i, j] * sc[i]) * sc[j]
            for k in range(j):
                e = e - L[i, k] * L[j, k]
            L[i, j] = e / L[j, j]
    return piv


def solve_step(S, min_inliers=MIN_INLIERS, min_pivot=MIN_PIVOT):
    """The step x = (w, tau) of one frame's sums, or None when the system is degenerate"""
    A, b = system(S)
    if not S[28] >= min_inliers:
        return None
    sc = _scale(A)
    L = np.zeros((6, 6))
    for j in range(6):
        d = (A[j, j] * sc[j]) * sc[j]
        for k in range(j):
            d = d - L[j, k] * L[j, k]
        if not d >= min_pivot:
            return None
        L[j, j] = math.sqrt(d)
        for i in range(j + 1, 6):
            e = (A[i, j] * sc[i]) * sc[j]
            for k in range(j):
                e = e - L[i, k] * L[j, k]
            L[i, j] = e / L[j, j]
    x = np.zeros(6)
    for i in range(6):
        e = -(b[i] * sc[i])
        for k in range(i):
            e = e - L[i, k] * x[k]
        x[i] = e / L[i, i]
    for i in range(5, -1, -1):
        e = x[i]
        for k in range(i + 1, 6):
            e = e - L[k, i] * x[k]
        x[i] = e / L[i, i]
    return x * sc


def apply_step(T, ref, x):
    """T <- dT T: dR = exp(w) (Rodrigues) about the reference centre, then tau"""
    th = math.sqrt((x[0] * x[0] + x[1] * x[1]) + x[2] * x[2])
    R = np.eye(3)
    if th > 0:
        k = x[:3] / th
        c, s = math.cos(th), math.sin(th)
        v = 1.0 - c
        Kx = np.array([[0.0, -k[2], k[1]], [k[2], 0.0, -k[0]], [-k[1], k[0], 0.0]])
        for i in range(3):
            for j in range(3):
                R[i, j] = ((c if i == j else 0.0) + s * Kx[i, j]) + (v * k[i]) * k[j]
    out = np.empty((3, 4))
    u = T[:, 3] - ref[:, 3]
    for i in range(3):
        for j in range(3):
            out[i, j] = (R[i, 0] * T[0, j] + R[i, 1] * T[1, j]) + R[i, 2] * T[2, j]
        out[i, 3] = (((R[i, 0] * u[0] + R[i, 1] * u[1]) + R[i, 2] * u[2]) + ref[i, 3]) + x[3 + i]
    return out


# ---- the whole schedule ---------------------------------------------------------------------------------------------
def model_maps(vol, origin, voxel_size, trunc, c2w, lv, dtype=np.float32):
    """um_tsdf_raycast at one level from the reference rows: (depth [n, h, w], normal [n, h, w, 3])"""
    fx, fy, cx, cy, h, w = lv
    K = [[fx, 0, cx], [0, fy, cy], [0, 0, 1]]
    d, _, nrm = RR.raycast(vol, origin, voxel_size, trunc, c2w, K, h, w, dtype(0), np.inf, dtype)
    return d, nrm


def track(vol, origin, voxel_size, trunc, depths, K, poses, n_levels=3, iterations=(4, 5, 10), max_distance=0.1,
          max_angle=20.0, min_inlier_fraction=0.3, dtype=np.float32, correction=None, min_pivot=MIN_PIVOT, history=None):
    """`TSDFVolume.track` on the volume planes (a dict of tsdf / weight [Z, Y, X] and color [3, Z, Y, X]): returns
    {'pose' float32 [n, 4, 4], 'tracked' bool [n], 'inliers' int64 [n], 'rmse' float32 [n], 'T' fp64 [n, 3, 4],
    'valid' [n], 'sums' [n, 30] of the acceptance pass}.  With a list `history`, each solve's (level, sums) is appended."""
    lvs = levels(K, np.asarray(depths).shape[1], np.asarray(depths).shape[2], n_levels)
    pyr = [np.asarray(depths, dtype)]
    for _ in lvs[1:]:
        pyr.append(downsample(pyr[-1], np.float32(trunc), dtype))
    nrm = [normals(d, *lv[:4], dtype=dtype) for d, lv in zip(pyr, lvs)]
    st, c2w, w2c = init(np.asarray(poses, np.float64), correction)
    models = [model_maps(vol, origin, voxel_size, trunc, c2w, lv, dtype) for lv in lvs]
    cos_max = np.float32(math.cos(math.radians(max_angle)))

    def reduce(level):
        fx, fy, cx, cy, _, _ = lvs[level]
        return sums(block_partials(pixel_terms(pyr[level], nrm[level], models[level][0], models[level][1], st["T"], c2w,
                                               w2c, fx, fy, cx, cy, np.float32(max_distance), cos_max, dtype)))

    its = tuple(iterations)[::-1]
    for level in reversed(range(n_levels)):
        for _ in range(its[level]):
            S = reduce(level)
            if history is not None:
                history.append((level, S))
            for f in range(len(S)):
                x = solve_step(S[f], min_pivot=min_pivot)
                if x is None:
                    st["degenerate"][f] += level == 0
                else:
                    st["T"][f] = apply_step(st["T"][f], st["ref"][f], x)
    S = reduce(0)
    tracked = (st["degenerate"] == 0) & (S[:, 28] >= min_inlier_fraction * S[:, 29])
    T = np.where(tracked[:, None, None], st["T"], st["ref"])
    pose = np.zeros((len(T), 4, 4), np.float32)
    pose[:, :3] = T.astype(np.float32)
    pose[:, 3, 3] = 1
    with np.errstate(invalid="ignore", divide="ignore"):
        rmse = np.where(S[:, 28] > 0, np.sqrt(S[:, 27] / np.maximum(S[:, 28], 1)), 0).astype(np.float32)
    return {"pose": pose, "tracked": tracked, "inliers": S[:, 28].astype(np.int64), "rmse": rmse, "T": T,
            "valid": S[:, 29], "sums": S}


def correction_after(T, P):
    """C = T P^-1 (fp64 rows [3, 4]) with P^-1 = (R_P^T, -R_P^T t_P), as um_icp_accept computes it"""
    P = np.asarray(P, np.float64)[:3]
    Pi = np.empty((3, 4))
    Pi[:, :3] = P[:, :3].T
    for i in range(3):
        Pi[i, 3] = -((P[0, i] * P[0, 3] + P[1, i] * P[1, 3]) + P[2, i] * P[2, 3])
    C = np.eye(4)
    C[:3] = _times(np.asarray(T, np.float64), Pi)
    return C


# ---- analytic scenes of several primitives ----------------------------------------------------------------------------
def render_union(scenes, K, P, h, w, du=0.0, dv=0.0):
    """Exact float64 z-depth [h, w] of the union of `refops_fusion.render` scenes: the nearest positive hit"""
    ds = np.stack([RF.render(s, K, P, h, w, du, dv) for s in scenes])
    ds = np.where(ds > 0, ds, np.inf)
    d = ds.min(0)
    return np.where(np.isfinite(d), d, 0.0)


CORNER = [("plane", [0.0, 1.0, 0.0], 0.55),             # the floor (y points down)
          ("plane", [1.0, 0.0, 0.0], 0.75),             # a side wall
          ("plane", [0.0, 0.0, 1.0], 2.4),              # the back wall
          ("sphere", [-0.25, 0.25, 1.9], 0.3)]


def corner_clip(n=5, h=48, w=64, seed=3):
    """The corner of a floor, two orthogonal walls and a sphere, seen by cameras near the origin looking into the corner
    (rotated by up to about 6 degrees about each axis): every frame sees all four primitives, which constrain all six
    degrees of freedom.  Returns (scenes, K, poses [n, 4, 4] float64)."""
    g = np.random.default_rng(seed)
    K = [[0.8 * w, 0, w / 2], [0, 0.8 * w, h / 2], [0, 0, 1]]
    look = RF.rot("y", 0.2) @ RF.rot("x", -0.15)
    poses = []
    for _ in range(n):
        R = look @ RF.rot("z", g.uniform(-0.1, 0.1)) @ RF.rot("y", g.uniform(-0.1, 0.1)) @ RF.rot("x", g.uniform(-0.1, 0.1))
        poses.append(RF.pose(R, g.uniform(-0.05, 0.05, 3)))
    return CORNER, K, np.stack(poses)


def perturb(P, g, max_translation=0.02, max_degrees=2.0):
    """P moved by a random translation of at most max_translation metres and rotated about its centre by at most
    max_degrees"""
    axis = g.normal(size=3)
    axis /= np.linalg.norm(axis)
    ang = math.radians(g.uniform(0.5, 1.0) * max_degrees)
    Kx = np.array([[0.0, -axis[2], axis[1]], [axis[2], 0.0, -axis[0]], [-axis[1], axis[0], 0.0]])
    R = np.eye(3) + math.sin(ang) * Kx + (1 - math.cos(ang)) * Kx @ Kx
    d = g.normal(size=3)
    d *= g.uniform(0.5, 1.0) * max_translation / np.linalg.norm(d)
    Q = np.array(P, np.float64)
    Q[:3, :3] = R @ Q[:3, :3]
    Q[:3, 3] = Q[:3, 3] + d
    return Q


def pose_error(P, Q):
    """(translation error in metres, rotation error in degrees) between camera-to-world poses P and Q"""
    P, Q = np.asarray(P, np.float64), np.asarray(Q, np.float64)
    dR = P[:3, :3].T @ Q[:3, :3]
    c = np.clip((np.trace(dR) - 1) / 2, -1, 1)
    return float(np.linalg.norm(P[:3, 3] - Q[:3, 3])), math.degrees(math.acos(c))
