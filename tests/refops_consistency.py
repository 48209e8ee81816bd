"""Executable statement of the multi-view geometric consistency of depth maps (`um_depth_consistency`) and of the export of
valid depths as points (`um_depth_points_count` / `um_depth_points`), include/unimatch_sm100.h; `filter_depths`,
`depth_points` and `DepthFusionRunner(consistency_views=k)` in unimatch_b200, in numpy.

`dtype=np.float32` evaluates them in the kernels' order of operations (each fma correctly rounded through
`oracle.submission_io.fma32`, every other operation an IEEE float32 operation, the square root correctly rounded), so it
is what the kernels compute bit for bit; `dtype=np.float64` is the same statement in float64.  Also the corrupted corner
clip the CPU tests filter.
"""
import numpy as np

import refops_fusion as RF
import refops_icp as RI
from oracle.submission_io import fma32


def _fma(a, b, c, dtype):
    return fma32(a, b, c) if dtype == np.float32 else np.asarray(a * b + c, dtype)


def _valid(d):
    return np.isfinite(d) & (d > 0)


def apply_rows(M, p, dtype):
    """Rows M [3, 4] applied to points p (x, y, z arrays): fma(M_r2, z, fma(M_r1, y, fma(M_r0, x, M_r3))) per row"""
    x, y, z = p
    return [_fma(M[r, 2], z, _fma(M[r, 1], y, _fma(M[r, 0], x, M[r, 3], dtype), dtype), dtype).astype(dtype)
            for r in range(3)]


def back_project(u, v, d, fx, fy, cx, cy, dtype):
    """((u - cx) / fx * d, (v - cy) / fy * d, d)"""
    xr = ((np.asarray(u, dtype) - cx).astype(dtype) / fx).astype(dtype)
    yr = ((np.asarray(v, dtype) - cy).astype(dtype) / fy).astype(dtype)
    return [(xr * d).astype(dtype), (yr * d).astype(dtype), np.asarray(d, dtype)]


def _camera(K, dtype):
    return tuple(dtype(v) for v in (K[0][0], K[1][1], K[0][2], K[1][2]))


def source_check(depths, c2w, w2c, K, r, s, max_pixel=1.0, max_relative=0.01, dtype=np.float32, details=False):
    """(consistent [h, w] bool, taps_ok [h, w] bool) of reference map r against source s: taps_ok marks the pixels with a
    valid depth whose source point is in front, inside [0, w-1] x [0, h-1] and has four valid taps.  With `details`, the
    reprojection error and the relative depth difference [h, w] follow (meaningful where taps_ok)."""
    D = np.asarray(depths, dtype)
    n, h, w = D.shape
    c2w, w2c = np.asarray(c2w, dtype), np.asarray(w2c, dtype)
    fx, fy, cx, cy = _camera(K, dtype)
    ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    xf, yf = xs.astype(dtype), ys.astype(dtype)
    d = D[r]
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        ok = _valid(d)
        c = apply_rows(w2c[s], apply_rows(c2w[r], back_project(xf, yf, d, fx, fy, cx, cy, dtype), dtype), dtype)
        ok &= c[2] > 0
        u = _fma(fx, (c[0] / c[2]).astype(dtype), cx, dtype).astype(dtype)
        v = _fma(fy, (c[1] / c[2]).astype(dtype), cy, dtype).astype(dtype)
        ok &= (u >= 0) & (u <= w - 1) & (v >= 0) & (v <= h - 1)
        u, v = np.where(ok, u, dtype(0)), np.where(ok, v, dtype(0))
        fx0, fy0 = np.floor(u), np.floor(v)
        x0, y0 = fx0.astype(np.int64), fy0.astype(np.int64)
        x1, y1 = np.minimum(x0 + 1, w - 1), np.minimum(y0 + 1, h - 1)
        S = D[s]
        d00, d01, d10, d11 = S[y0, x0], S[y0, x1], S[y1, x0], S[y1, x1]
        ok &= _valid(d00) & _valid(d01) & _valid(d10) & _valid(d11)
        ax, ay = (u - fx0).astype(dtype), (v - fy0).astype(dtype)
        top = _fma(ax, (d01 - d00).astype(dtype), d00, dtype).astype(dtype)
        bot = _fma(ax, (d11 - d10).astype(dtype), d10, dtype).astype(dtype)
        ds = _fma(ay, (bot - top).astype(dtype), top, dtype).astype(dtype)
        b = apply_rows(w2c[r], apply_rows(c2w[s], back_project(u, v, ds, fx, fy, cx, cy, dtype), dtype), dtype)
        taps_ok = ok.copy()
        ok &= b[2] > 0
        u2 = _fma(fx, (b[0] / b[2]).astype(dtype), cx, dtype).astype(dtype)
        v2 = _fma(fy, (b[1] / b[2]).astype(dtype), cy, dtype).astype(dtype)
        dx, dy = (u2 - xf).astype(dtype), (v2 - yf).astype(dtype)
        err = np.sqrt(_fma(dy, dy, (dx * dx).astype(dtype), dtype).astype(dtype)).astype(dtype)
        rel = (np.abs((b[2] - d).astype(dtype)) / d).astype(dtype)
        ok &= (err < dtype(max_pixel)) & (rel < dtype(max_relative))
    return (ok, taps_ok, err, rel) if details else (ok, taps_ok)


def consistency(depths, c2w, w2c, K, refs, sources, max_pixel=1.0, max_relative=0.01, min_views=2, dtype=np.float32):
    """(views uint8 [R, h, w], filtered depth [R, h, w]) of um_depth_consistency; entries outside [0, n) are no source"""
    D = np.asarray(depths, dtype)
    n, h, w = D.shape
    sources = np.asarray(sources)
    views = np.zeros((len(refs), h, w), np.uint8)
    out = np.zeros((len(refs), h, w), dtype)
    for i, r in enumerate(refs):
        if not 0 <= r < n:
            continue
        count = np.zeros((h, w), np.int64)
        for s in sources[i]:
            if 0 <= s < n:
                count += source_check(D, c2w, w2c, K, r, s, max_pixel, max_relative, dtype)[0]
        views[i] = count
        out[i] = np.where(count >= min_views, D[r], dtype(0))
    return views, out


def points(depths, frames, c2w, K, dtype=np.float32):
    """(points [P, 3], colors uint8 [P, 3]) of the valid depths, frame-major, then row-major pixel"""
    D = np.asarray(depths, dtype)
    n, h, w = D.shape
    fx, fy, cx, cy = _camera(K, dtype)
    ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    pts, cols = [], []
    for t in range(n):
        ok = _valid(D[t])
        p = apply_rows(np.asarray(c2w[t], dtype), back_project(xs[ok].astype(dtype), ys[ok].astype(dtype), D[t][ok], fx, fy,
                                                               cx, cy, dtype), dtype)
        pts.append(np.stack(p, -1))
        cols.append(np.asarray(frames)[t][ok])
    return np.concatenate(pts).reshape(-1, 3), np.concatenate(cols).reshape(-1, 3)


def sequence_sources(n, before, after):
    """The table `fusion.sequence_sources` builds, written out row by row"""
    rows = []
    for t in range(n):
        row = [t - k if t - k >= 0 else -1 for k in range(1, before + 1)]
        row += [t + k if t + k < n else -1 for k in range(1, after + 1)]
        rows.append(row)
    return np.array(rows, np.int32).reshape(n, before + after)


def corrupt(depths, seed=0, outlier_fraction=0.02, patch=8, scale=1.3):
    """The depths with random outliers (a fraction of the valid pixels set to depths uniform in [0.5, 4] m) and one
    patch x patch square per frame scaled by `scale`: (corrupted float32 [n, h, w], corrupted mask bool [n, h, w])"""
    g = np.random.default_rng(seed)
    d = np.array(depths, np.float32)
    n, h, w = d.shape
    mask = np.zeros(d.shape, bool)
    for t in range(n):
        y, x = g.integers(0, h - patch), g.integers(0, w - patch)
        d[t, y:y + patch, x:x + patch] *= np.float32(scale)
        mask[t, y:y + patch, x:x + patch] = d[t, y:y + patch, x:x + patch] > 0
    out = (g.random(d.shape) < outlier_fraction) & (d > 0)
    d[out] = g.uniform(0.5, 4.0, out.sum()).astype(np.float32)
    return d, mask | out


def clip_depths(name, n=5, h=48, w=64):
    """(depths float32 [n, h, w] exact, K, poses float32 [n, 4, 4], scenes) of the sphere, tilted-plane or corner clip"""
    if name == "corner":
        scenes, K, P = RI.corner_clip(n, h, w)
        D = np.stack([RI.render_union(scenes, K, p, h, w) for p in P])
    else:
        scene, K, P = (RF.sphere_clip if name == "sphere" else RF.tilted_plane_clip)(n, h, w)
        scenes = [scene]
        D = np.stack([RF.render(scene, K, p, h, w) for p in P])
    return D.astype(np.float32), np.asarray(K, np.float32), P.astype(np.float32), scenes
