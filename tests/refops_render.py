"""Executable statement of the TSDF ray cast (`um_tsdf_raycast`, include/unimatch_sm100.h; `TSDFVolume.render`), in numpy,
vectorised over rays with a masked marching loop.

`dtype=np.float64` is the statement the analytic tests compare with.  `dtype=np.float32` evaluates it in the kernel's
order of operations (each fma correctly rounded through `oracle.submission_io.fma32`, every other operation an IEEE
float32 operation), so it is what the kernel computes bit for bit.  The per-voxel gradient of the normals is
`refops_mesh.gradients`, the mesh's.
"""
import numpy as np

import refops_mesh as RM
from oracle.submission_io import fma32


def _fma(a, b, c, dtype):
    return fma32(a, b, c) if dtype == np.float32 else np.asarray(a * b + c, dtype)


def _lerp(f, a, b, dtype):
    return _fma(f, (b - a).astype(dtype), a, dtype)


def _trilinear(v, f, dtype):
    """v [8, m] corner values (corner c = bx + 2 by + 4 bz), f [3, m] fractions: along x, then y, then z"""
    x00, x10 = _lerp(f[0], v[0], v[1], dtype), _lerp(f[0], v[2], v[3], dtype)
    x01, x11 = _lerp(f[0], v[4], v[5], dtype), _lerp(f[0], v[6], v[7], dtype)
    return _lerp(f[2], _lerp(f[1], x00, x10, dtype), _lerp(f[1], x01, x11, dtype), dtype)


def rays(c2w, K, h, w, origin, voxel_size, dims, near=0.0, far=np.inf, dtype=np.float64):
    """(gd [3, R], go [3, R], t_lo [R], t_hi [R], ok [R]) of the n x h x w rays (R = n h w, view-major, then row, column):
    the ray in grid coordinates g(t) = fma(t, gd, go) and its marching range; ok is False where the ray misses the box
    of voxel centres (or a dimension is below 2)."""
    M = np.asarray(c2w, dtype).reshape(-1, 3, 4)
    n = len(M)
    fx, fy, cx, cy = (dtype(v) for v in (K[0][0], K[1][1], K[0][2], K[1][2]))
    vs = dtype(voxel_size)
    ys, xs = np.meshgrid(np.arange(h, dtype=dtype), np.arange(w, dtype=dtype), indexing="ij")
    xc = np.broadcast_to((xs - cx) / fx, (n, h, w)).reshape(-1)
    yc = np.broadcast_to((ys - cy) / fy, (n, h, w)).reshape(-1)
    per_ray = lambda col: np.repeat(col, h * w)                   # noqa: E731  one value per view -> per ray
    t_lo = np.full(n * h * w, dtype(near), dtype)
    t_hi = np.full(n * h * w, dtype(far), dtype)
    ok = np.full(n * h * w, min(dims) >= 2)
    gd, go = np.zeros((3, n * h * w), dtype), np.zeros((3, n * h * w), dtype)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        for a in range(3):
            d = _fma(per_ray(M[:, a, 0]), xc, _fma(per_ray(M[:, a, 1]), yc, per_ray(M[:, a, 2]), dtype), dtype)
            gd[a] = d / vs
            go[a] = ((per_ray(M[:, a, 3]) - dtype(origin[a])) / vs - dtype(0.5)).astype(dtype)
            ok &= np.isfinite(gd[a]) & np.isfinite(go[a])
            top = dtype(dims[a] - 1)
            flat = gd[a] == 0
            ok &= ~flat | ((go[a] >= 0) & (go[a] <= top))
            t0, t1 = (-go[a] / gd[a]).astype(dtype), ((top - go[a]) / gd[a]).astype(dtype)
            t_lo = np.where(flat, t_lo, np.fmax(t_lo, np.fmin(t0, t1)))
            t_hi = np.where(flat, t_hi, np.fmin(t_hi, np.fmax(t0, t1)))
    ok &= (t_lo <= t_hi) & np.isfinite(t_hi)
    return gd, go, t_lo, t_hi, ok


def _cell(gd, go, t, dims, dtype):
    """(linear index of the cell's low corner [m], fractions [3, m], corner indices [8, m]) of the samples at t"""
    X, Y, Z = dims
    idx, f = [], []
    for a in range(3):
        g = _fma(t, gd[a], go[a], dtype)
        i = np.clip(np.floor(g), 0, dims[a] - 2).astype(np.int64)
        idx.append(i)
        f.append((g - i.astype(dtype)).astype(dtype))
    base = (idx[2] * Y + idx[1]) * X + idx[0]
    corners = np.stack([base + (c & 1) + ((c >> 1) & 1) * X + (c >> 2) * X * Y for c in range(8)])
    return base, np.stack(f), corners, idx


def raycast(vol, origin, voxel_size, trunc, c2w, K, h, w, near=0.0, far=np.inf, dtype=np.float64, counts=False):
    """depth [n, h, w], colour uint8 [n, h, w, 3] and normal [n, h, w, 3] of the volume (a dict of tsdf / weight
    [Z, Y, X] and color [3, Z, Y, X]) seen through the camera-to-world rows c2w [n, 3, 4] with intrinsics K at h x w;
    with `counts`, also the number of samples each ray evaluated [n, h, w]."""
    F = np.asarray(vol["tsdf"], dtype).reshape(-1)
    Wt = np.asarray(vol["weight"], dtype).reshape(-1)
    C = np.asarray(vol["color"], dtype).reshape(3, -1)
    Z, Y, X = np.asarray(vol["tsdf"]).shape
    dims = (X, Y, Z)
    n = len(np.asarray(c2w).reshape(-1, 3, 4))
    R = n * h * w
    gd, go, t_lo, t_hi, ok = rays(c2w, K, h, w, origin, voxel_size, dims, near, far, dtype)
    sf, sc = dtype(voxel_size) * dtype(0.5), dtype(trunc) * dtype(0.5)
    n_samples = np.zeros(R, np.int64)

    def sample(t, sel):
        n_samples[sel] += 1
        _, f, corners, _ = _cell(gd[:, sel], go[:, sel], t, dims, dtype)
        known = (Wt[corners] > 0).all(0)
        with np.errstate(invalid="ignore", over="ignore"):
            val = _trilinear(F[corners], f, dtype)
        return known, np.where(known, val, dtype(0)).astype(dtype)

    def step(ta, s, hi):
        tb = np.fmin((ta + s).astype(dtype), hi)
        return np.where(tb > ta, tb, hi)

    sel = np.nonzero(ok)[0]
    ta = t_lo[sel]
    Ak, AF = sample(ta, sel)
    hit_ray, hit_ta, hit_tb, hit_Fa, hit_Fb = [], [], [], [], []
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        while len(sel):
            go_on = ta < t_hi[sel]
            sel, ta, Ak, AF = sel[go_on], ta[go_on], Ak[go_on], AF[go_on]
            if not len(sel):
                break
            hi = t_hi[sel]
            a_fine = Ak & (AF < 1)
            tb = step(ta, np.where(a_fine, sf, sc).astype(dtype), hi)
            Bk, BF = sample(tb, sel)
            back = ~a_fine & Bk & (BF < 1)                        # a coarse step onto a fine sample is taken back
            if back.any():
                tb[back] = step(ta[back], sf, hi[back])
                Bk[back], BF[back] = sample(tb[back], sel[back])
            cross = Ak & Bk & ((AF < 0) != (BF < 0))
            hit = cross & (BF < 0)
            hit_ray.append(sel[hit]), hit_ta.append(ta[hit]), hit_tb.append(tb[hit])
            hit_Fa.append(AF[hit]), hit_Fb.append(BF[hit])
            keep = ~cross
            sel, ta, Ak, AF = sel[keep], tb[keep], Bk[keep], BF[keep]

    depth = np.zeros(R, dtype)
    color = np.zeros((R, 3), np.uint8)
    normal = np.zeros((R, 3), dtype)
    ray = np.concatenate(hit_ray) if hit_ray else np.zeros(0, np.int64)
    if len(ray):
        ta, tb, Fa, Fb = (np.concatenate(v) for v in (hit_ta, hit_tb, hit_Fa, hit_Fb))
        G = RM.gradients(vol, dtype).reshape(-1, 3)
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            s = (Fa / (Fa - Fb)).astype(dtype)
            depth[ray] = _fma(s, (tb - ta).astype(dtype), ta, dtype)
            shade = []
            for t in (ta, tb):
                _, f, corners, _ = _cell(gd[:, ray], go[:, ray], t, dims, dtype)
                shade.append(([_trilinear(C[ch][corners], f, dtype) for ch in range(3)],
                              [_trilinear(G[:, a][corners], f, dtype) for a in range(3)]))
            (ca, ga), (cb, gb) = shade
            for ch in range(3):
                color[ray, ch] = np.clip(np.rint(_lerp(s, ca[ch], cb[ch], dtype)), 0, 255).astype(np.uint8)
            nv = [_lerp(s, ga[a], gb[a], dtype) for a in range(3)]
            l2 = _fma(nv[2], nv[2], _fma(nv[1], nv[1], (nv[0] * nv[0]).astype(dtype), dtype), dtype)
            length = np.sqrt(l2).astype(dtype)
            for a in range(3):
                normal[ray, a] = np.where(length == 0, dtype(0), nv[a] / length)
    out = (depth.reshape(n, h, w), color.reshape(n, h, w, 3), normal.reshape(n, h, w, 3))
    return out + (n_samples.reshape(n, h, w),) if counts else out
