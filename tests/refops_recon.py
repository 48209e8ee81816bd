"""Executable statement of the point-cloud ops (`um_cloud_*`, include/unimatch_sm100.h; `nearest_neighbors`,
`voxel_down_sample` and `reconstruction_metrics` in unimatch_b200), in numpy.

`brute_nearest` is the definition: the fp32 s of every pair in the stated order, the least s, ties to the least index.
`grid_nearest` is the kernel's ring search over the same cell table, with its lower bounds; the CPU tests check that it
equals the brute-force scan bit for bit whatever the cell size, which is what makes the pruning exact.
"""
import math

import numpy as np

from oracle.submission_io import fma32

MAX_CELLS_PER_AXIS = 2 ** 21


def sq_dist32(q, p):
    """s(q, p) in fp32: dx = q.x - p.x, ...; s = fmaf(dz, dz, fmaf(dy, dy, dx * dx)); q [..., 3], p [..., 3] float32"""
    d = (np.asarray(q, np.float32) - np.asarray(p, np.float32)).astype(np.float32)
    with np.errstate(over="ignore"):
        s = (d[..., 0] * d[..., 0]).astype(np.float32)
    s = fma32(d[..., 1], d[..., 1], s).astype(np.float32)
    return fma32(d[..., 2], d[..., 2], s).astype(np.float32)


def brute_nearest(queries, points, chunk=512):
    """(distance float32 [Q], index int64 [Q]): the least fp32 s over all points, ties to the least index"""
    Q, P = np.asarray(queries, np.float32), np.asarray(points, np.float32)
    dist, idx = np.empty(len(Q), np.float32), np.empty(len(Q), np.int64)
    for a in range(0, len(Q), chunk):
        s = sq_dist32(Q[a:a + chunk, None, :], P[None, :, :])
        idx[a:a + chunk] = np.argmin(s, axis=1)               # the first minimum: the least index among ties
        dist[a:a + chunk] = np.sqrt(s[np.arange(len(s)), idx[a:a + chunk]])
    return dist, idx


def cell_coords(points, origin, cell):
    """t = ((double)p - o) / c per axis, float64 [n, 3]"""
    return (np.asarray(points, np.float32).astype(np.float64) - np.asarray(origin, np.float64)) / np.float64(cell)


def cell_keys(points, origin, cell, dims):
    """floor(t) clamped to [0, g - 1] per axis, and the key (k_z g_y + k_y) g_x + k_x"""
    t = cell_coords(points, origin, cell)
    g = np.asarray(dims, np.int64)
    k = np.clip(np.floor(np.clip(t, -1.0, g.astype(np.float64))), 0, g - 1).astype(np.int64)
    return (k[:, 2] * g[1] + k[:, 1]) * g[0] + k[:, 0], k


def axis_gap(t, k, cell):
    """The kernel's per-axis lower bound (metres) on |q - p| for p in cell k, from the query's t (float64)"""
    d = max(k - t, t - (k + 1.0), 0.0)
    return max(d - (2.0 ** -20 + 2.0 ** -45 * abs(t)), 0.0) * cell


def beyond(lb, best):
    return lb * (1.0 - 2.0 ** -20) - 2.0 ** -140 > float(best)


def grid_nearest(queries, points, origin, cell, dims):
    """The kernel's search, query by query (small inputs): rings of cells around the query's clamped cell, cells skipped
    and rings stopped by the stated bounds.  Returns (distance, index) like brute_nearest."""
    Q, P = np.asarray(queries, np.float32), np.asarray(points, np.float32)
    keys, _ = cell_keys(P, origin, cell, dims)
    order = np.argsort(keys, kind="stable")
    skeys = keys[order]
    gx, gy, gz = dims
    ncell = gx * gy * gz
    start = np.searchsorted(skeys, np.arange(ncell), "left")
    end = np.searchsorted(skeys, np.arange(ncell), "right")
    inv = 1.0 / float(cell)
    dist, idx = np.empty(len(Q), np.float32), np.empty(len(Q), np.int64)
    for qi, q in enumerate(Q):
        t = [(float(q[a]) - float(origin[a])) * inv for a in range(3)]
        j = [0 if t[a] < 0 else (dims[a] - 1 if t[a] >= dims[a] - 1 else int(math.floor(t[a]))) for a in range(3)]
        own = [axis_gap(t[a], j[a], cell) ** 2 for a in range(3)]
        best, bi = np.float32(np.inf), 2 ** 31 - 1

        def visit(k):
            nonlocal best, bi
            c = (k[2] * gy + k[1]) * gx + k[0]
            if start[c] == end[c] or beyond(sum(axis_gap(t[a], k[a], cell) ** 2 for a in range(3)), best):
                return
            rows = order[start[c]:end[c]]
            s = sq_dist32(q[None, :], P[rows])
            for si, pi in zip(s, rows):
                if si < best or (si == best and pi < bi):
                    best, bi = si, int(pi)

        r = 0
        while True:
            if r > 0:
                cands = [axis_gap(t[a], j[a] + side * r, cell) ** 2 + own[(a + 1) % 3] + own[(a + 2) % 3]
                         for a in range(3) for side in (-1, 1) if 0 <= j[a] + side * r < dims[a]]
                if not cands or beyond(min(cands), best):
                    break
            for kz in range(max(j[2] - r, 0), min(j[2] + r, gz - 1) + 1):
                for ky in range(max(j[1] - r, 0), min(j[1] + r, gy - 1) + 1):
                    if abs(kz - j[2]) == r or abs(ky - j[1]) == r:
                        xs = range(max(j[0] - r, 0), min(j[0] + r, gx - 1) + 1)
                    else:
                        xs = [x for x in (j[0] - r, j[0] + r) if 0 <= x < gx]
                    for kx in xs:
                        visit((kx, ky, kz))
            r += 1
        dist[qi], idx[qi] = np.sqrt(best), bi
    return dist, idx


def down_sample_grid(points, voxel_size):
    """Open3D's voxel grid of a non-empty set: origin = min_bound - v / 2 (float64) and dims = floor((max_bound - origin)
    / v) + 1 per axis; more than 2^21 cells on an axis is a ValueError"""
    P = np.asarray(points, np.float32).astype(np.float64)
    v = float(voxel_size)
    origin = P.min(0) - v / 2
    dims = np.floor((P.max(0) - origin) / v).astype(np.int64) + 1
    if (dims > MAX_CELLS_PER_AXIS).any():
        raise ValueError("voxel_down_sample: %s cells per axis is more than 2^21" % dims.tolist())
    return origin.tolist(), v, tuple(int(d) for d in dims)


def down_sample(points, voxel_size):
    """Each occupied cell's mean (float64 sums in input order, divided by the count, rounded to float32), ordered by key"""
    P = np.asarray(points, np.float32)
    if len(P) == 0:
        return np.zeros((0, 3), np.float32)
    origin, v, dims = down_sample_grid(P, voxel_size)
    keys, _ = cell_keys(P, origin, v, dims)
    order = np.argsort(keys, kind="stable")
    sk = keys[order]
    heads = np.flatnonzero(np.r_[True, sk[1:] != sk[:-1]])
    counts = np.diff(np.r_[heads, len(sk)])
    acc = np.zeros((len(heads), 3), np.float64)
    sp = P[order].astype(np.float64)
    for j in range(int(counts.max())):                            # sequential per cell, vectorised across cells
        live = counts > j
        acc[live] += sp[heads[live] + j]
    return (acc / counts[:, None]).astype(np.float32)


def metrics(pred, gt, threshold=0.05, down_sample_size=0.02):
    """The stated metrics from the float32 nearest distances: acc, comp, chamfer, prec, recall, fscore, n_pred, n_gt"""
    P, G = np.asarray(pred, np.float32).reshape(-1, 3), np.asarray(gt, np.float32).reshape(-1, 3)
    if down_sample_size is not None:
        P, G = down_sample(P, down_sample_size), down_sample(G, down_sample_size)
    out = {"n_pred": len(P), "n_gt": len(G)}
    if len(P) == 0 or len(G) == 0:
        return dict(out, **{k: math.nan for k in ("acc", "comp", "chamfer", "prec", "recall", "fscore")})
    t = np.float32(threshold)
    d_pred, d_gt = brute_nearest(P, G)[0], brute_nearest(G, P)[0]
    return dict(out, **from_distances(d_pred, d_gt, t))


def from_distances(d_pred, d_gt, t):
    acc, comp = float(np.sum(d_pred, dtype=np.float64)) / len(d_pred), float(np.sum(d_gt, dtype=np.float64)) / len(d_gt)
    prec, recall = float(np.count_nonzero(d_pred < t)) / len(d_pred), float(np.count_nonzero(d_gt < t)) / len(d_gt)
    fscore = 2 * prec * recall / (prec + recall) if prec + recall > 0 else 0.0
    return {"acc": acc, "comp": comp, "chamfer": (acc + comp) / 2, "prec": prec, "recall": recall, "fscore": fscore}
