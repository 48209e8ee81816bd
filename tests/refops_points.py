"""Executable statement of the query point tracks (`um_track_points_forward` / `um_track_points_backward`,
include/unimatch_sm100.h; `track_points` and `PointTrackRunner` in unimatch_b200/inference.py), in numpy (test
infrastructure, like tests/refops_tracks.py, whose `bilinear` it uses).

A query (t_q, y, x) is at p = (x, y), visible, in frame t_q.  Forward, frame t > t_q uses pair (t-1, t), its forward flow
F [2,H,W] and fwd_occ O [H,W]; backward, frame t < t_q uses pair (t, t+1), its backward flow B (frame t+1 -> t) and bwd_occ
Ob.  Both are `refops_tracks.chain_tracks`'s step:
    p_t = p_prev + bilinear(F, p_prev),  vis_t = vis_prev and bilinear(O, p_prev) < 0.5 and p_t inside [0,W-1] x [0,H-1],
with p_prev the track in frame t-1 (forward) or t+1 (backward).  Masks None: nothing occluded.

`dtype=np.float64` is the statement the tests compare with; `dtype=np.float32` is what the kernels compute bit for bit.
"""
import numpy as np

import refops_tracks as RT


def _step(p, v, flow, occ, dtype):
    """one step of every track: p [N,2], v [N] bool, flow [2,H,W], occ [H,W] or None -> (p, v, sampled mask)"""
    _, h, w = flow.shape
    x, y = p[:, 0], p[:, 1]
    d = RT.bilinear(np.asarray(flow, dtype), x, y)
    o = np.zeros_like(x) if occ is None else RT.bilinear(np.asarray(occ, dtype)[None], x, y)[0]
    p = np.stack((x + d[0], y + d[1]), axis=-1)
    with np.errstate(invalid="ignore"):
        v = v & (o < 0.5) & (p[:, 0] >= 0) & (p[:, 0] <= w - 1) & (p[:, 1] >= 0) & (p[:, 1] <= h - 1)
    return p, v, o


def track_points(flows, flows_bwd, fwd_occ, bwd_occ, queries, dtype=np.float64):
    """flows / flows_bwd [T-1,2,H,W], fwd_occ / bwd_occ [T-1,H,W] or None, queries [N,3] (t_q, y, x), t_q integer in [0,T).
    Returns {'tracks' [N,T,2] (x, y), 'visible' [N,T] bool, 'o' [N,T] the mask each frame's test sampled (0 at t_q)}."""
    flows = np.asarray(flows, dtype)
    n = flows.shape[0]
    q = np.asarray(queries, dtype)
    tq = q[:, 0].astype(np.int64)
    start = np.stack((q[:, 2], q[:, 1]), axis=-1)
    nq, nt = q.shape[0], n + 1
    tracks = np.empty((nq, nt, 2), dtype)
    visible = np.empty((nq, nt), bool)
    osamp = np.zeros((nq, nt), dtype)
    tracks[np.arange(nq), tq] = start
    visible[np.arange(nq), tq] = True
    for direction in ("forward", "backward"):
        p, v = start.copy(), np.ones(nq, bool)
        pairs = range(n) if direction == "forward" else range(n - 1, -1, -1)
        for j in pairs:
            if direction == "forward":
                active, frame = tq <= j, j + 1
                flow, occ = flows[j], None if fwd_occ is None else fwd_occ[j]
            else:
                active, frame = tq > j, j
                flow, occ = flows_bwd[j], None if bwd_occ is None else bwd_occ[j]
            np2, nv, o = _step(p, v, flow, occ, dtype)
            p, v = np.where(active[:, None], np2, p), np.where(active, nv, v)
            tracks[active, frame], visible[active, frame], osamp[active, frame] = p[active], v[active], o[active]
    return {"tracks": tracks, "visible": visible, "o": osamp}


def visibility_mismatches(got_visible, ref, queries, h, w, eps_p, eps_o):
    """(queries whose visibility differs from the statement somewhere, of those the ones NOT explained by a test within
    rounding of a threshold at the first frame, walking away from t_q in each direction, where they part)"""
    diff = np.asarray(got_visible).astype(bool) != ref["visible"]
    x, y = ref["tracks"][..., 0], ref["tracks"][..., 1]
    edge = np.minimum(np.minimum(np.abs(x), np.abs(x - (w - 1))), np.minimum(np.abs(y), np.abs(y - (h - 1))))
    near = (edge <= eps_p) | (np.abs(ref["o"] - 0.5) <= eps_o)
    tq = np.asarray(queries)[:, 0].astype(np.int64)
    parted = unexplained = 0
    for i in range(diff.shape[0]):
        fwd, bwd = diff[i, tq[i] + 1:], diff[i, :tq[i]][::-1]
        firsts = ([tq[i] + 1 + int(np.argmax(fwd))] if fwd.any() else []) + ([tq[i] - 1 - int(np.argmax(bwd))] if bwd.any()
                                                                              else [])
        if firsts:
            parted += 1
            unexplained += not all(near[i, t] for t in firsts)
    return parted, unexplained


def random_queries(nq, nt, h, w, seed, frames=None):
    """nq seeded queries [nq,3] float32 (t_q, y, x): fractional positions inside the frame, a few exactly on its edges and
    corners, t_q drawn from `frames` (default: every frame)"""
    rng = np.random.default_rng(seed)
    frames = np.arange(nt) if frames is None else np.asarray(frames)
    q = np.empty((nq, 3), np.float32)
    q[:, 0] = rng.choice(frames, nq)
    q[:, 1] = rng.random(nq) * (h - 1)
    q[:, 2] = rng.random(nq) * (w - 1)
    edges = [(0, 0), (0, w - 1), (h - 1, 0), (h - 1, w - 1), (0, (w - 1) / 2), ((h - 1) / 2, w - 1), (h - 1, 3.5),
             (2.25, 0)]
    for i, (y, x) in enumerate(edges[:nq]):
        q[i, 1], q[i, 2] = y, x
    return q
