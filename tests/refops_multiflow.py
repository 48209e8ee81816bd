"""Executable statement of the multi-flow dense point tracks (`um_multi_flow_tracks` and `um_fb_consistency_error`,
include/unimatch_sm100.h; `multi_flow_tracks` and `MultiFlowTrackRunner` in unimatch_b200/inference.py), in numpy (test
infrastructure, like tests/refops_tracks.py), and an analytic occluder clip.

Sources of frame t >= 1: `multi_flow_sources(t, gaps, anchor)`, the package's one definition of the schedule.  Per pair
(s, t): F its forward flow, O = fwd_occ of the forward-backward check and E = |F + warp(B, F)|, the residual that check
compares with alpha (|F| + |B|) + beta.  Frame 0: x = p, sigma2 = 0, v = 1.  From source s, with refops_tracks.bilinear:
    x = x_s + bilinear(F, x_s),  sigma2 = sigma2_s + bilinear(E, x_s)^2,
    valid = v_s and bilinear(O, x_s) < 0.5 and x inside [0, W-1] x [0, H-1]
(x and valid are exactly `refops_tracks.chain_tracks`'s step).  Frame t takes the valid candidate of smallest sigma2, the
first in source order on ties, visible; if none is valid, the smallest sigma2 of all present candidates, invisible.

`dtype=np.float64` is the statement the tests compare with.  `dtype=np.float32` evaluates it in the kernels' order of
operations (the fma of the residual included, through `oracle.submission_io.fma32`), so it is what they compute bit for bit.
"""
import numpy as np

import refops_tracks as RT
from oracle.submission_io import fma32
from unimatch_b200.inference import multi_flow_sources


def _fma(a, b, c, dtype):
    return fma32(a, b, c) if dtype == np.float32 else a * b + c


def _warp(img, px, py, dtype):
    """fb_consistency_kernel's sample_flow: img [B, 2, H, W] at pixel positions px / py [B, H, W] -> [B, 2, H, W]:
    bilinear_sample's normalise / un-normalise (align_corners=True), the ATen weights and the four taps as fmas, zero
    padding"""
    b, _, h, w = img.shape
    sx, sy = dtype(w - 1), dtype(h - 1)
    two, one, half = dtype(2), dtype(1), dtype(0.5)
    with np.errstate(invalid="ignore", over="ignore"):
        ix = ((two * px / sx - one) + one) * half * sx
        iy = ((two * py / sy - one) + one) * half * sy
        fx, fy = np.floor(ix), np.floor(iy)
        xe, ye = fx + one, fy + one
        wts = ((xe - ix) * (ye - iy), (ix - fx) * (ye - iy), (xe - ix) * (iy - fy), (ix - fx) * (iy - fy))
    x0 = np.clip(np.nan_to_num(fx, nan=-2.0), -2, w + 1).astype(np.int64)
    y0 = np.clip(np.nan_to_num(fy, nan=-2.0), -2, h + 1).astype(np.int64)
    bi = np.arange(b)[:, None, None]
    acc = np.zeros((2, b, h, w), dtype)
    for wt, (dy, dx) in zip(wts, ((0, 0), (0, 1), (1, 0), (1, 1))):
        yy, xx = y0 + dy, x0 + dx
        ok = (yy >= 0) & (yy < h) & (xx >= 0) & (xx < w)
        for c in range(2):
            v = img[bi, c, np.clip(yy, 0, h - 1), np.clip(xx, 0, w - 1)]
            acc[c] = np.where(ok, _fma(wt, v, acc[c], dtype), acc[c])
    return acc


def fb_residual(fwd, bwd, alpha=0.01, beta=0.5, dtype=np.float64):
    """fwd / bwd planar [B, 2, H, W] -> (fwd_occ [B, H, W] in {0, 1}, fwd_err [B, H, W]), the forward half of
    `forward_backward_consistency_check` with the residual it thresholds"""
    fwd, bwd = np.asarray(fwd, dtype), np.asarray(bwd, dtype)
    b, _, h, w = fwd.shape
    ys, xs = np.meshgrid(np.arange(h, dtype=dtype), np.arange(w, dtype=dtype), indexing="ij")
    fu, fv, bu, bv = fwd[:, 0], fwd[:, 1], bwd[:, 0], bwd[:, 1]
    wb = _warp(bwd, xs + fu, ys + fv, dtype)
    with np.errstate(invalid="ignore", over="ignore"):
        dx, dy = fu + wb[0], fv + wb[1]
        err = np.sqrt(_fma(dx, dx, dy * dy, dtype))
        mag = np.sqrt(_fma(fu, fu, fv * fv, dtype)) + np.sqrt(_fma(bu, bu, bv * bv, dtype))
        thr = _fma(dtype(alpha), mag, dtype(beta), dtype)
        return (err > thr).astype(dtype), err.astype(dtype)


def multi_flow_tracks(flows, occ, err, gaps, anchor, dtype=np.float64, states=None):
    """flows [T-1, K, 2, H, W], occ / err [T-1, K, H, W] (entry (t-1, k): pair (source k of t, t); absent entries are not
    read).  Returns {'tracks' [T-1,H,W,2], 'visible' [T-1,H,W] bool, 'uncertainty' [T-1,H,W]} for frames 1 .. T-1 and
    'candidates': per frame, the list of (k, x, sigma2, valid) of its present candidates.  `states`: {frame: (pos, sigma2,
    vis)} to take a source frame's state from instead of this evaluation's own (one step from given states)."""
    flows = np.asarray(flows, dtype)
    n, k, _, h, w = flows.shape
    start, vis0 = RT.track_start(h, w, dtype)
    own = {0: (start, np.zeros((h, w), dtype), vis0)}
    tracks = np.empty((n, h, w, 2), dtype)
    visible = np.empty((n, h, w), bool)
    sigma = np.empty((n, h, w), dtype)
    cands = []
    for t in range(1, n + 1):
        found = np.zeros((h, w), bool)
        bx, bs = np.full((h, w, 2), np.nan, dtype), np.full((h, w), np.nan, dtype)
        vx, vs = bx.copy(), bs.copy()
        anyc = np.zeros((h, w), bool)
        here = []
        for j, s in enumerate(multi_flow_sources(t, gaps, anchor)):
            if s < 0:
                continue
            pos, sg, vis = (states or own).get(s, own.get(s))
            pos, sg = np.asarray(pos, dtype), np.asarray(sg, dtype)
            step = RT.chain_tracks(flows[t - 1, j][None], np.asarray(occ[t - 1, j], dtype)[None], state=(pos, vis),
                                   dtype=dtype)
            x, valid = step["tracks"][0], step["visible"][0]
            e = RT.bilinear(np.asarray(err[t - 1, j], dtype)[None], pos[..., 0], pos[..., 1])[0]
            with np.errstate(invalid="ignore", over="ignore"):
                s2 = sg + e * e
                take = valid & (~found | (s2 < vs))
                take_any = ~anyc | (s2 < bs)
            vx[take], vs[take] = x[take], s2[take]
            found |= take
            bx[take_any], bs[take_any] = x[take_any], s2[take_any]
            anyc |= take_any
            here.append((j, x, s2, valid))
        x = np.where(found[..., None], vx, bx)
        s2 = np.where(found, vs, bs)
        tracks[t - 1], visible[t - 1], sigma[t - 1] = x, found, s2
        own[t] = (x, s2, found)
        cands.append(here)
    return {"tracks": tracks, "visible": visible, "uncertainty": sigma, "candidates": cands}


def pair_flows(flows_of_pair, n, gaps, anchor, h, w):
    """[T-1, K, 2, H, W] forward and backward flows of the schedule's pairs from `flows_of_pair(s, t)` -> (fwd, bwd) planar
    [2, H, W] each; absent entries are NaN (never read)"""
    k = len(gaps) + anchor
    fwd = np.full((n, k, 2, h, w), np.nan, np.float32)
    bwd = np.full((n, k, 2, h, w), np.nan, np.float32)
    for t in range(1, n + 1):
        for j, s in enumerate(multi_flow_sources(t, gaps, anchor)):
            if s >= 0:
                fwd[t - 1, j], bwd[t - 1, j] = flows_of_pair(s, t)
    return fwd, bwd


class OccluderClip:
    """A background that translates by `bg` whole pixels per frame and an opaque `size` x `size` square at `corner` in frame
    0 that crosses it at `sq` whole pixels per frame.  The exact flows of every pair (s, t) are known: a pixel of frame s on
    the square moves with the square, every other pixel with the background (forward); a pixel of frame t on the square
    came with the square, every other pixel with the background (backward)."""

    def __init__(self, frames=24, h=40, w=96, bg=(1, 0), sq=(4, 0), size=10, corner=(2, 15)):
        self.frames, self.h, self.w, self.bg, self.sq, self.size, self.corner = frames, h, w, bg, sq, size, corner
        self.ys, self.xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")

    def square(self, f, x=None, y=None):
        """bool: (x, y) (default every pixel) lies on the square in frame f"""
        x = self.xs if x is None else x
        y = self.ys if y is None else y
        x0, y0 = self.corner[0] + self.sq[0] * f, self.corner[1] + self.sq[1] * f
        return (x >= x0) & (x < x0 + self.size) & (y >= y0) & (y < y0 + self.size)

    def flows(self, s, t):
        d = t - s
        fwd = np.where(self.square(s)[None], np.array(self.sq)[:, None, None] * d, np.array(self.bg)[:, None, None] * d)
        bwd = np.where(self.square(t)[None], -np.array(self.sq)[:, None, None] * d, -np.array(self.bg)[:, None, None] * d)
        return fwd.astype(np.float32), bwd.astype(np.float32)

    def truth(self):
        """(true positions [T, H, W, 2] of frame 0's background pixels, covered [T, H, W] by the square, inside [T, H, W],
        background [H, W]: the pixels of frame 0 that are not on the square)"""
        t = np.arange(self.frames)[:, None, None]
        x = self.xs[None] + self.bg[0] * t
        y = self.ys[None] + self.bg[1] * t
        covered = np.stack([self.square(f, x[f], y[f]) for f in range(self.frames)])
        inside = (x >= 0) & (x <= self.w - 1) & (y >= 0) & (y <= self.h - 1)
        return np.stack((x, y), -1).astype(np.float64), covered, inside, ~self.square(0)
