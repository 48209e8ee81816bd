"""Executable statement of the dense point tracks (`um_chain_tracks`, include/unimatch_sm100.h; `chain_tracks` and
`VideoTrackRunner` in unimatch_b200/inference.py), in numpy (test infrastructure, like tests/refops.py).

Tracks start at every pixel of the first frame: p_0(y, x) = (x, y), vis_0 = 1.  Step t uses pair (t-1, t), its forward
flow F [2, H, W] and forward occlusion mask O [H, W] (None: nothing occluded):
    d = bilinear(F, p_{t-1}),  o = bilinear(O, p_{t-1}),  p_t = p_{t-1} + d,
    vis_t = vis_{t-1} and o < 0.5 and 0 <= p_t.x <= W-1 and 0 <= p_t.y <= H-1,
with bilinear the reference's `bilinear_sample` (geometry.py:41-62) in pixel coordinates: align_corners=True, zero padding,
i.e. `flow_warp(F, p - grid)` (geometry.py:65-72) read at the track.  An invisible track stays invisible and is still moved.

`dtype=np.float64` is the statement the tests compare with.  `dtype=np.float32` evaluates the same expression in the order
of operations the header fixes, each numpy float32 operation correctly rounded, so it is what the kernel computes bit for bit.
"""
import numpy as np


def track_start(h, w, dtype=np.float64):
    """(pos [H,W,2] = (x, y) at every pixel, vis [H,W] bool all True)"""
    ys, xs = np.meshgrid(np.arange(h, dtype=dtype), np.arange(w, dtype=dtype), indexing="ij")
    return np.stack((xs, ys), axis=-1), np.ones((h, w), dtype=bool)


def bilinear(img, x, y):
    """img [C, H, W], x / y [H, W] pixel coordinates of img's dtype -> [C, H, W]:
    gy (gx v00 + fx v01) + fy (gx v10 + fx v11) with x0 = floor(x), fx = x - x0, gx = 1 - fx (likewise y) and 0 for a corner
    outside the image.  A track with x <= -1, x >= W, y <= -1, y >= H or a NaN coordinate samples 0."""
    c, h, w = img.shape
    dt = img.dtype
    near = (x > -1) & (x < w) & (y > -1) & (y < h)
    x = np.where(near, x, 0).astype(dt)
    y = np.where(near, y, 0).astype(dt)
    x0, y0 = np.floor(x), np.floor(y)
    fx, fy = x - x0, y - y0
    gx, gy = dt.type(1) - fx, dt.type(1) - fy
    xi, yi = x0.astype(np.int64), y0.astype(np.int64)

    def corner(dy, dx):
        yy, xx = yi + dy, xi + dx
        inside = near & (yy >= 0) & (yy < h) & (xx >= 0) & (xx < w)
        v = img[:, np.clip(yy, 0, h - 1), np.clip(xx, 0, w - 1)]
        return np.where(inside[None], v, dt.type(0))

    top = gx * corner(0, 0) + fx * corner(0, 1)
    bot = gx * corner(1, 0) + fx * corner(1, 1)
    return np.where(near[None], gy * top + fy * bot, dt.type(0))


def chain_tracks(flow, occ=None, state=None, dtype=np.float64):
    """flow [n, 2, H, W], occ [n, H, W] or None, state (pos [H,W,2], vis [H,W]) or None (track_start).
    Returns {'tracks' [n,H,W,2], 'visible' [n,H,W] bool, 'o' [n,H,W] the sampled masks (0 without occ),
    'state' (pos, vis) after the last flow}.  A given state is not modified."""
    flow = np.asarray(flow, dtype=dtype)
    n, _, h, w = flow.shape
    pos, vis = track_start(h, w, dtype) if state is None else state
    p = np.asarray(pos, dtype=dtype).copy()
    v = np.asarray(vis).astype(bool)
    tracks = np.empty((n, h, w, 2), dtype)
    visible = np.empty((n, h, w), bool)
    osamp = np.zeros((n, h, w), dtype)
    for t in range(n):
        x, y = p[..., 0], p[..., 1]
        d = bilinear(flow[t], x, y)
        if occ is not None:
            osamp[t] = bilinear(np.asarray(occ[t], dtype=dtype)[None], x, y)[0]
        p = np.stack((x + d[0], y + d[1]), axis=-1)
        with np.errstate(invalid="ignore"):
            v = v & (osamp[t] < 0.5) & (p[..., 0] >= 0) & (p[..., 0] <= w - 1) & (p[..., 1] >= 0) & (p[..., 1] <= h - 1)
        tracks[t], visible[t] = p, v
    return {"tracks": tracks, "visible": visible, "o": osamp, "state": (p, v)}


def near_threshold(tracks, o, h, w, eps_p, eps_o):
    """[n,H,W] bool: step t's visibility test is within eps_p pixels of a frame edge or within eps_o of o = 0.5, where
    rounding may decide it either way"""
    x, y = tracks[..., 0], tracks[..., 1]
    edge = np.minimum(np.minimum(np.abs(x), np.abs(x - (w - 1))), np.minimum(np.abs(y), np.abs(y - (h - 1))))
    return (edge <= eps_p) | (np.abs(o - 0.5) <= eps_o)


def visibility_mismatches(got_visible, ref, h, w, eps_p, eps_o):
    """(tracks whose visibility differs from the statement at some step, of those the ones NOT explained by a test within
    rounding of a threshold at the first step where they part).  Visibility only ever drops, so the first differing step
    is where the two took different sides of one test."""
    diff = np.asarray(got_visible).astype(bool) != ref["visible"]
    parted = diff.any(axis=0)
    first = np.argmax(diff, axis=0)
    near = near_threshold(ref["tracks"], ref["o"], h, w, eps_p, eps_o)
    explained = np.take_along_axis(near, first[None], axis=0)[0]
    return int(parted.sum()), int((parted & ~explained).sum())


def smooth_flows(n, h, w, amp, seed, drift=(0.0, 0.0)):
    """n seeded smooth random flows [n, 2, H, W] float32: a Gaussian grid of standard deviation `amp` pixels every 24 pixels,
    upsampled bilinearly, plus a constant drift (dx, dy) that carries tracks out of the frame"""
    rng = np.random.default_rng(seed)
    gh, gw = max(2, h // 24), max(2, w // 24)
    coarse = rng.standard_normal((n, 2, gh, gw)) * amp
    yy = np.linspace(0, gh - 1, h)
    xx = np.linspace(0, gw - 1, w)
    y0 = np.minimum(np.floor(yy).astype(int), gh - 2)
    x0 = np.minimum(np.floor(xx).astype(int), gw - 2)
    fy, fx = (yy - y0)[:, None], (xx - x0)[None, :]
    c = coarse
    out = ((1 - fy) * ((1 - fx) * c[..., y0[:, None], x0[None]] + fx * c[..., y0[:, None], x0[None] + 1]) +
           fy * ((1 - fx) * c[..., y0[:, None] + 1, x0[None]] + fx * c[..., y0[:, None] + 1, x0[None] + 1]))
    out[:, 0] += drift[0]
    out[:, 1] += drift[1]
    return np.ascontiguousarray(out, dtype=np.float32)


def lipschitz(flow):
    """Largest difference between horizontally or vertically neighbouring flow values: bilinear(F, .) moves by at most twice
    that per pixel the sampling point moves, inside the frame."""
    f = np.asarray(flow, np.float64)
    return max(np.abs(np.diff(f, axis=-1)).max(initial=0.0), np.abs(np.diff(f, axis=-2)).max(initial=0.0))


def step_rounding(tracks, flow):
    """Bound on what fp32 adds to one step's position: the rounding of p + d (half a unit in the last place of the largest
    |p|) and the sampled d (ten roundings relative to the largest |F|: the weights, four products and three sums)"""
    pmax = float(np.nanmax(np.abs(np.where(np.isfinite(tracks), tracks, 0)), initial=1.0))
    fmax = float(np.abs(np.asarray(flow, np.float64)).max(initial=0.0))
    return 0.5 * float(np.spacing(np.float32(pmax))) + 10 * 2.0 ** -24 * fmax


def chain_tolerance(tracks, flow):
    """Bound on |fp32 - float64| after each of the n steps, for tracks whose path stays inside the frame: each step's
    rounding, grown by the flow's slope (1 + 2 L) per step"""
    eps, grow = step_rounding(tracks, flow), 1.0 + 2.0 * lipschitz(flow)
    n = np.asarray(flow).shape[0]
    return np.array([eps * sum(grow ** k for k in range(t + 1)) for t in range(n)])
