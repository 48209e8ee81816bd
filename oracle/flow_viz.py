"""Restatement of the reference's flow visualisation, `flow_to_image` (utils/flow_viz.py:240-275, with
`make_color_wheel` :145-192 and `compute_color` :195-236) -- the colouring the video driver applies to every predicted flow
(evaluate_flow.py:767-768) -- written so that the precision of every step is explicit.

numpy evaluates the reference on a float32 [H,W,2] flow as follows, and so does this module:
  * unknown-flow markers, |u| or |v| > 1e7 (UNKNOWN_FLOW_THRESH, :140, :254-256), are zeroed before the statistics;
  * rad = sqrt(u**2 + v**2) and its maximum are FLOAT32 (:264-265);
  * `maxrad + np.finfo(float).eps` is a float64 scalar, so the normalised u, v (:267-268) and everything after them --
    rad, arctan2, the wheel interpolation, floor(255 * col) (:211-234) -- are FLOAT64;
  * unknown pixels are painted black (:272-273).
Because maxrad is rounded to float32, the pixel of largest flow often normalises to a radius slightly above 1 and takes the
x0.75 "out of range" branch (:233); a float32 statement gets those pixels visibly wrong.
"""
import numpy as np

UNKNOWN_FLOW_THRESH = 1e7
NCOLS = 55


def color_wheel():
    """Middlebury colour wheel [55, 3] (make_color_wheel, flow_viz.py:145-192): RY 15, YG 6, GC 4, CB 11, BM 13, MR 6."""
    segs = []
    ramp = lambda n: np.floor(255 * np.arange(n) / n)
    full = lambda n: np.full(n, 255.0)
    zero = lambda n: np.zeros(n)
    segs.append(np.stack([full(15), ramp(15), zero(15)], 1))              # red -> yellow
    segs.append(np.stack([255 - ramp(6), full(6), zero(6)], 1))          # yellow -> green
    segs.append(np.stack([zero(4), full(4), ramp(4)], 1))                # green -> cyan
    segs.append(np.stack([zero(11), 255 - ramp(11), full(11)], 1))       # cyan -> blue
    segs.append(np.stack([ramp(13), zero(13), full(13)], 1))             # blue -> magenta
    segs.append(np.stack([full(6), zero(6), 255 - ramp(6)], 1))          # magenta -> red
    return np.concatenate(segs, 0)


def flow_to_image(flow):
    """float32 flow [H, W, 2] -> uint8 RGB [H, W, 3] (flow_viz.py:240-275)."""
    flow = np.asarray(flow, dtype=np.float32)
    u, v = flow[..., 0].copy(), flow[..., 1].copy()
    unknown = (np.abs(u) > UNKNOWN_FLOW_THRESH) | (np.abs(v) > UNKNOWN_FLOW_THRESH)
    u[unknown] = 0
    v[unknown] = 0
    rad32 = np.sqrt(u * u + v * v)                                        # float32
    maxrad = max(np.float32(-1), rad32.max())                             # float32 scalar
    den = np.float64(maxrad) + np.finfo(np.float64).eps                   # float64 from here on
    u64, v64 = u.astype(np.float64) / den, v.astype(np.float64) / den
    rad = np.sqrt(u64 * u64 + v64 * v64)
    a = np.arctan2(-v64, -u64) / np.pi
    fk = (a + 1) / 2 * (NCOLS - 1) + 1
    k0 = np.floor(fk).astype(np.int64)
    k1 = k0 + 1
    k1[k1 == NCOLS + 1] = 1
    f = fk - k0
    wheel = color_wheel()
    img = np.zeros(u.shape + (3,), np.uint8)
    inside = rad <= 1
    for ch in range(3):
        col0, col1 = wheel[k0 - 1, ch] / 255, wheel[k1 - 1, ch] / 255
        col = (1 - f) * col0 + f * col1
        col = np.where(inside, 1 - rad * (1 - col), col * 0.75)
        img[..., ch] = np.floor(255 * col)
    img[unknown] = 0
    return img


def flow_to_image_batch(flow):
    """Planar float32 flows [N, 2, H, W] (numpy or torch) -> uint8 [N, H, W, 3]."""
    flow = np.asarray(flow, dtype=np.float32)
    return np.stack([flow_to_image(np.ascontiguousarray(f.transpose(1, 2, 0))) for f in flow], 0)
