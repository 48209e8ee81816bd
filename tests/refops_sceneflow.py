"""Executable statement of stereo scene flow's two kernels (include/unimatch_sm100.h: `um_warp_disparity` and
`um_scene_flow_stats`; `warp_disparity`, `infer_scene_flow` and `validate_scene_flow` in unimatch_b200), in numpy (test
infrastructure, like tests/refops_tracks.py).

Warp: for pixel p = (x, y) of frame t with flow (u, v), q = (x + u, y + v); in_frame = 0 <= q.x <= W-1 and 0 <= q.y <= H-1;
disp_1 = bilinear(disp_next, clamp(q)), the clamp being fminf(fmaxf(., 0), size - 1) (a NaN coordinate clamps to 0) and
bilinear `refops_tracks.bilinear` (align_corners=True, gy (gx v00 + fx v01) + fy (gx v10 + fx v11)).  `dtype=np.float64`
is the statement; `dtype=np.float32` evaluates it in the header's order, each numpy float32 operation correctly rounded, so
it is what the kernel computes bit for bit.

Counts: KITTI 2015's devkit outliers, with the fp32 per-pixel expressions of um_eval_stats's UM_EVS_D1 and UM_EVF_OUTLIER
columns, in the column layout of `ops.sf_col`.
"""
import numpy as np

from refops_tracks import bilinear

SF_COLS = 32


def sf_col(s, r, m, k):
    return ((s * 2 + r) * 4 + m) * 2 + k


def warp_disparity(disp_next, flow, dtype=np.float64):
    """disp_next [B,H,W], flow [B,2,H,W] -> (disp_1 [B,H,W] of `dtype`, in_frame [B,H,W] bool)"""
    d = np.asarray(disp_next, np.float32).astype(dtype)
    f = np.asarray(flow, np.float32).astype(dtype)
    b, h, w = d.shape
    ys, xs = np.meshgrid(np.arange(h, dtype=dtype), np.arange(w, dtype=dtype), indexing="ij")
    out, inside = np.empty((b, h, w), dtype), np.empty((b, h, w), bool)
    for i in range(b):
        qx, qy = xs + f[i, 0], ys + f[i, 1]
        with np.errstate(invalid="ignore"):
            inside[i] = (qx >= 0) & (qx <= w - 1) & (qy >= 0) & (qy <= h - 1)
            cx = np.where(np.isnan(qx), 0, np.clip(qx, 0, w - 1)).astype(dtype)
            cy = np.where(np.isnan(qy), 0, np.clip(qy, 0, h - 1)).astype(dtype)
        out[i] = bilinear(d[i][None], cx, cy)[0]
    return out, inside


def disparity_outliers(gt, pred):
    """(valid, outlier) of UM_EVS_D1's fp32 expressions: gt > 0; |gt - pred| > 3 and |gt - pred| / gt > 0.05"""
    gt, pred = np.asarray(gt, np.float32), np.asarray(pred, np.float32)
    valid = gt > 0
    with np.errstate(invalid="ignore", divide="ignore"):
        e = np.abs(gt - pred)
        return valid, valid & (e > np.float32(3)) & (e / gt > np.float32(0.05))


def flow_outliers(gt, valid, pred):
    """(valid, outlier) of UM_EVF_OUTLIER's fp32 expressions on planar [..., 2, H, W] flows: valid >= 0.5; epe > 3 and
    epe / |gt| > 0.05"""
    gt, pred = np.asarray(gt, np.float32), np.asarray(pred, np.float32)
    v = np.asarray(valid, np.float32) >= np.float32(0.5)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        du, dv = pred[..., 0, :, :] - gt[..., 0, :, :], pred[..., 1, :, :] - gt[..., 1, :, :]
        epe = np.sqrt(du * du + dv * dv)
        mag = np.sqrt(gt[..., 0, :, :] * gt[..., 0, :, :] + gt[..., 1, :, :] * gt[..., 1, :, :])
        return v, v & (epe > np.float32(3)) & (epe / mag > np.float32(0.05))


def scene_flow_counts(disp0, disp1, flow, occ, noc=None, obj=None):
    """Count table [B, 32] (int64) of predictions disp0 / disp1 [B,H,W] and flow [B,2,H,W] against `occ` (and `noc`), dicts
    of 'disp0', 'disp1' [B,H,W], 'flow' [B,2,H,W] and 'flow_valid' [B,H,W]; obj [B,H,W] (nonzero = foreground) or None."""
    b = np.shape(disp0)[0]
    fg = np.zeros(np.shape(disp0), bool) if obj is None else np.asarray(obj, np.float32) != 0
    out = np.zeros((b, SF_COLS), np.int64)
    for s, gt in enumerate((occ, noc)):
        if gt is None:
            continue
        v0, o0 = disparity_outliers(gt["disp0"], disp0)
        v1, o1 = disparity_outliers(gt["disp1"], disp1)
        vf, of = flow_outliers(gt["flow"], gt["flow_valid"], flow)
        vs = v0 & v1 & vf
        os_ = vs & (o0 | o1 | of)
        for r, region in enumerate((~fg, fg)):
            for m, (v, o) in enumerate(((v0, o0), (v1, o1), (vf, of), (vs, os_))):
                out[:, sf_col(s, r, m, 0)] = (v & region).reshape(b, -1).sum(1)
                out[:, sf_col(s, r, m, 1)] = (o & region).reshape(b, -1).sum(1)
    return out
