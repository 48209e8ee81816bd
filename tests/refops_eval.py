"""CPU statement of the evaluation op `eval_stats` (test infrastructure, like tests/refops.py): the per-pixel fp32 torch / numpy
expressions of the reference's validate_* loops (evaluate_flow.py, evaluate_stereo.py, loss/stereo_metric.py,
loss/depth_loss.py:compute_errors), every operation correctly rounded, with the per-sample sums accumulated in float64.  The `-m gpu` tests compare the CUDA
op with it, and `register_cpu_kernels()` installs it -- together with every op of refops.py -- as a CPU kernel inside the
test process, so the validation drivers' host logic runs on a machine without a GPU."""
import numpy as np
import torch

import refops
from unimatch_b200 import ops


def _in_image(flow_gt):
    """utils/utils.py:compute_out_of_boundary_mask of planar GT flows [B, 2, H, W] -> bool [B, H, W]"""
    b, _, h, w = flow_gt.shape
    ys, xs = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    corres = torch.stack((xs, ys), 0).float()[None] + flow_gt
    m = (corres[:, 0] >= 0) & (corres[:, 0] <= w - 1) & (corres[:, 1] >= 0) & (corres[:, 1] <= h - 1)
    return m & (flow_gt[:, 0].abs() <= w - 1) & (flow_gt[:, 1].abs() <= h - 1)


def _s(x):
    return x.double().sum().item()


def _sqrt(x):
    """Correctly rounded fp32 square root (numpy, like the kernel's __fsqrt_rn).  torch's CPU float `sqrt` is not correctly
    rounded: in torch 2.11 it is one ulp off on about 0.7% of inputs, on every CPU capability level."""
    return torch.from_numpy(np.sqrt(x.contiguous().numpy()))


def _flow_rows(pred, gt, valid, noc_valid, mask_mode, max_val):
    epe = _sqrt(torch.sum((pred - gt) ** 2, dim=1))
    mag = _sqrt(torch.sum(gt ** 2, dim=1))
    if mask_mode == ops.EVAL_MASK_ALL:
        m = torch.ones_like(epe, dtype=torch.bool)
    elif mask_mode == ops.EVAL_MASK_VALID:
        m = valid >= 0.5
    else:
        m = (valid * (mag < max_val)) >= 0.5
    out = (epe > 3.0) & ((epe / mag) > 0.05)
    bins = (mag < 10, (mag >= 10) * (mag <= 40), mag > 40)
    matched = ((noc_valid > 0.5) & (_in_image(gt) > 0.5)) if noc_valid is not None else None
    rows = []
    for b in range(epe.shape[0]):
        e, mb = epe[b], m[b]
        row = [mb.sum().item(), _s(e[mb]), (e[mb] > 1).sum().item(), (e[mb] > 3).sum().item(), (e[mb] > 5).sum().item(),
               out[b][mb].sum().item()]
        for s in bins:
            sel = s[b] & mb
            row += [sel.sum().item(), _s(e[sel])]
        if matched is None:
            row += [0, 0.0, 0, 0.0]
        else:
            mt = matched[b] & mb
            um = ~matched[b] & mb
            row += [mt.sum().item(), _s(e[mt]), um.sum().item(), _s(e[um])]
        rows.append(row)
    return rows


def _stereo_rows(pred, gt, max_val):
    rows = []
    for b in range(pred.shape[0]):
        m = gt[b] > 0
        if max_val > 0:
            m = m & (gt[b] < max_val)
        d_est, d_gt = pred[b][m], gt[b][m]
        e = torch.abs(d_gt - d_est)
        rows.append([m.sum().item(), _s(e), ((e > 3) & (e / d_gt > 0.05)).sum().item(), (e > 1).sum().item(),
                     (e > 2).sum().item(), (e > 3).sum().item()])
    return rows


def _depth_rows(pred, gt, valid, eval_min, eval_max):
    rows = []
    with np.errstate(all="ignore"):
        for b in range(pred.shape[0]):
            m = (gt[b] > eval_min) & (gt[b] < eval_max)
            if valid is not None:
                m = m & (valid[b] > 0.5)
            m = m.numpy()
            g, p = gt[b].numpy()[m], pred[b].numpy()[m]
            thresh = np.maximum((g / p), (p / g))
            d = g - p
            f64 = lambda x: float(np.sum(x.astype(np.float64)))   # noqa: E731
            rows.append([int(m.sum()), f64(np.abs(d) / g), f64((d ** 2) / g), f64(d ** 2), f64((np.log(g) - np.log(p)) ** 2),
                         int((thresh < 1.25).sum()), int((thresh < 1.25 ** 2).sum()), int((thresh < 1.25 ** 3).sum())])
    return rows


def eval_stats(pred, gt, valid, noc_valid, task, mask_mode, max_val, eval_min, eval_max):
    """[B, S] float64 statistics table, columns ops.EVAL_COLS[task]"""
    pred, gt = pred.float(), gt.float()
    if task == ops.EVAL_FLOW:
        rows = _flow_rows(pred, gt, valid, noc_valid, mask_mode, max_val)
    elif task == ops.EVAL_STEREO:
        rows = _stereo_rows(pred, gt, max_val)
    else:
        rows = _depth_rows(pred, gt, valid, eval_min, eval_max)
    return torch.tensor(rows, dtype=torch.float64).reshape(pred.shape[0], len(ops.EVAL_COLS[task]))


ALL = ["eval_stats"]

_registered = []


def register_cpu_kernels():
    refops.register_cpu_kernels()
    if _registered:
        return
    lib = torch.library.Library("unimatch_sm100", "IMPL", "CPU")
    g = globals()
    for name in ALL:
        lib.impl(name, g[name])
    _registered.append(lib)
