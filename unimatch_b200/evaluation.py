"""Batched validation on the device: the reference's `--eval` loops with their results dicts, keys and values.

`validate_flow` (evaluate_flow.py:160-638: validate_chairs / validate_things / validate_sintel / validate_kitti),
`validate_stereo` (evaluate_stereo.py:302-708: validate_things / validate_kitti15 / validate_eth3d / validate_middlebury) and
`validate_depth` (evaluate_depth.py:22-293: validate_scannet / validate_demon) take the model and any sequence or iterable of
the reference datasets' samples -- the reference's own dataset objects can be passed as they are:

  * flow:   tuples (img1, img2, flow_gt, valid[, noc_valid])            (dataloader/flow/datasets.py)
  * stereo: dicts with 'left', 'right', 'disp'                           (dataloader/stereo/datasets.py)
  * depth:  dicts with 'img_ref', 'img_tgt', 'intrinsics', 'pose', 'depth', 'valid'   (dataloader/depth/datasets.py)

Where the reference runs one pair per `model(...)` call and copies every prediction to the host to compute its metrics there,
these drivers group samples of equal size into batches of `batch` (one open batch per size, flushed when full and at the end),
upload them through pinned memory, pad with the reference's `InputPadder` mode, run the model and reduce the unpadded
predictions to per-sample statistics with one `um_eval_stats` launch per batch.  The statistics tables stay on the device
until the single download at the end; the flow and stereo drivers issue no other host synchronisation (the depth model
synchronises once per batch for its `torch.inverse`).  The metrics are then formed on the host in float64, following each
reference loop -- including its quirks, listed in each driver's docstring.
"""
import numpy as np
import torch

from . import ops
from .inference import InputPadder, _resize

_OPS = torch.ops.unimatch_sm100

_FLOW_PADDING = {"chairs": None, "things": "sintel", "sintel": "sintel", "kitti": "kitti"}   # InputPadder mode per protocol
_STEREO_PROTOCOLS = {"things": ("d1",), "kitti15": ("d1", "3px"), "eth3d": ("1px",), "middlebury": ("2px",)}
_DEPTH_PROTOCOLS = ("scannet", "demon")
_DEPTH_NAMES = ("abs_rel", "sq_rel", "rmse", "rmse_log", "a1", "a2", "a3")


def _col(task, name):
    return ops.EVAL_COLS[task].index(name)


def _upload(t, device):
    t = t.float()
    if device.type == "cuda":
        return t.pin_memory().to(device, non_blocking=True)
    return t.to(device)


def _download(table):
    """The one device -> host copy of a driver: into pinned memory, then wait for that copy only."""
    if table.device.type != "cuda":
        return table.numpy()
    host = torch.empty(table.shape, dtype=table.dtype, pin_memory=True)
    host.copy_(table, non_blocking=True)
    done = torch.cuda.Event()
    done.record()
    done.synchronize()
    return host.numpy()


def _statistics(samples, batch, device, run, columns):
    """Per-sample statistics table [N, columns] (float64, dataset order) of `samples`, an iterable of tuples of CPU tensors
    (None for an absent optional tensor) grouped by the shape of their first tensor into batches of `batch`; `run(*tensors)`
    gets each batch stacked on the device and returns its [n, columns] device table."""
    if batch < 1:
        raise ValueError("batch must be positive")
    device = torch.device(device)
    open_batches, order, tables = {}, [], []

    def flush(shape):
        items = open_batches.pop(shape)
        fields = [None if items[0][1][k] is None else _upload(torch.stack([it[1][k] for it in items]), device)
                  for k in range(len(items[0][1]))]
        tables.append(run(*fields))
        order.extend(i for i, _ in items)

    for i, fields in enumerate(samples):
        fields = tuple(None if f is None else torch.as_tensor(f) for f in fields)
        shape = tuple(fields[0].shape)
        open_batches.setdefault(shape, []).append((i, fields))
        if len(open_batches[shape]) == batch:
            flush(shape)
    for shape in list(open_batches):
        flush(shape)
    if not tables:
        return np.zeros((0, columns))
    host = _download(torch.cat(tables))
    out = np.empty_like(host)
    out[np.asarray(order)] = host
    return out


def _ratio(num, den):
    """num / den in float64; an empty selection gives NaN, as the mean of an empty array does."""
    return float(np.float64(num) / den) if den else float("nan")


# ---------------------------------------------------------------------------------------------------------------- flow
@torch.no_grad()
def validate_flow(model, dataset, *, protocol, dstype="clean", batch=8, device="cuda", padding_factor=8,
                  with_speed_metric=False, evaluate_matched_unmatched=False, average_over_pixels=True, max_val_flow=400,
                  **model_kwargs):
    """The results dict of evaluate_flow.py's `validate_<protocol>` on `dataset`, `protocol` one of 'chairs', 'things',
    'sintel', 'kitti'.  `dstype` names the pass in the keys: 'clean' / 'final' (Sintel: 'sintel_<dstype>_*'; Things:
    'things_clean_*' / 'things_final_*', 'frames_cleanpass' / 'frames_finalpass' accepted).  `model_kwargs` go to `model(...)`
    (attn_type, attn_splits_list, corr_radius_list, prop_radius_list, num_reg_refine).

    Masks and padding as in the reference: Chairs is not padded, Things and Sintel use InputPadder mode 'sintel', KITTI mode
    'kitti'.  Chairs and Sintel average over EVERY pixel and ignore `valid`; Things evaluates `valid * (|gt| < max_val_flow)
    >= 0.5`, KITTI `valid >= 0.5`.  Kept quirks:
      * speed-bin means ('_s0_10', '_s10_40', '_s40+') are over the concatenated pixels of the samples where the bin is
        non-empty; with `average_over_pixels=False` (KITTI) they are means of the per-sample means over those samples;
      * Sintel's matched / unmatched means (`evaluate_matched_unmatched`, samples need `noc_valid`) take both from the samples
        whose matched set is non-empty only;
      * KITTI's 'kitti_f1' is x100, the mean of a float32 0/1 array (so a float32 value); `average_over_pixels=False` makes
        'kitti_epe' the mean of per-sample means (an empty sample gives NaN there, as `.mean()` does)."""
    if protocol not in _FLOW_PADDING:
        raise ValueError("validate_flow: protocol must be one of %s" % sorted(_FLOW_PADDING))
    if model_kwargs.setdefault("task", "flow") != "flow":
        raise ValueError("validate_flow drives the flow task only")
    matched = protocol == "sintel" and evaluate_matched_unmatched
    mode = _FLOW_PADDING[protocol]
    mask_mode = {"chairs": ops.EVAL_MASK_ALL, "sintel": ops.EVAL_MASK_ALL, "things": ops.EVAL_MASK_VALID_MAX,
                 "kitti": ops.EVAL_MASK_VALID}[protocol]

    def samples():
        for s in dataset:
            if matched and len(s) < 5:
                raise ValueError("validate_flow: evaluate_matched_unmatched needs (img1, img2, flow_gt, valid, noc_valid) samples")
            yield (s[0], s[1], s[2], s[3] if mask_mode != ops.EVAL_MASK_ALL else None, s[4] if matched else None)

    def run(img1, img2, flow_gt, valid, noc):
        padder = None
        if mode is not None:
            padder = InputPadder(img1.shape, mode=mode, padding_factor=padding_factor)
            img1, img2 = padder.pad(img1, img2)
        pred = model(img1, img2, **model_kwargs)["flow_preds"][-1]
        if padder is not None:
            pred = padder.unpad(pred)
        return _OPS.eval_stats(pred, flow_gt, valid, noc, ops.EVAL_FLOW, mask_mode, float(max_val_flow), 0.0, 0.0)

    T = _statistics(samples(), batch, device, run, len(ops.EVAL_FLOW_COLS))
    return _flow_results(T, protocol, dstype, with_speed_metric, matched, average_over_pixels)


def _flow_results(T, protocol, dstype, with_speed_metric, matched, average_over_pixels):
    c = {k: T[:, _col(ops.EVAL_FLOW, k)] for k in ops.EVAL_FLOW_COLS}
    n = c["n"].sum()
    if protocol == "sintel":
        prefix = "sintel_" + dstype
    elif protocol == "things":
        prefix = "things_" + {"frames_cleanpass": "clean", "frames_finalpass": "final"}.get(dstype, dstype)
    else:
        prefix = protocol
    res = {}
    if protocol == "kitti":
        if average_over_pixels:
            res["kitti_epe"] = _ratio(c["epe"].sum(), n)
        else:
            with np.errstate(invalid="ignore", divide="ignore"):
                res["kitti_epe"] = float(np.mean(c["epe"] / c["n"]))
        # np.mean of the float32 0/1 outlier array is a float32, and 100 * that stays float32 (evaluate_flow.py:613)
        res["kitti_f1"] = float(np.float32(100) * np.float32(c["outlier"].sum() / n)) if n else float("nan")
    else:
        res[prefix + "_epe"] = _ratio(c["epe"].sum(), n)
        if protocol != "things":
            for px in ("1px", "3px", "5px"):
                res["%s_%s" % (prefix, px)] = _ratio(c[px].sum(), n)
    if with_speed_metric:
        for key, b in (("_s0_10", "s0_10"), ("_s10_40", "s10_40"), ("_s40+", "s40")):
            bn, be = c[b + "_n"], c[b + "_epe"]
            if protocol == "kitti" and not average_over_pixels:
                nz = bn > 0
                res[prefix + key] = float(np.sum(be[nz] / bn[nz]) / nz.sum()) if nz.any() else float("nan")
            else:
                res[prefix + key] = _ratio(be.sum(), bn.sum())
    if matched:
        keep = c["matched_n"] > 0
        res[prefix + "_matched"] = _ratio(c["matched_epe"][keep].sum(), c["matched_n"][keep].sum())
        res[prefix + "_unmatched"] = _ratio(c["unmatched_epe"][keep].sum(), c["unmatched_n"][keep].sum())
    return res


# -------------------------------------------------------------------------------------------------------------- stereo
@torch.no_grad()
def validate_stereo(model, dataset, *, protocol, batch=8, device="cuda", padding_factor=16, inference_size=None,
                    max_disp=400, **model_kwargs):
    """The results dict of evaluate_stereo.py's `validate_<protocol>` on `dataset`, `protocol` one of 'things', 'kitti15',
    'eth3d', 'middlebury'.  Inputs are padded with InputPadder mode 'sintel', or resized to `inference_size` with the
    disparity resized back and rescaled by the width ratio.  The mask is `gt > 0`, and `gt < max_disp` for 'things'.

    Kept quirks: samples with an empty mask are skipped (the reference does not even run the model on them), and every metric
    is the mean over the remaining samples of the per-sample means -- end-point error and the float32 D1 / n-px ratios
    (torch means, so float32 values) accumulated in that order."""
    if protocol not in _STEREO_PROTOCOLS:
        raise ValueError("validate_stereo: protocol must be one of %s" % sorted(_STEREO_PROTOCOLS))
    if model_kwargs.setdefault("task", "stereo") != "stereo":
        raise ValueError("validate_stereo drives the stereo task only")
    limit = float(max_disp) if protocol == "things" else 0.0

    def run(left, right, disp):
        ori = tuple(left.shape[-2:])
        if inference_size is None:
            padder = InputPadder(left.shape, padding_factor=padding_factor)
            left, right = padder.pad(left, right)
            pred = padder.unpad(model(left, right, **model_kwargs)["flow_preds"][-1])
        else:
            size = (int(inference_size[0]), int(inference_size[1]))
            pred = model(_resize(left, size), _resize(right, size), **model_kwargs)["flow_preds"][-1]
            pred = _resize(pred.unsqueeze(1), ori, [ori[1] / float(size[1])]).squeeze(1)
        return _OPS.eval_stats(pred, disp, None, None, ops.EVAL_STEREO, 0, limit, 0.0, 0.0)

    T = _statistics(((s["left"], s["right"], s["disp"]) for s in dataset), batch, device, run, len(ops.EVAL_STEREO_COLS))
    return _stereo_results(T, protocol)


def _stereo_results(T, protocol):
    c = {k: T[:, _col(ops.EVAL_STEREO, k)] for k in ops.EVAL_STEREO_COLS}
    sums = {"epe": 0.0}
    sums.update({k: 0.0 for k in _STEREO_PROTOCOLS[protocol]})
    valid_samples = 0
    for i in range(T.shape[0]):
        n = c["n"][i]
        if n == 0:
            continue
        valid_samples += 1
        sums["epe"] += float(np.float32(c["abs"][i] / n))
        for k in _STEREO_PROTOCOLS[protocol]:
            sums[k] += float(np.float32(c[k][i] / n))
    return {"%s_%s" % (protocol, k): (v / valid_samples if valid_samples else float("nan")) for k, v in sums.items()}


# --------------------------------------------------------------------------------------------------------------- depth
@torch.no_grad()
def validate_depth(model, dataset, *, protocol, batch=8, device="cuda", padding_factor=16, inference_size=None,
                   num_depth_candidates=64, eval_min_depth=0.5, eval_max_depth=10, min_depth=0.5, max_depth=10,
                   **model_kwargs):
    """The results dict of evaluate_depth.py's `validate_<protocol>` on `dataset` (`protocol` 'scannet' or 'demon', the same
    loop): abs_rel, sq_rel, rmse, rmse_log, a1, a2, a3 of loss/depth_loss.py:compute_errors.  Inputs are padded with
    InputPadder mode 'kitti', or resized to `inference_size` with the depth resized back (not rescaled, as in the reference).
    The mask is `eval_min_depth < gt < eval_max_depth & valid > 0.5`; `min_depth` / `max_depth` are metric, the model gets
    their inverses.

    Kept quirk: samples with an empty mask are skipped, but the per-sample metrics are summed and divided by the number of
    samples in the dataset, skipped ones included (evaluate_depth.py:148)."""
    if protocol not in _DEPTH_PROTOCOLS:
        raise ValueError("validate_depth: protocol must be one of %s" % list(_DEPTH_PROTOCOLS))
    if model_kwargs.setdefault("task", "depth") != "depth":
        raise ValueError("validate_depth drives the depth task only")

    def run(img_ref, img_tgt, intrinsics, pose, depth, valid):
        ori = tuple(img_ref.shape[-2:])
        if inference_size is None:
            padder = InputPadder(img_ref.shape, mode="kitti", padding_factor=padding_factor)
            img_ref, img_tgt = padder.pad(img_ref, img_tgt)
        else:
            size = (int(inference_size[0]), int(inference_size[1]))
            img_ref, img_tgt = _resize(img_ref, size), _resize(img_tgt, size)
        pred = model(img_ref, img_tgt, intrinsics=intrinsics, pose=pose, min_depth=1. / max_depth, max_depth=1. / min_depth,
                     num_depth_candidates=num_depth_candidates, **model_kwargs)["flow_preds"][-1]
        pred = padder.unpad(pred) if inference_size is None else _resize(pred.unsqueeze(1), ori).squeeze(1)
        return _OPS.eval_stats(pred, depth, valid, None, ops.EVAL_DEPTH, 0, 0.0, float(eval_min_depth), float(eval_max_depth))

    fields = ("img_ref", "img_tgt", "intrinsics", "pose", "depth", "valid")
    T = _statistics((tuple(s[k] for k in fields) for s in dataset), batch, device, run, len(ops.EVAL_DEPTH_COLS))
    return _depth_results(T)


def _depth_results(T):
    c = {k: T[:, _col(ops.EVAL_DEPTH, k)] for k in ops.EVAL_DEPTH_COLS}
    error_sum = np.zeros(len(_DEPTH_NAMES))
    for i in range(T.shape[0]):
        n = c["n"][i]
        if n == 0:
            continue
        error_sum += [c["abs_rel"][i] / n, c["sq_rel"][i] / n, np.sqrt(c["sq"][i] / n), np.sqrt(c["log_sq"][i] / n),
                      c["a1"][i] / n, c["a2"][i] / n, c["a3"][i] / n]
    num_samples = T.shape[0]
    return {k: (float(v / num_samples) if num_samples else float("nan")) for k, v in zip(_DEPTH_NAMES, error_sum)}
