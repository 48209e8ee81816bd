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

`validate_scene_flow` scores stereo scene flow (`infer_scene_flow`) with KITTI 2015's D1, D2, Fl and SF outliers
(`um_scene_flow_stats`), on the same batching and single download.

`tapvid_metrics` scores point tracks (e.g. `PointTrackRunner`'s) with TAP-Vid's metrics, in numpy on the host.
"""
import os

import numpy as np
import torch

from . import ops
from .inference import InputPadder, _resize, depth_to_image, infer_scene_flow

_OPS = torch.ops.unimatch_sm100

_FLOW_PADDING = {"chairs": None, "things": "sintel", "sintel": "sintel", "kitti": "kitti"}   # InputPadder mode per protocol
_STEREO_PROTOCOLS = {"things": ("d1",), "kitti15": ("d1", "3px"), "eth3d": ("1px",), "middlebury": ("2px",)}
_DEPTH_PROTOCOLS = ("scannet", "demon")
_DEPTH_NAMES = ("abs_rel", "sq_rel", "rmse", "rmse_log", "a1", "a2", "a3")


def _col(task, name):
    return ops.EVAL_COLS[task].index(name)


def _upload(t, device, keep_uint8=False):
    """A stacked host field on `device` through pinned memory, as float32 (uint8 kept as it is with `keep_uint8`)"""
    if not (keep_uint8 and t.dtype == torch.uint8):
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


def _statistics(samples, batch, device, run, columns, on_batch=None, keep_uint8=False):
    """Per-sample statistics table [N, columns] (float64, dataset order) of `samples`, an iterable of tuples of CPU tensors
    (None for an absent optional tensor) grouped by the shape of their first tensor into batches of `batch`; `run(*tensors)`
    gets each batch stacked on the device and returns its [n, columns] device table.  `on_batch(indices, table)`, when
    given, follows each `run` with the batch's dataset indices and its device table.  With `keep_uint8`, uint8 fields (frames
    as decoded) are uploaded as they are rather than as float32."""
    if batch < 1:
        raise ValueError("batch must be positive")
    device = torch.device(device)
    open_batches, order, tables = {}, [], []

    def flush(shape):
        items = open_batches.pop(shape)
        fields = [None if items[0][1][k] is None else _upload(torch.stack([it[1][k] for it in items]), device, keep_uint8)
                  for k in range(len(items[0][1]))]
        tables.append(run(*fields))
        order.extend(i for i, _ in items)
        if on_batch is not None:
            on_batch([i for i, _ in items], tables[-1])

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
class _DepthVisNames:
    """The file names `save_vis_depth` gives the samples (evaluate_depth.py:133-138, :272-276): the reference's
    `valid_samples` numbering, 1-based over the samples with a non-empty mask in dataset order, as `%04d_depth_pred.png`
    (scannet) or `%04d.png` (demon).  Batches arrive grouped by size, so out of dataset order: `add(indices, counts)` takes
    a batch's dataset indices and mask counts and returns the [(index, name)] whose number is now known, in dataset
    order; an empty-mask sample gets no name."""

    def __init__(self, protocol):
        self.pattern = "%04d_depth_pred.png" if protocol == "scannet" else "%04d.png"
        self.counts = {}
        self.next_index = 0
        self.valid_samples = 0

    def add(self, indices, counts):
        self.counts.update(zip(indices, counts))
        named = []
        while self.next_index in self.counts:
            if self.counts.pop(self.next_index) > 0:
                self.valid_samples += 1
                named.append((self.next_index, self.pattern % self.valid_samples))
            self.next_index += 1
        return named


@torch.no_grad()
def validate_depth(model, dataset, *, protocol, batch=8, device="cuda", padding_factor=16, inference_size=None,
                   num_depth_candidates=64, eval_min_depth=0.5, eval_max_depth=10, min_depth=0.5, max_depth=10,
                   save_vis_depth=False, save_dir=None, writers=4, **model_kwargs):
    """The results dict of evaluate_depth.py's `validate_<protocol>` on `dataset` (`protocol` 'scannet' or 'demon', the same
    loop): abs_rel, sq_rel, rmse, rmse_log, a1, a2, a3 of loss/depth_loss.py:compute_errors.  Inputs are padded with
    InputPadder mode 'kitti', or resized to `inference_size` with the depth resized back (not rescaled, as in the reference).
    The mask is `eval_min_depth < gt < eval_max_depth & valid > 0.5`; `min_depth` / `max_depth` are metric, the model gets
    their inverses.

    Kept quirk: samples with an empty mask are skipped, but the per-sample metrics are summed and divided by the number of
    samples in the dataset, skipped ones included (evaluate_depth.py:148).

    `save_vis_depth` writes, into `save_dir` (created if missing), the `viz_depth_tensor(1 / depth)` picture of every
    sample with a non-empty mask, named as the reference names it (`_DepthVisNames`).  The pictures are painted on the
    device (`depth_to_image`) from the unpadded or resized-back predictions the metrics are computed from, downloaded with
    the batch's mask counts (one wait per batch) and written by `writers` threads.  Without it the driver does exactly what
    it does otherwise."""
    if protocol not in _DEPTH_PROTOCOLS:
        raise ValueError("validate_depth: protocol must be one of %s" % list(_DEPTH_PROTOCOLS))
    if model_kwargs.setdefault("task", "depth") != "depth":
        raise ValueError("validate_depth drives the depth task only")
    if save_vis_depth and save_dir is None:
        raise ValueError("validate_depth: save_vis_depth needs save_dir")
    pictures = []                                        # the last batch's device pictures, with save_vis_depth

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
        if save_vis_depth:
            pictures[:] = [depth_to_image(pred)]
        return _OPS.eval_stats(pred, depth, valid, None, ops.EVAL_DEPTH, 0, 0.0, float(eval_min_depth), float(eval_max_depth))

    fields = ("img_ref", "img_tgt", "intrinsics", "pose", "depth", "valid")
    samples = (tuple(s[k] for k in fields) for s in dataset)
    if not save_vis_depth:
        T = _statistics(samples, batch, device, run, len(ops.EVAL_DEPTH_COLS))
        return _depth_results(T)
    from .submission import _WriterPool, _write_picture
    os.makedirs(save_dir, exist_ok=True)
    names, held = _DepthVisNames(protocol), {}
    pool = _WriterPool(writers, torch.device(device).type == "cuda")

    def on_batch(indices, table):
        slot, host, ready = pool.stage({"vis": pictures.pop(), "n": table[:, _col(ops.EVAL_DEPTH, "n")]})
        if ready is not None:
            ready.synchronize()
        for i, n, pic in zip(indices, host["n"], host["vis"]):
            if n > 0:
                held[i] = pic.copy()                    # the staging slot is reused two batches later
        for i, name in names.add(indices, host["n"]):
            pool.submit(slot, None, _write_picture, os.path.join(save_dir, name), held.pop(i))

    try:
        T = _statistics(samples, batch, device, run, len(ops.EVAL_DEPTH_COLS), on_batch)
    except BaseException as e:
        pool.close(error=e)
        raise
    pool.close()
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


# ---------------------------------------------------------------------------------------------------------- scene flow
_SF_VIEWS = ("left0", "right0", "left1", "right1")
_SF_GT = ("disp0", "disp1", "flow", "flow_valid")
_SF_NOC = ("disp0_noc", "disp1_noc", "flow_noc", "flow_noc_valid")


def _scene_flow_fields(s, index, noc, obj):
    """The tensors of scene-flow sample `index` in the order `validate_scene_flow`'s batches take them, checked: four uint8
    views [H,W,3] of one size, the ground truth at that size, the noc maps and obj_map when the dataset has them."""
    if not isinstance(s, dict):
        raise ValueError("validate_scene_flow: sample %d is not a dict" % index)
    keys = _SF_VIEWS + _SF_GT + (_SF_NOC if noc else ()) + (("obj_map",) if obj else ())
    if any(k in s for k in _SF_NOC) and not all(k in s for k in _SF_NOC):
        raise ValueError("validate_scene_flow: sample %d has some of the noc maps %s but not all" % (index, list(_SF_NOC)))
    missing = [k for k in keys if k not in s]
    if missing:
        raise ValueError("validate_scene_flow: sample %d lacks %s" % (index, missing))
    if (all(k in s for k in _SF_NOC), "obj_map" in s) != (noc, obj):
        raise ValueError("validate_scene_flow: sample %d differs from the first in its noc maps or obj_map" % index)
    f = {k: torch.as_tensor(s[k]) for k in keys}
    h, w = f["left0"].shape[:2] if f["left0"].dim() == 3 else (-1, -1)
    for k in _SF_VIEWS:
        if f[k].dtype != torch.uint8 or tuple(f[k].shape) != (h, w, 3):
            raise ValueError("validate_scene_flow: sample %d: the views must be uint8 [H,W,3] of one size (%s is %s)"
                             % (index, k, list(f[k].shape)))
    for k in keys[4:]:
        shape = (2, h, w) if k in ("flow", "flow_noc") else (h, w)
        if tuple(f[k].shape) != shape:
            raise ValueError("validate_scene_flow: sample %d: %s must be %s" % (index, k, list(shape)))
    # the order `validate_scene_flow`'s run() takes: views, gt, the four noc maps or four Nones, obj_map or None
    return (tuple(f[k] for k in _SF_VIEWS + _SF_GT) + (tuple(f[k] for k in _SF_NOC) if noc else (None,) * len(_SF_NOC))
            + ((f["obj_map"],) if obj else (None,)))


@torch.no_grad()
def validate_scene_flow(stereo_model, flow_model, dataset, *, batch=8, device="cuda", stereo_kwargs=None, flow_kwargs=None,
                        stereo_padding_factor=16, flow_padding_factor=32, stereo_inference_size=None,
                        flow_inference_size=None):
    """KITTI 2015 scene-flow results of `infer_scene_flow` on `dataset`: the devkit's D1, D2, Fl and SF outlier rates.

    Samples are dicts with uint8 'left0', 'right0', 'left1', 'right1' [H,W,3] and the ground truth as float maps: 'disp0',
    'disp1' [H,W] (KITTI's PNG / 256, 0 = no ground truth), 'flow' [2,H,W] and 'flow_valid' [H,W] (>= 0.5 = valid).  Optional,
    in every sample or in none: 'disp0_noc', 'disp1_noc', 'flow_noc', 'flow_noc_valid' (the non-occluded set, the same
    encoding) and 'obj_map' [H,W] (nonzero = foreground).
    Per set (occ = all pixels, noc) and region: a disparity pixel is valid where its gt > 0 and an outlier where e > 3 and
    e / gt > 0.05 (e = |gt - pred|; D1 on disp_0, D2 on disp_1); a flow pixel is valid where flow_valid >= 0.5 and an outlier
    where epe > 3 and epe / |gt| > 0.05 (Fl); an SF pixel is valid where all three are and an outlier where any of the three
    is.  Each value is 100 * outliers / valid pixels over the whole dataset, summed in float64 as the devkit sums them.
    Returns `kitti_sf_{occ,noc}_{d1,d2,fl,sf}_{bg,fg,all}`; without noc maps there are no noc keys, without obj_map the fg
    keys are NaN (every pixel is background), and an empty set gives NaN.

    These are not comparable bit for bit with `validate_stereo(protocol='kitti15')` / `validate_flow(protocol='kitti')`:
    those follow the reference's padding validators, this follows the inference geometry of `infer_scene_flow` (resize to a
    multiple of the padding factor and back), the geometry the runner and the submission writer use.
    Samples of one size form batches of `batch` (one open batch per size), one `um_scene_flow_stats` launch per batch, one
    download at the end."""
    first = {}

    def samples():
        for i, s in enumerate(dataset):
            if not first:
                first.update(noc=isinstance(s, dict) and all(k in s for k in _SF_NOC),
                             obj=isinstance(s, dict) and "obj_map" in s)
            yield _scene_flow_fields(s, i, first["noc"], first["obj"])

    def run(left0, right0, left1, right1, disp0, disp1, flow, valid, nd0, nd1, nf, nv, obj):
        out = infer_scene_flow(stereo_model, flow_model, left0, right0, left1, right1, stereo_kwargs=stereo_kwargs,
                               flow_kwargs=flow_kwargs, stereo_padding_factor=stereo_padding_factor,
                               flow_padding_factor=flow_padding_factor, stereo_inference_size=stereo_inference_size,
                               flow_inference_size=flow_inference_size)
        # the frames travel as uint8; a ground-truth map or obj_map given as uint8 is widened here, on the device
        maps = [None if t is None else t.float() for t in (disp0, disp1, flow, valid, nd0, nd1, nf, nv, obj)]
        return _OPS.scene_flow_stats(out["disp_0"], out["disp_1"], out["flow"], *maps)

    T = _statistics(samples(), batch, device, run, ops.SF_COLS, keep_uint8=True)
    return scene_flow_results(T.sum(axis=0) if len(T) else np.zeros(ops.SF_COLS), first.get("noc", False))


def scene_flow_results(counts, noc):
    """The results dict of a summed count table [SF_COLS] (columns `ops.sf_col`): 100 * outliers / valid per set, metric
    and region, 'all' = bg + fg; NaN for an empty set; the noc keys only when `noc`."""
    res = {}
    for s, set_name in enumerate(ops.SF_SETS[:2 if noc else 1]):
        for m, metric in enumerate(ops.SF_METRICS):
            n = [counts[ops.sf_col(s, r, m, 0)] for r in range(2)]
            o = [counts[ops.sf_col(s, r, m, 1)] for r in range(2)]
            for key, num, den in (("bg", o[0], n[0]), ("fg", o[1], n[1]), ("all", o[0] + o[1], n[0] + n[1])):
                res["kitti_sf_%s_%s_%s" % (set_name, metric, key)] = _ratio(100.0 * np.float64(num), den)
    return res


# ---------------------------------------------------------------------------------------------------------- point tracks
TAPVID_THRESHOLDS = (1, 2, 4, 8, 16)


def tapvid_metrics(query_points, gt_occluded, gt_tracks, pred_occluded, pred_tracks, query_mode):
    """TAP-Vid's point-tracking metrics per video, in numpy (the arrays are tiny).

    `query_points` [B,N,3] (t_q, y, x); `gt_occluded` / `pred_occluded` [B,N,T] bool; `gt_tracks` / `pred_tracks` [B,N,T,2]
    (x, y).  Coordinates are compared as given: TAP-Vid's protocol rescales them to 256x256 first, which is the caller's job.
    The evaluation points of a track are its frames t > t_q (`query_mode='first'`) or t != t_q (`'strided'`).
      * occlusion_accuracy: share of evaluation points where the predicted and true occlusion agree;
      * for d in 1, 2, 4, 8, 16 with within = |pred - gt|^2 < d^2 and vis = not occluded:
        pts_within_d = sum(within & gt_vis & eval) / sum(gt_vis & eval),
        jaccard_d = TP / (sum(gt_vis & eval) + FP), TP = sum(within & gt_vis & pred_vis & eval),
        FP = sum((~gt_vis | ~within) & pred_vis & eval);
      * average_pts_within_thresh and average_jaccard: their means over the five d.
    Every value is float64 of shape [B]; 0 / 0 gives NaN."""
    if query_mode not in ("first", "strided"):
        raise ValueError("tapvid_metrics: query_mode is 'first' or 'strided'")
    qp = np.asarray(query_points)
    gt_occ, pred_occ = np.asarray(gt_occluded).astype(bool), np.asarray(pred_occluded).astype(bool)
    gt, pred = np.asarray(gt_tracks, np.float64), np.asarray(pred_tracks, np.float64)
    b, n, t = gt_occ.shape
    if qp.shape != (b, n, 3) or pred_occ.shape != (b, n, t) or gt.shape != (b, n, t, 2) or pred.shape != (b, n, t, 2):
        raise ValueError("tapvid_metrics: query_points [B,N,3], occlusions [B,N,T] and tracks [B,N,T,2] must agree")
    tq = np.round(qp[..., 0]).astype(np.int64)[..., None]
    frames = np.arange(t)[None, None]
    evals = frames > tq if query_mode == "first" else frames != tq

    def ratio(num, den):
        with np.errstate(invalid="ignore", divide="ignore"):
            return np.asarray(num, np.float64) / np.asarray(den, np.float64)

    out = {"occlusion_accuracy": ratio(((gt_occ == pred_occ) & evals).sum((1, 2)), evals.sum((1, 2)))}
    gt_vis, pred_vis = ~gt_occ, ~pred_occ
    dist2 = ((pred - gt) ** 2).sum(-1)
    visible = (gt_vis & evals).sum((1, 2))
    for d in TAPVID_THRESHOLDS:
        within = dist2 < d * d
        out["pts_within_%d" % d] = ratio((within & gt_vis & evals).sum((1, 2)), visible)
        tp = (within & gt_vis & pred_vis & evals).sum((1, 2))
        fp = ((~gt_vis | ~within) & pred_vis & evals).sum((1, 2))
        out["jaccard_%d" % d] = ratio(tp, visible + fp)
    out["average_pts_within_thresh"] = np.mean([out["pts_within_%d" % d] for d in TAPVID_THRESHOLDS], axis=0)
    out["average_jaccard"] = np.mean([out["jaccard_%d" % d] for d in TAPVID_THRESHOLDS], axis=0)
    return out
