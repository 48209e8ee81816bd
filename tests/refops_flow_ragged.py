"""Statement of the ragged flow ops (test infrastructure, like tests/refops_ragged.py): every item of a ragged op is what
the uniform op gives on that image alone, so each function below calls the uniform op once per item, on the inputs'
device -- the CUDA op on a GPU, the CPU statements of refops_video / refops.py otherwise.  `refops.register_cpu_kernels()`
installs the three new ops as CPU kernels inside the test process; `resize_bilinear_ragged` here states the op with
RAGGED_TRANSPOSE and is called directly (the op's registered statement is tests/refops_ragged.py's, without the flag).
`composed_flow_reference` states what `MixedSizeFlowRunner` computes, from existing functions only."""
import torch

from refops_ragged import _fits, items_of
from unimatch_b200 import ops

_OPS = torch.ops.unimatch_sm100


def frames_to_planar_ragged(frames, items, h_max, w_max, h_out, w_out):
    """frame i -> um_frames_to_planar of [1, h_i, w_i, 3] alone, transposed when the item says so; a skipped item leaves
    zeros here (the kernel leaves its image unwritten)"""
    out = torch.zeros((items.shape[0], 3, h_out, w_out), device=frames.device)
    for n, it in enumerate(items_of(items)):
        if _fits(it, h_max, w_max, 3, frames.numel()):
            h, w, o = int(it["h"]), int(it["w"]), int(it["offset"])
            f = frames.reshape(-1)[o:o + 3 * h * w].view(1, h, w, 3).contiguous()
            out[n] = _OPS.frames_to_planar(f, h_out, w_out, bool(int(it["flags"]) & ops.RAGGED_TRANSPOSE))[0]
    return out


def resize_bilinear_ragged(x, items, h_max, w_max, out_numel):
    """item i -> um_resize_bilinear of image i alone with scale [items[i].scale] and the flip; with RAGGED_TRANSPOSE the
    resize goes to (w_i, h_i) and the item is its transpose; an item at the input size (swapped for a transposed one)
    without the flip is image i as it is (transposed)"""
    out = torch.zeros((out_numel,), device=x.device)
    for n, it in enumerate(items_of(items)):
        if not _fits(it, h_max, w_max, 1, out_numel):
            continue
        h, w, o = int(it["h"]), int(it["w"]), int(it["offset"])
        flip = bool(int(it["flags"]) & ops.RAGGED_FLIP_X)
        t = bool(int(it["flags"]) & ops.RAGGED_TRANSPOSE)
        ho, wo = (w, h) if t else (h, w)
        if (ho, wo) == tuple(x.shape[-2:]) and not flip:
            v = x[n, 0]
        else:
            v = _OPS.resize_bilinear(x[n:n + 1].contiguous(), ho, wo, [float(it["scale"])], flip)[0, 0]
        out[o:o + h * w] = (v.transpose(0, 1) if t else v).reshape(-1)
    return out


def flow_to_image_ragged(flow, flow_items, out, picture_items, h_max, w_max):
    """picture i -> um_flow_to_image of flow i alone, at its own byte offset; skipped unless both descriptors fit and agree"""
    flat = out.view(-1)
    for f, p in zip(items_of(flow_items), items_of(picture_items)):
        h, w = int(f["h"]), int(f["w"])
        if (h, w) == (int(p["h"]), int(p["w"])) and _fits(f, h_max, w_max, 2, flow.numel()) and _fits(p, h_max, w_max, 3, out.numel()):
            pic = torch.empty((1, h, w, 3), dtype=torch.uint8, device=flow.device)
            _OPS.flow_to_image(flow.reshape(-1)[int(f["offset"]):int(f["offset"]) + 2 * h * w].view(1, 2, h, w).contiguous(), pic)
            flat[int(p["offset"]):int(p["offset"]) + 3 * h * w] = pic.reshape(-1)


def fb_consistency_ragged(flow, flow_items, occ, occ_items, h_max, w_max, alpha, beta):
    """masks of pair i -> um_fb_consistency of its forward and backward flow alone; skipped unless the four descriptors fit
    and have one size of at least 2 x 2"""
    fi, oi = items_of(flow_items), items_of(occ_items)
    n = len(fi) // 2
    for i in range(n):
        four = (fi[i], fi[n + i], oi[i], oi[n + i])
        h, w = int(fi[i]["h"]), int(fi[i]["w"])
        if any((int(it["h"]), int(it["w"])) != (h, w) for it in four) or h < 2 or w < 2:
            continue
        if not all(_fits(it, h_max, w_max, per, buf.numel()) for it, per, buf in zip(four, (2, 2, 1, 1), (flow, flow, occ, occ))):
            continue
        fwd, bwd = (flow.reshape(-1)[int(it["offset"]):int(it["offset"]) + 2 * h * w].view(1, 2, h, w).contiguous()
                    for it in four[:2])
        for it, m in zip(four[2:], _OPS.fb_consistency(fwd, bwd, float(alpha), float(beta))):
            occ.view(-1)[int(it["offset"]):int(it["offset"]) + h * w] = m.reshape(-1)


def composed_flow_reference(model, call, pairs, batch, max_buckets, padding_factor=32, inference_size=None,
                            pred_bidir_flow=False, pred_bwd_flow=False, fwd_bwd_consistency_check=False, only=None):
    """{index: result} of `MixedSizeFlowRunner`'s steps over `pairs` (host uint8 (image1, image2) [h, w, 3]), recomputed from
    existing functions only: the steps formed by `_batches` with the same bucket rule, each filled with its last pair; every
    frame brought to the bucket size by `um_frames_to_planar` alone (with its portrait transpose), concatenated, the two
    views swapped for `pred_bwd_flow`; one forward per step, as `infer_flow` calls it; `_flow_outputs` (the rest of
    `infer_flow`) once per distinct original size in the step, on the whole step batch, each pair's result taken from the
    call for its own size; the pictures from `flow_to_image`.  `only`: a set of indices; steps holding none are skipped."""
    from unimatch_b200.inference import _batches, _flow_outputs, _frame_geometry, flow_to_image

    def geometry(p):
        return _frame_geometry(p[0].shape[0], p[0].shape[1], padding_factor, inference_size, "flow")

    res = {}
    for step in _batches(list(enumerate(pairs)), batch, lambda s: geometry(s[1])[2], max_buckets):
        if only is not None and not any(i in only for i, _ in step):
            continue
        size = geometry(step[0][1])[2]
        full = [step[min(i, len(step) - 1)] for i in range(batch)]
        views = [torch.cat([_OPS.frames_to_planar(torch.as_tensor(p[side])[None].cuda().contiguous(), size[0], size[1],
                                                  geometry(p)[0]) for _, p in full]) for side in range(2)]
        if pred_bwd_flow:
            views.reverse()
        flow = model(views[0], views[1], pred_bidir_flow=pred_bidir_flow, task="flow", **call)["flow_preds"][-1]
        for shape in sorted({tuple(p[0].shape[:2]) for _, p in step}):
            transposed, ori, _ = _frame_geometry(shape[0], shape[1], padding_factor, inference_size, "flow")
            out = _flow_outputs(flow, ori, size, transposed, pred_bidir_flow, fwd_bwd_consistency_check)
            for i, (index, p) in enumerate(step):
                if tuple(p[0].shape[:2]) == shape:
                    r = {k: v[i].contiguous().cpu() for k, v in out.items()}
                    for k in [k for k in r if k.startswith("flow")]:
                        r[k.replace("flow", "vis")] = flow_to_image(r[k][None].cuda())[0].cpu()
                    res[index] = r
    return res

