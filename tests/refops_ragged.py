"""Statement of the ragged stereo ops (test infrastructure, like tests/refops_stereo.py): every item of a ragged op is what
the uniform op gives on that image alone, so each function below calls the uniform op once per item, on the inputs'
device -- the CUDA op on a GPU, the CPU statements of refops_depth / refops_stereo / refops.py otherwise.
`refops.register_cpu_kernels()` installs these as the CPU kernels of the ragged ops inside the test process.
`composed_stereo_reference` states what `MixedSizeStereoRunner` computes, from existing functions only."""
import numpy as np
import torch

import refops_depth
from unimatch_b200 import ops
from unimatch_b200.inference import RAGGED_ITEM

_OPS = torch.ops.unimatch_sm100


def items_of(table):
    """uint8 [n, 24] descriptor table (any device) -> numpy records (offset, h, w, scale, flags)"""
    return table.cpu().contiguous().numpy().view(RAGGED_ITEM).reshape(-1)


def table(recs, device=None):
    """records (offset, h, w, scale, flags) -> uint8 [n, 24] descriptor table on `device`, a tensor that owns its memory: the
    inverse of items_of"""
    t = np.array(list(recs), RAGGED_ITEM).view(np.uint8).reshape(-1, ops.RAGGED_ITEM_BYTES)
    return torch.from_numpy(t.copy()).to(device)


def _fits(it, h_max, w_max, per_pixel, numel):
    h, w, o = int(it["h"]), int(it["w"]), int(it["offset"])
    return 0 < h <= h_max and 0 < w <= w_max and o >= 0 and o + per_pixel * h * w <= numel


def frames_to_planar_normalized_ragged(frames, items, h_max, w_max, h_out, w_out, mean, std):
    """frame i -> um_frames_to_planar_normalized of [1, h_i, w_i, 3] alone; a skipped item leaves zeros here (the kernel
    leaves its image unwritten)"""
    out = torch.zeros((items.shape[0], 3, h_out, w_out), device=frames.device)
    for n, it in enumerate(items_of(items)):
        if _fits(it, h_max, w_max, 3, frames.numel()):
            h, w, o = int(it["h"]), int(it["w"]), int(it["offset"])
            f = frames.reshape(-1)[o:o + 3 * h * w].view(1, h, w, 3).contiguous()
            out[n] = _OPS.frames_to_planar_normalized(f, h_out, w_out, list(mean), list(std))[0]
    return out


def resize_bilinear_ragged(x, items, h_max, w_max, out_numel):
    """item i -> um_resize_bilinear of image i alone with scale [items[i].scale] and the flip; an item at the input size
    without the flip is image i as it is"""
    out = torch.zeros((out_numel,), device=x.device)
    for n, it in enumerate(items_of(items)):
        if not _fits(it, h_max, w_max, 1, out_numel):
            continue
        h, w, o = int(it["h"]), int(it["w"]), int(it["offset"])
        flip = bool(int(it["flags"]) & ops.RAGGED_FLIP_X)
        if (h, w) == tuple(x.shape[-2:]) and not flip:
            v = x[n, 0]
        else:
            v = _OPS.resize_bilinear(x[n:n + 1].contiguous(), h, w, [float(it["scale"])], flip)[0, 0]
        out[o:o + h * w] = v.reshape(-1)
    return out


def disparity_to_image_ragged(disp, items, out, h_max, w_max):
    """picture i -> um_disparity_to_image of disparity i alone, at 3 * offset bytes"""
    flat = out.view(-1)
    for it in items_of(items):
        if _fits(it, h_max, w_max, 1, min(disp.numel(), out.numel() // 3)):
            h, w, o = int(it["h"]), int(it["w"]), int(it["offset"])
            pic = torch.empty((1, h, w, 3), dtype=torch.uint8, device=disp.device)
            _OPS.disparity_to_image(disp.reshape(-1)[o:o + h * w].view(1, h, w).contiguous(), pic)
            flat[3 * o:3 * (o + h * w)] = pic.reshape(-1)


def composed_stereo_reference(model, call, pairs, batch, max_buckets, padding_factor=16, inference_size=None,
                              pred_bidir_disp=False, pred_right_disp=False, only=None):
    """{index: result} of `MixedSizeStereoRunner`'s steps over `pairs` (host uint8 (left, right) [h, w, 3]), recomputed from
    existing functions only: the steps formed by `_batches` with the same bucket rule, each filled with its last pair; the
    frames normalised on the host, each brought to the bucket size with `_resize`, concatenated; `_stereo_outputs` once per
    distinct original size in the step, on the whole step batch, each pair's result taken from the call for its own size;
    the pictures from `disparity_to_image`.  `only`: a set of indices; steps holding none of them are skipped."""
    from unimatch_b200.inference import _batches, _inference_size, _resize, _stereo_outputs, disparity_to_image
    from unimatch_b200.synthetic import IMAGENET_MEAN, IMAGENET_STD

    def bucket(s):
        return _inference_size(tuple(s[1][0].shape[:2]), padding_factor, inference_size)

    res = {}
    for step in _batches(list(enumerate(pairs)), batch, bucket, max_buckets):
        if only is not None and not any(i in only for i, _ in step):
            continue
        size = bucket(step[0])
        full = [step[min(i, len(step) - 1)] for i in range(batch)]
        views = []
        for side in range(2):
            planes = [refops_depth.normalize_frames(torch.as_tensor(p[side])[None], IMAGENET_MEAN, IMAGENET_STD).cuda()
                      for _, p in full]
            views.append(torch.cat([_resize(x, size) for x in planes]))
        for ori in sorted({tuple(p[0].shape[:2]) for _, p in step}):
            out = _stereo_outputs(model, views[0], views[1], ori, size, pred_bidir_disp, pred_right_disp, dict(call))
            for i, (index, p) in enumerate(step):
                if tuple(p[0].shape[:2]) == ori:
                    r = {k: v[i].cpu() for k, v in out.items()}
                    for k in list(r):
                        r[k.replace("disp", "vis")] = disparity_to_image(r[k].cuda()).cpu()
                    res[index] = r
    return res

