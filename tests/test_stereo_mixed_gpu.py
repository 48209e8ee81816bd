"""Mixed-size stereo streaming on the device: each ragged kernel against the per-image kernel on mixed odd sizes, bit for bit,
and `MixedSizeStereoRunner` against the same steps recomputed from existing functions only.

The composed reference of a step: its pairs (the short step filled with its last pair) normalised on the host, each frame
brought to the bucket size with `_resize`, concatenated; `_stereo_outputs` called once per distinct original size in the
step on the whole step batch, each pair's result taken from the call for its own size; the pictures from
`disparity_to_image`.  The forward is deterministic for a shape (the tile-to-CTA assignment depends on the shape only), so
the repeated forwards agree with the runner's, and everything else is the per-image device code the ragged kernels share."""
import numpy as np
import pytest
import torch

import refops_depth
import refops_ragged
from oracle import disp_viz as OD
from unimatch_b200 import MixedSizeStereoRunner, ops
from unimatch_b200.inference import disparity_to_image
from unimatch_b200.synthetic import (IMAGENET_MEAN, IMAGENET_STD, synthetic_batch, synthetic_model, synthetic_stereo_frames,
                                     workload_call)

pytestmark = pytest.mark.gpu
_OPS = torch.ops.unimatch_sm100
FLIP = ops.RAGGED_FLIP_X


def _packed(sizes):
    offsets, off = [], 0
    for h, w in sizes:
        offsets.append(off)
        off += h * w
    return offsets, off


def test_frames_to_planar_normalized_ragged_equals_per_frame():
    """down- and upsampled frames and one at the output size (exactly its normalised samples)"""
    sizes = [(37, 53), (19, 23), (40, 56), (61, 77), (40, 31)]
    g = torch.Generator().manual_seed(3)
    frames = [torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8) for h, w in sizes]
    offsets, total = _packed(sizes)
    packed = torch.cat([f.reshape(-1) for f in frames]).cuda()
    items = refops_ragged.table([(3 * o, h, w, 1.0, 0) for o, (h, w) in zip(offsets, sizes)], "cuda")
    mean, std = list(IMAGENET_MEAN), list(IMAGENET_STD)
    out = _OPS.frames_to_planar_normalized_ragged(packed, items, 64, 80, 40, 56, mean, std)
    ref = refops_ragged.frames_to_planar_normalized_ragged(packed, items, 64, 80, 40, 56, mean, std)
    assert torch.equal(out, ref)
    exact = refops_depth.normalize_frames(frames[2][None], IMAGENET_MEAN, IMAGENET_STD)[0]
    assert torch.equal(out[2].cpu(), exact)
    for i, f in enumerate(frames):
        one = _OPS.frames_to_planar_normalized(f[None].cuda().contiguous(), 40, 56, mean, std)
        assert torch.equal(out[i], one[0]), i


def test_resize_bilinear_ragged_equals_per_image():
    """scaled, flipped, up- and downsampled items, and items at the input size with and without the flip; a non-finite
    value passes through untouched where the item is copied"""
    n, h, w = 6, 24, 40
    g = torch.Generator().manual_seed(7)
    x = torch.randn((n, 1, h, w), generator=g) * 30
    x[2, 0, 5, 6] = float("inf")
    x[3, 0, 7, 8] = float("nan")
    x = x.cuda()
    sizes = [(37, 53), (17, 29), (24, 40), (24, 40), (51, 77), (13, 40)]
    flags = [0, FLIP, 0, FLIP, FLIP, 0]
    scales = [np.float32(53 / float(w)), np.float32(29 / float(w)), 1.0, 1.0, np.float32(77 / float(w)), 1.0]
    offsets, total = _packed(sizes)
    items = refops_ragged.table([(o, hh, ww, s, f) for o, (hh, ww), s, f in zip(offsets, sizes, scales, flags)], "cuda")
    out = _OPS.resize_bilinear_ragged(x, items, 64, 80, total)
    ref = refops_ragged.resize_bilinear_ragged(x, items, 64, 80, total)
    assert torch.equal(out.isnan(), ref.isnan()) and torch.equal(out.nan_to_num(), ref.nan_to_num())
    assert torch.equal(out[offsets[2]:offsets[3]].view(h, w), x[2, 0])                     # copied, inf included
    for i, ((hh, ww), s, f) in enumerate(zip(sizes, scales, flags)):
        if i == 2:
            continue
        one = _OPS.resize_bilinear(x[i:i + 1].contiguous(), hh, ww, [float(s)], bool(f))[0, 0].reshape(-1)
        got = out[offsets[i]:offsets[i] + hh * ww]
        assert torch.equal(got.isnan(), one.isnan()) and torch.equal(got.nan_to_num(), one.nan_to_num()), i


def test_disparity_to_image_ragged_equals_per_image():
    """mixed odd sizes with a constant image, a NaN, +inf and -inf; the per-image scratch is reset inside every call"""
    sizes = [(37, 53), (1, 1), (29, 61), (40, 33), (17, 19), (23, 45)]
    g = torch.Generator().manual_seed(11)
    disps = [torch.rand((h, w), generator=g) * 180 - 3 for h, w in sizes]
    disps[2][:] = 42.5
    disps[3][10, 11] = float("nan")
    disps[4][3, 3] = float("inf")
    disps[5][0, 0] = float("-inf")
    offsets, total = _packed(sizes)
    packed = torch.cat([d.reshape(-1) for d in disps]).cuda()
    items = refops_ragged.table([(o, h, w, 1.0, 0) for o, (h, w) in zip(offsets, sizes)], "cuda")
    pics = torch.zeros((3 * total,), dtype=torch.uint8, device="cuda")
    for _ in range(2):
        _OPS.disparity_to_image_ragged(packed, items, pics, 48, 64)
    ref = torch.zeros_like(pics)
    refops_ragged.disparity_to_image_ragged(packed, items, ref, 48, 64)
    assert torch.equal(pics, ref)
    for i, ((h, w), d) in enumerate(zip(sizes, disps)):
        pic = pics[3 * offsets[i]:3 * (offsets[i] + h * w)].view(h, w, 3).cpu()
        assert torch.equal(pic, disparity_to_image(d.cuda()).cpu()), i
        assert np.array_equal(pic.numpy(), OD.vis_disparity(d.numpy())), i
    for i in (1, 2, 3, 4, 5):
        assert (pics[3 * offsets[i]:3 * (offsets[i] + sizes[i][0] * sizes[i][1])].view(-1, 3).cpu() ==
                torch.from_numpy(OD.INFERNO_BGR[0])).all(), i


# A KITTI-like interleaved mix (heights and widths a few pixels apart); with padding 32 they fall into the (128, 256) and
# (128, 224) buckets, and one pair is at (128, 256) itself, so its disparity is not resized back
MIX = [(120, 250), (100, 220), (128, 256), (118, 245), (100, 220), (121, 249), (120, 250)]
CAP = (128, 256)


def _pairs(sizes, seed):
    out = []
    for i, (h, w) in enumerate(sizes):
        left, right = synthetic_stereo_frames(1, h, w, seed=seed + i)
        out.append((left[0].numpy(), right[0].numpy()))
    return out


CASES = {                    # sizes, batch, max_buckets, runner arguments
    "inference_size": (MIX, 2, 4, dict(inference_size=(96, 192))),
    "buckets": (MIX, 2, 4, dict()),
    "bidir": (MIX, 2, 4, dict(pred_bidir_disp=True)),
    "right_only": (MIX, 2, 4, dict(pred_right_disp=True)),
    "eager": (MIX, 2, 4, dict(pred_bidir_disp=True, use_graph=False)),
    "short_tail": (MIX[:5], 3, 4, dict()),
    "max_buckets": (MIX + [(90, 150), (120, 250), (91, 151)], 2, 1, dict()),
    "pictures_only": (MIX, 2, 4, dict(pred_bidir_disp=True, return_disp=False)),
}


@pytest.mark.parametrize("workload", ["gmstereo-scale2", "gmstereo-scale2-regrefine3"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_mixed_runner_equals_composed_reference(workload, case):
    sizes, batch, max_buckets, kw = CASES[case]
    kw = dict(kw)
    m, call = synthetic_model(workload), workload_call(workload, drop=("task",))
    pairs = _pairs(sizes, seed=40)
    return_disp = kw.get("return_disp", True)
    runner = MixedSizeStereoRunner(m, CAP, batch, "cuda", padding_factor=32, visualize=True, max_buckets=max_buckets, **kw,
                                   **call)
    got = [(i, {k: v.clone() for k, v in r.items()}) for i, r in runner.run(pairs)]
    assert sorted(i for i, _ in got) == list(range(len(pairs)))                  # every index exactly once
    kw.pop("use_graph", None), kw.pop("return_disp", None)
    ref = refops_ragged.composed_stereo_reference(m, call, pairs, batch, max_buckets, padding_factor=32, **kw)
    bidir = kw.get("pred_bidir_disp", False)
    keys = {"disp", "vis"} | ({"disp_right", "vis_right"} if bidir else set())
    if not return_disp:
        keys = {k for k in keys if k.startswith("vis")}
    for i, r in got:
        assert set(r) == keys, (case, i)
        h, w = sizes[i]
        for k in keys:
            assert tuple(r[k].shape[:2]) == (h, w), (case, i, k)
            assert torch.equal(r[k], ref[i][k]), (case, i, k)
    assert runner.stats["pairs"] == len(pairs)
    if case == "max_buckets":
        assert runner.stats["captures"] > 2 and len(runner.buckets) == 1
    if case == "inference_size":
        assert runner.stats["captures"] == 1 and runner.stats["steps"] == 4


def test_mixed_runner_survives_other_shapes():
    """capture two buckets, evict the module's cached planes with forwards at other batch sizes and shapes, check that the
    runner still holds every buffer its graphs write, then replay bit for bit"""
    m, call = synthetic_model("gmstereo-scale2"), workload_call("gmstereo-scale2", drop=("task",))
    pairs = _pairs(MIX, seed=70)
    runner = MixedSizeStereoRunner(m, CAP, 2, "cuda", padding_factor=32, visualize=True, **call)
    r1 = {i: {k: v.clone() for k, v in r.items()} for i, r in runner.run(pairs)}
    assert len(runner.buckets) == 2
    captured = {t.data_ptr() for t in m.cached_buffers()}
    captured_keys = set(m._attn_ws) | set(m._pad_ws)
    assert captured
    for n, h, w in [(1, 384, 512), (3, 384, 512), (2, 320, 448), (1, 256, 384), (4, 256, 384)]:
        d = {k: v.cuda() for k, v in synthetic_batch("stereo", n, h, w).items()}
        m(d["img0"], d["img1"], **workload_call("gmstereo-scale2"))
    assert captured_keys - (set(m._attn_ws) | set(m._pad_ws)), "the runner's planes were not evicted: the scenario was not reached"
    held = {t.data_ptr() for _, _, bufs in runner.buckets.values() for t in bufs}
    assert captured <= held, "cached buffers the runner's graphs write are no longer referenced"
    r2 = {i: {k: v.clone() for k, v in r.items()} for i, r in runner.run(pairs)}
    assert runner.stats["captures"] == 2
    for i in r1:
        assert torch.equal(r1[i]["disp"], r2[i]["disp"]) and torch.equal(r1[i]["vis"], r2[i]["vis"]), i
