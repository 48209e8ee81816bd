"""Stereo streaming on the device: the disparity colouring kernel against the reference's pictures and the oracle (bit for
bit: there is no transcendental function in it), into strided pictures, and `StereoRunner` against `infer_stereo` on the
same pairs normalised on the host and uploaded as float.

The runner's disparities equal `infer_stereo`'s bit for bit: `um_frames_to_planar_normalized` is exactly the host
normalisation at equal size and bit-identical to the resize of the normalised frames otherwise, the reference side runs the
same batch of pairs (so every kernel sees the same shapes and sums in the same order), and everything after the input
conversion is the same code (`_stereo_outputs`)."""
import os

import numpy as np
import pytest
import torch

import refops_depth
from oracle import disp_viz as OD
from unimatch_b200 import UniMatch
from unimatch_b200.inference import StereoRunner, disparity_to_image, infer_stereo
from unimatch_b200.spec import WORKLOADS
from unimatch_b200.synthetic import (BENCH_WEIGHTS, IMAGENET_MEAN, IMAGENET_STD, synthetic_batch, synthetic_state_dict,
                                     synthetic_stereo_frames)

pytestmark = pytest.mark.gpu
GOLD = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_disp_vis.pt"))


def test_disparity_to_image_matches_reference_golden():
    for name, g in sorted(GOLD.items()):
        assert torch.equal(disparity_to_image(g["disp"].cuda()).cpu(), g["image"]), name


def test_disparity_to_image_full_size_batch():
    """16 x 544 x 960 (bench config3's batch) with a constant image and an image holding one NaN, against the oracle"""
    g = torch.Generator().manual_seed(31)
    coarse = torch.rand((16, 1, 17, 30), generator=g) * 190.0 - 5.0
    disp = torch.nn.functional.interpolate(coarse, size=(544, 960), mode="bilinear", align_corners=True)[:, 0]
    disp = (disp + torch.randn(disp.shape, generator=g)).float().contiguous()
    disp[3] = 42.5
    disp[7, 100, 200] = float("nan")
    dd = disp.cuda()
    out = disparity_to_image(dd)
    torch.cuda.synchronize()
    ref = OD.vis_disparity_batch(disp.numpy())
    assert np.array_equal(out.cpu().numpy(), ref)
    assert (ref[3] == OD.INFERNO_BGR[0]).all() and (ref[7] == OD.INFERNO_BGR[0]).all()
    for _ in range(3):
        disparity_to_image(dd, out)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(50):
        disparity_to_image(dd, out)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 50
    nbytes = dd.numel() * (4 + 4 + 3)                # disparity read by both passes, picture written once
    print("disparity_to_image 16x544x960 on %s: %.4f ms, %.1f MB moved, %.0f GB/s" % (torch.cuda.get_device_name(), ms,
                                                                                     nbytes / 1e6, nbytes / ms / 1e6))


def test_disparity_to_image_strided_output():
    disp = GOLD["odd_37x53"]["disp"].cuda()
    big = torch.zeros((2, 37, 2 * 53, 3), dtype=torch.uint8, device="cuda")
    disparity_to_image(disp, big[:, :, 53:])
    assert torch.equal(big[:, :, 53:].cpu(), GOLD["odd_37x53"]["image"]) and not big[:, :, :53].any()
    tall = torch.zeros((3, 40, 53, 3), dtype=torch.uint8, device="cuda")       # 2 images into 3 slots of 3 extra rows
    disparity_to_image(disp, tall[:2, :37])
    assert torch.equal(tall[:2, :37].cpu(), GOLD["odd_37x53"]["image"]) and not tall[:, 37:].any() and not tall[2].any()


def _model(workload):
    cfg = WORKLOADS[workload]
    m = UniMatch(**cfg["model"]).eval()
    m.load_state_dict(synthetic_state_dict(seed=326, **BENCH_WEIGHTS, **cfg["model"]))
    call = {k: v for k, v in cfg["call"].items() if k != "task"}
    return m.cuda(), call, cfg


def _reference(m, call, lefts, rights, batch, **kw):
    """infer_stereo on the runner's steps (short last step filled with its last pair), frames normalised on the host"""
    nl, nr = (refops_depth.normalize_frames(f, IMAGENET_MEAN, IMAGENET_STD) for f in (lefts, rights))
    res = []
    for s in range(0, len(nl), batch):
        idx = [min(i, len(nl) - 1) for i in range(s, s + batch)]
        out = infer_stereo(m, nl[idx].cuda(), nr[idx].cuda(), **kw, **call)
        res += [{k: v[i].cpu() for k, v in out.items()} for i in range(min(batch, len(nl) - s))]
    return res


CASES = {                      # frame size, pairs, batch, runner / infer_stereo arguments
    "resized": ((250, 370), 4, 2, dict(padding_factor=32)),
    "inference_size": ((256, 384), 4, 2, dict(padding_factor=32, inference_size=(192, 320))),
    "bidir": ((256, 384), 4, 2, dict(padding_factor=32, pred_bidir_disp=True)),
    "right_only": ((250, 370), 4, 2, dict(padding_factor=32, pred_right_disp=True)),
    "eager": ((256, 384), 4, 2, dict(padding_factor=32, pred_bidir_disp=True)),
    "short_tail": ((256, 384), 5, 2, dict(padding_factor=32)),
}


@pytest.mark.parametrize("workload", ["gmstereo-scale2", "gmstereo-scale2-regrefine3"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_stereo_runner_equals_infer_stereo(workload, case):
    (h, w), n, batch, kw = CASES[case]
    m, call, _ = _model(workload)
    lefts, rights = synthetic_stereo_frames(n, h, w, seed=13)
    runner = StereoRunner(m, (h, w), batch, "cuda", visualize=True, use_graph=case != "eager", **kw, **call)
    got = [{k: v.clone() for k, v in r.items()} for r in runner.run(zip(lefts.numpy(), rights.numpy()))]
    ref = _reference(m, call, lefts, rights, batch, **kw)
    bidir = kw.get("pred_bidir_disp", False)
    assert len(got) == len(ref) == n
    for i, (r, e) in enumerate(zip(got, ref)):
        assert set(r) == ({"disp", "disp_right", "vis", "vis_right"} if bidir else {"disp", "vis"})
        for k in e:
            assert tuple(r[k].shape) == (h, w)
            assert torch.equal(r[k], e[k]), (case, i, k, (r[k] - e[k]).abs().max().item())
            v = r[k.replace("disp", "vis")]
            assert torch.equal(v, disparity_to_image(r[k].cuda()).cpu()), (case, i, k)
            assert np.array_equal(v.numpy(), OD.vis_disparity(r[k].numpy())), (case, i, k)


def test_stereo_runner_pictures_only():
    m, call, _ = _model("gmstereo-scale2")
    lefts, rights = synthetic_stereo_frames(3, 256, 384, seed=5)
    runner = StereoRunner(m, (256, 384), 2, "cuda", padding_factor=32, pred_bidir_disp=True, visualize=True, return_disp=False,
                          **call)
    got = [{k: v.clone() for k, v in r.items()} for r in runner.run(zip(lefts, rights))]
    ref = _reference(m, call, lefts, rights, 2, padding_factor=32, pred_bidir_disp=True)
    assert len(got) == 3
    for r, e in zip(got, ref):
        assert set(r) == {"vis", "vis_right"}
        assert np.array_equal(r["vis"].numpy(), OD.vis_disparity(e["disp"].numpy()))
        assert np.array_equal(r["vis_right"].numpy(), OD.vis_disparity(e["disp_right"].numpy()))
    with pytest.raises(ValueError):                           # a pair of another size
        list(runner.run([(lefts[0, :128], rights[0, :128])]))


def test_stereo_runner_survives_other_shapes():
    """capture, evict the module's cached planes with forwards at other batch sizes and shapes, check that the runner still
    holds every buffer its graphs write, then replay bit for bit"""
    m, call, cfg = _model("gmstereo-scale2")
    lefts, rights = synthetic_stereo_frames(4, 384, 512, seed=3)
    runner = StereoRunner(m, (384, 512), 2, "cuda", **call)
    items = list(zip(lefts.numpy(), rights.numpy()))
    r1 = [{k: v.clone() for k, v in r.items()} for r in runner.run(items)]
    captured = {t.data_ptr() for t in m.cached_buffers()}
    captured_keys = set(m._attn_ws) | set(m._pad_ws)
    assert captured
    for n, h, w in [(1, 384, 512), (3, 384, 512), (2, 320, 448), (1, 256, 384), (4, 256, 384)]:
        d = {k: v.cuda() for k, v in synthetic_batch("stereo", n, h, w).items()}
        m(d["img0"], d["img1"], **cfg["call"])
    assert captured_keys - (set(m._attn_ws) | set(m._pad_ws)), "the runner's planes were not evicted: the scenario was not reached"
    held = {t.data_ptr() for t in runner._held_buffers}
    assert captured <= held, "cached buffers the runner's graphs write are no longer referenced"
    r2 = [{k: v.clone() for k, v in r.items()} for r in runner.run(items)]
    for a, b in zip(r1, r2):
        assert torch.equal(a["disp"], b["disp"])
