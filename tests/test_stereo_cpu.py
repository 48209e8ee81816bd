"""Stereo streaming without a device: the oracle's disparity visualisation against the reference's pictures
(golden_disp_vis.pt) and against the table compiled into the library, argument checks of `um_disparity_to_image`,
`disparity_to_image` and `StereoRunner`, and the host logic of `_stereo_from_frames` (the runner's step: uint8 frames
normalised and resized by one op, the hflip batching, the forward, the resize back) through the CPU statements of the ops,
against the oracle's `infer_stereo` on frames normalised on the host."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import refops
import refops_depth
from cases import O
from oracle import disp_viz as OD
from unimatch_b200 import UniMatch, ops
from unimatch_b200.inference import StereoRunner, _stereo_from_frames, disparity_to_image
from unimatch_b200.spec import WORKLOADS
from unimatch_b200.synthetic import (BENCH_WEIGHTS, IMAGENET_MEAN, IMAGENET_STD, synthetic_model, synthetic_state_dict,
                                     synthetic_stereo_frames, workload_call)

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = torch.load(os.path.join(HERE, "golden", "golden_disp_vis.pt"))


@pytest.mark.parametrize("name", sorted(GOLD))
def test_oracle_vis_disparity_matches_reference(name):
    g = GOLD[name]
    assert np.array_equal(OD.vis_disparity_batch(g["disp"].numpy()), g["image"].numpy())


def test_non_finite_images_take_colour_zero():
    for name in ("one_1x1", "constant", "nan_pos", "nan_neg", "inf_pos", "inf_neg"):
        img = GOLD[name]["image"].reshape(-1, 3)
        assert (img == torch.tensor([4, 0, 0], dtype=torch.uint8)).all(), name


def test_library_table_equals_oracle_table():
    src = open(os.path.join(os.path.dirname(HERE), "unimatch_b200", "csrc", "um_misc.cu")).read()
    body = re.search(r"kInferno\[768\]\s*=\s*\{(.*?)\};", src, flags=re.S).group(1)
    table = np.array([int(v) for v in body.replace(",", " ").split()], np.uint8).reshape(256, 3)
    assert np.array_equal(table, OD.INFERNO_BGR)


def test_disparity_to_image_bad_arguments_are_reported_without_a_gpu():
    one = ctypes.c_void_p(1024)
    good = dict(row=3 * 8, image=3 * 8 * 4, n=2, h=4, w=8)
    assert ops.LIB.um_disparity_to_image(None, one, 24, 96, one, 2, 4, 8, None) == -22
    assert b"um_disparity_to_image" in ops.LIB.um_last_error()
    for change in (dict(row=3 * 8 - 1), dict(image=3 * 8 * 4 - 1), dict(n=0), dict(h=0), dict(w=-1)):
        a = dict(good, **change)
        rc = ops.LIB.um_disparity_to_image(one, one, a["row"], a["image"], one, a["n"], a["h"], a["w"], None)
        assert rc == -22, change
        assert b"um_disparity_to_image" in ops.LIB.um_last_error(), change
    assert ops.LIB.um_disparity_to_image(one, one, 24, 96, None, 2, 4, 8, None) == -22          # no scratch


def test_disparity_to_image_shape_errors():
    refops.register_cpu_kernels()
    for bad in (torch.zeros(5), torch.zeros((1, 1, 4, 5)), torch.zeros((2, 0, 5)), torch.zeros((4, 5), dtype=torch.int32)):
        with pytest.raises(ValueError):
            disparity_to_image(bad)
    with pytest.raises(ValueError):
        disparity_to_image(torch.zeros((2, 4, 5)), torch.zeros((2, 4, 5, 3), dtype=torch.uint8)[:1])
    with pytest.raises(ValueError):
        disparity_to_image(torch.zeros((2, 4, 5)), torch.zeros((2, 4, 5, 3)))
    g = GOLD["odd_37x53"]                                        # the CPU statement, [N,H,W] and [H,W]
    assert torch.equal(disparity_to_image(g["disp"]), g["image"])
    assert torch.equal(disparity_to_image(g["disp"][1]), g["image"][1])


def test_synthetic_stereo_frames_is_seeded_uint8():
    (a, b), (c, d) = synthetic_stereo_frames(3, 20, 30, seed=3), synthetic_stereo_frames(3, 20, 30, seed=3)
    assert a.dtype == b.dtype == torch.uint8 and tuple(a.shape) == tuple(b.shape) == (3, 20, 30, 3)
    assert torch.equal(a, c) and torch.equal(b, d)
    assert not torch.equal(a[0], a[1])
    assert not torch.equal(a, synthetic_stereo_frames(3, 20, 30, seed=4)[0])


def _stereo_setup():
    cfg = WORKLOADS["gmstereo-scale2"]
    sd = synthetic_state_dict(seed=326, **BENCH_WEIGHTS, **cfg["model"])
    mk = {k: cfg["model"][k] for k in ("num_scales", "upsample_factor", "reg_refine")}
    return synthetic_model("gmstereo-scale2", "cpu"), sd, mk, workload_call("gmstereo-scale2", drop=("task",))


@pytest.mark.parametrize("bidir,right,size", [(False, False, None), (False, False, (96, 160)), (True, False, None),
                                              (False, True, None)])
def test_stereo_from_frames_host_logic_cpu(bidir, right, size):
    """2 pairs of 100x150, resized to 128x160 (padding 32) or to the inference size, against the oracle's infer_stereo on
    the frames normalised on the host as the reference's data pipeline does"""
    refops.register_cpu_kernels()
    m, sd, mk, call = _stereo_setup()
    left, rightv = synthetic_stereo_frames(2, 100, 150, seed=9)
    got = _stereo_from_frames(m, torch.cat((left, rightv), 0), padding_factor=32, inference_size=size, pred_bidir_disp=bidir,
                              pred_right_disp=right, **call)
    nl, nr = (refops_depth.normalize_frames(f, IMAGENET_MEAN, IMAGENET_STD) for f in (left, rightv))
    ref = O.infer_stereo(lambda a, b: O.forward(sd, a, b, task="stereo", **mk, **call)["flow_preds"][-1], nl, nr, 32, size,
                         bidir, right)
    assert set(got) == set(ref) == ({"disp", "disp_right"} if bidir else {"disp"})
    for k in ref:
        assert tuple(got[k].shape) == tuple(ref[k].shape) == (2, 100, 150)
        err = (got[k] - ref[k]).abs()
        assert err.mean().item() <= 2e-2 and err.max().item() <= 2e-1, (k, err.mean().item(), err.max().item())


def test_stereo_runner_argument_errors():
    """rejected before any device work (the constructor would otherwise create a CUDA stream first)"""
    m = UniMatch(num_scales=2, upsample_factor=4).eval()
    for kw in (dict(pred_bidir_disp=True, pred_right_disp=True), dict(return_disp=False), dict(task="flow"), dict(batch=0),
               dict(batch=-2)):
        args = dict(dict(batch=2), **kw)
        with pytest.raises(ValueError):
            StereoRunner(m, (64, 96), args.pop("batch"), "cuda", **args)
