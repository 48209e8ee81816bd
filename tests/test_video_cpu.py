"""Video inference without a device: the oracle's flow visualisation against the reference's pictures (golden_vis.pt), and
the host logic of `infer_flow_video` (frames encoded once, consecutive pairs, portrait transpose, resize, bidirectional flow,
consistency check, swapped pairs) through the CPU statements of the ops, against the oracle's `infer_flow` pair by pair."""
import os

import numpy as np
import pytest
import torch

import cases
import refops_video
from cases import O
from oracle import flow_viz as OV
from unimatch_b200 import UniMatch
from unimatch_b200.inference import infer_flow_video
from unimatch_b200.synthetic import synthetic_video

GOLD_VIS = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_vis.pt"))


@pytest.mark.parametrize("name", sorted(GOLD_VIS))
def test_oracle_flow_to_image_matches_reference(name):
    g = GOLD_VIS[name]
    got = OV.flow_to_image_batch(g["flow"].numpy())
    assert np.array_equal(got, g["image"].numpy())


def test_flow_to_image_fixed_points():
    img = OV.flow_to_image(np.zeros((3, 4, 2), np.float32))
    assert (img == 255).all()                                               # zero flow is white
    f = np.ones((3, 4, 2), np.float32)
    f[0, 0] = (1e9, 0.0)
    img = OV.flow_to_image(f)
    assert (img[0, 0] == 0).all() and (img[1:] != 0).any()                  # unknown marker is black


def test_synthetic_video_is_seeded_uint8():
    a, b = synthetic_video(4, 20, 30, seed=3), synthetic_video(4, 20, 30, seed=3)
    assert a.dtype == torch.uint8 and tuple(a.shape) == (4, 20, 30, 3) and torch.equal(a, b)
    assert not torch.equal(a[0], a[1])


def _tiny_model():
    cfg, sd, _, call = cases.e2e_setup("e2e_gmflow_s1_bidir")
    m = UniMatch(**cfg["model"]).eval()
    m.load_state_dict(sd)
    kw = {k: v for k, v in call.items() if k != "pred_bidir_flow"}
    mk = {k: cfg["model"][k] for k in ("num_scales", "upsample_factor", "reg_refine")}
    return m, sd, kw, mk


@pytest.mark.parametrize("T,hw,size,bidir,bwd", [
    (5, (40, 56), None, False, False),                # landscape, resized to the next multiple of 16
    (3, (56, 40), None, False, False),                # portrait: transposed for the model
    (3, (40, 56), (48, 80), False, False),            # fixed inference size
    (3, (48, 64), None, True, False),                 # bidirectional + consistency check
    (3, (48, 64), None, False, True),                 # backward flow (pairs swapped)
])
def test_infer_flow_video_host_logic_cpu(T, hw, size, bidir, bwd):
    refops_video.register_cpu_kernels()
    m, sd, kw, mk = _tiny_model()
    frames = synthetic_video(T, *hw, seed=7)
    got = infer_flow_video(m, frames, padding_factor=16, inference_size=size, pred_bidir_flow=bidir, pred_bwd_flow=bwd,
                           fwd_bwd_consistency_check=bidir, **kw)

    def fwd_fn(a, b, bd):
        return O.forward(sd, a, b, pred_bidir_flow=bd, **mk, **kw)["flow_preds"][-1]

    planar = frames.permute(0, 3, 1, 2).float()
    a, b = (planar[1:], planar[:-1]) if bwd else (planar[:-1], planar[1:])
    keys = {"flow", "flow_bwd", "fwd_occ", "bwd_occ"} if bidir else {"flow"}
    assert set(got) == keys
    for t in range(T - 1):
        ref = O.infer_flow(fwd_fn, a[t:t + 1], b[t:t + 1], 16, inference_size=size, pred_bidir_flow=bidir,
                           fwd_bwd_consistency_check=bidir)
        for k in ("flow", "flow_bwd") if bidir else ("flow",):
            assert got[k].shape == (T - 1, 2, *hw)
            r = ref[k][0]
            assert (got[k][t] - r).abs().max().item() <= 2e-3 * max(r.abs().max().item(), 1.0), (k, t)
        if bidir:
            for k in ("fwd_occ", "bwd_occ"):
                assert (got[k][t] != ref[k][0]).float().mean().item() < 0.02, (k, t)


def test_infer_flow_video_argument_errors():
    refops_video.register_cpu_kernels()
    m, _, kw, _ = _tiny_model()
    frames = synthetic_video(3, 32, 48)
    with pytest.raises(ValueError):
        infer_flow_video(m, frames[:1], padding_factor=16, **kw)
    with pytest.raises(ValueError):
        infer_flow_video(m, frames, padding_factor=16, fwd_bwd_consistency_check=True, **kw)
    with pytest.raises(ValueError):
        infer_flow_video(m, frames, padding_factor=16, **dict(kw, task="stereo"))
