"""Depth inference over posed frame sequences on the device: the normalising frame-upload kernel against the resize kernel on
frames normalised as the reference pipeline does (bit for bit), `forward_encoded(task="depth")` against `forward` (bit for
bit), `infer_depth_sequence` against pairwise `infer_depth` on the same pairs and relative poses, and the streaming
`DepthSequenceRunner` (carried frame and pose across steps, short tail, eager and graph-replayed).

Sequence results are compared within 1e-4 of the largest depth, not bit for bit: um_conv2d_tc sums the K chunks of a tile in
an order rotated by the CTA that owns it, which depends on how many frames are encoded together (see UniMatch.encode_frames),
and with `pred_bidir_depth` the sequence drivers invert the relative poses on the host in numpy, where `forward` uses
torch.inverse on the device."""
import numpy as np
import pytest
import torch

import refops_depth
from unimatch_b200.inference import DepthSequenceRunner, infer_depth, infer_depth_sequence
from unimatch_b200.synthetic import (IMAGENET_MEAN, IMAGENET_STD, synthetic_batch, synthetic_model, synthetic_posed_sequence,
                                     workload_call)

pytestmark = pytest.mark.gpu
_OPS = torch.ops.unimatch_sm100
_DEPTH_RANGE = ("min_depth", "max_depth", "num_depth_candidates")


@pytest.mark.parametrize("hw,size", [((48, 80), (48, 80)), ((37, 53), (64, 96)), ((90, 120), (64, 96)), ((37, 53), (41, 67))])
def test_frames_to_planar_normalized_equals_resize(hw, size):
    frames = synthetic_posed_sequence(3, *hw, seed=5)[0]
    got = _OPS.frames_to_planar_normalized(frames.cuda(), size[0], size[1], list(IMAGENET_MEAN), list(IMAGENET_STD))
    norm = refops_depth.normalize_frames(frames, IMAGENET_MEAN, IMAGENET_STD)            # on the CPU, as the reference does
    ref = _OPS.resize_bilinear(norm.cuda().contiguous(), size[0], size[1], None, False)
    assert torch.equal(got, ref)
    if tuple(size) == tuple(hw):
        assert torch.equal(got.cpu(), norm)


@pytest.mark.parametrize("workload", ["gmdepth-scale1", "gmdepth-scale1-regrefine1"])
@pytest.mark.parametrize("bidir", [False, True])
def test_forward_encoded_depth_equals_forward(workload, bidir):
    m, call = synthetic_model(workload), workload_call(workload)
    d = {k: v.cuda() for k, v in synthetic_batch("depth", 2, 64, 96).items()}
    ref = m(d["img0"], d["img1"], intrinsics=d["intrinsics"], pose=d["pose"], pred_bidir_depth=bidir, **call)["flow_preds"]
    B = d["img0"].shape[0]
    feats = m.encode_frames(torch.cat((d["img0"], d["img1"]), 0), task="depth")
    cams = m.depth_cameras(d["intrinsics"], d["pose"], m.upsample_factor, call["min_depth"], call["max_depth"],
                           call["num_depth_candidates"], bidir)
    kw = {k: v for k, v in call.items() if k != "num_depth_candidates"}
    got = m.forward_encoded([f[:B] for f in feats], [f[B:] for f in feats], cameras=cams, pred_bidir_depth=bidir, **kw)["flow_preds"]
    assert len(got) == len(ref)
    for a, b in zip(got, ref):
        assert torch.equal(a, b)


def _close(got, ref, what, rel=1e-4):
    err = (got.float() - ref.float()).abs().max().item()
    assert err <= rel * ref.abs().max().item(), (what, err)


def _pairwise(m, kw, frames, K, poses, bidir, size=None):
    """`infer_depth` on the consecutive pairs of CPU-normalised frames, relative poses by the reference's expression"""
    norm = refops_depth.normalize_frames(frames, IMAGENET_MEAN, IMAGENET_STD).cuda()
    p = poses.numpy()
    rel = torch.from_numpy(np.stack([np.linalg.inv(p[t + 1]) @ p[t] for t in range(len(p) - 1)])).cuda()
    return infer_depth(m, norm[:-1], norm[1:], K.cuda()[None].repeat(len(p) - 1, 1, 1), rel, padding_factor=16,
                       inference_size=size, pred_bidir_depth=bidir, **kw)


@pytest.mark.parametrize("size,bidir", [(None, False), (None, True), ((112, 176), False), ((112, 176), True)])
def test_infer_depth_sequence_equals_pairwise(size, bidir):
    m, call = synthetic_model("gmdepth-scale1-regrefine1"), workload_call("gmdepth-scale1-regrefine1")
    kw = {k: v for k, v in call.items() if k not in _DEPTH_RANGE + ("task",)}
    frames, K, poses = synthetic_posed_sequence(7, 128, 192, seed=11)
    got = infer_depth_sequence(m, frames.cuda(), K, poses, padding_factor=16, inference_size=size, pred_bidir_depth=bidir, **kw)
    ref = _pairwise(m, kw, frames, K, poses, bidir, size)
    assert set(got) == set(ref) == ({"depth", "depth_bwd"} if bidir else {"depth"})
    for k in ref:
        assert got[k].shape == ref[k].shape == (6, 128, 192)
        _close(got[k], ref[k], k)


def test_depth_sequence_runner_eager_and_graph():
    """11 frames of 90x150 (inference size 96x160), batch 4: frame 0 primes the carried pyramid and pose, then three steps of
    4 / 4 / 2 (+2 repeats) new frames.  Graph replay and eager runs agree bit for bit."""
    m, call = synthetic_model("gmdepth-scale1-regrefine1"), workload_call("gmdepth-scale1-regrefine1")
    kw = {k: v for k, v in call.items() if k not in _DEPTH_RANGE + ("task",)}
    frames, K, poses = synthetic_posed_sequence(11, 90, 150, seed=21)
    ref = infer_depth_sequence(m, frames.cuda(), K, poses, pred_bidir_depth=True, **kw)
    runs = {}
    for use_graph in (False, True):
        runner = DepthSequenceRunner(m, (90, 150), 4, "cuda", K, use_graph=use_graph, pred_bidir_depth=True, **kw)
        runs[use_graph] = [{k: v.clone() for k, v in r.items()} for r in runner.run(zip(frames.numpy(), poses.numpy()))]
    for res in runs.values():
        assert len(res) == 10
        for t, r in enumerate(res):
            assert set(r) == {"depth", "depth_bwd"}
            _close(r["depth"], ref["depth"][t].cpu(), "depth %d" % t)
            _close(r["depth_bwd"], ref["depth_bwd"][t].cpu(), "depth_bwd %d" % t)
    for a, b in zip(runs[False], runs[True]):
        assert torch.equal(a["depth"], b["depth"]) and torch.equal(a["depth_bwd"], b["depth_bwd"])
