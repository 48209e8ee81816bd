"""Depth inference over posed sequences without a device: the synthetic posed sequence has a true match, the relative poses
(and inverses) the drivers and the runner's staging upload are the reference's numpy expression bit for bit, arguments are
validated, and the host logic of `infer_depth_sequence` (frames encoded once, consecutive pairs, resize, bidirectional depth)
matches pairwise `infer_depth` through the CPU statements of the ops."""
import numpy as np
import pytest
import torch

import refops
import refops_depth
from unimatch_b200.inference import DepthSequenceRunner, _relative_poses, infer_depth, infer_depth_sequence
from unimatch_b200.synthetic import IMAGENET_MEAN, IMAGENET_STD, synthetic_model, synthetic_posed_sequence, workload_call

_WL = "gmdepth-scale1-regrefine1"


def _ref_relative(p, bidir):
    """evaluate_depth.py:344-350, pair by pair, plus the inverses for the backward streams"""
    rel = [np.linalg.inv(p[t + 1].astype(np.float32)) @ p[t].astype(np.float32) for t in range(len(p) - 1)]
    return rel + [np.linalg.inv(r) for r in rel] if bidir else rel


def test_synthetic_posed_sequence_has_a_true_match():
    frames, K, poses = synthetic_posed_sequence(5, 24, 40, seed=3, plane_depth=2.0)
    again = synthetic_posed_sequence(5, 24, 40, seed=3, plane_depth=2.0)
    assert frames.dtype == torch.uint8 and tuple(frames.shape) == (5, 24, 40, 3) and torch.equal(frames, again[0])
    assert tuple(K.shape) == (3, 3) and poses.dtype == torch.float32 and tuple(poses.shape) == (5, 4, 4)
    for t, rel in enumerate(_ref_relative(poses.numpy(), False)):
        # a point on the plane at depth 2 moves by f * tx / z px from frame t to frame t + 1 (rotation-free camera)
        dx = K[0, 0].item() * rel[0, 3] / 2.0
        s = int(round(dx))
        assert abs(dx - s) < 1e-4 and np.allclose(rel[:3, :3], np.eye(3)) and abs(rel[1, 3]) == abs(rel[2, 3]) == 0
        a, b = frames[t], frames[t + 1]
        if s >= 0:
            assert torch.equal(b[:, s:], a[:, :40 - s])
        else:
            assert torch.equal(b[:, :40 + s], a[:, -s:])


@pytest.mark.parametrize("bidir", [False, True])
def test_relative_poses_are_the_reference_expression(bidir):
    p = np.random.default_rng(0).normal(size=(6, 4, 4)).astype(np.float64)
    p[:, 3] = (0, 0, 0, 1)
    got = _relative_poses([q.astype(np.float32) for q in p], bidir)
    ref = _ref_relative(p, bidir)
    assert got.dtype == np.float32 and got.shape == (len(ref), 4, 4)
    assert all(np.array_equal(g, r) for g, r in zip(got, ref))


@pytest.mark.parametrize("bidir", [False, True])
def test_runner_staging_uploads_reference_relative_poses(bidir):
    """The runner's host staging on CPU buffers: a step of 4 pairs continuing from the carried pose, and a short tail step
    padded with repeats of its last item (relative pose of the repeat = inv(p) @ p)."""
    B, h, w = 4, 6, 8
    r = object.__new__(DepthSequenceRunner)
    r.batch, r.bidir = B, bidir
    r.pin = [torch.empty((B, h, w, 3), dtype=torch.uint8) for _ in range(2)]
    r.dev_in = [torch.empty((B, h, w, 3), dtype=torch.uint8) for _ in range(2)]
    n = (2 if bidir else 1) * B
    r.pose_pin = [torch.empty((n, 4, 4)) for _ in range(2)]
    r.pose_dev = [torch.empty((n, 4, 4)) for _ in range(2)]
    frames, _, poses = synthetic_posed_sequence(7, h, w, seed=9)
    poses = poses.numpy() + np.random.default_rng(1).normal(scale=0.01, size=(7, 4, 4)).astype(np.float32)   # non-trivial
    r.prev_pose = poses[0]
    items = list(zip(frames.numpy(), poses))
    r._stage_host(0, items[1:5])
    r._stage_host(1, items[5:7])
    for slot, seq in ((0, poses[0:5]), (1, [poses[4], poses[5], poses[6], poses[6], poses[6]])):
        ref = _ref_relative(np.stack(seq), bidir)
        assert all(np.array_equal(r.pose_dev[slot][i].numpy(), ref[i]) for i in range(n)), slot
    assert torch.equal(r.dev_in[0], frames[1:5]) and torch.equal(r.dev_in[1], frames[[5, 6, 6, 6]])
    assert np.array_equal(r.prev_pose, poses[6])


def test_infer_depth_sequence_argument_errors():
    m, kw = synthetic_model(_WL, "cpu"), workload_call(_WL, drop=("task", "min_depth", "max_depth", "num_depth_candidates"))
    frames, K, poses = synthetic_posed_sequence(3, 32, 48)
    bad = [
        dict(frames=frames[:1], poses=poses[:1]),                                  # T < 2
        dict(poses=poses[:2]),                                                     # pose count != T
        dict(frames=frames.int()),                                                 # integer frames that are not uint8
        dict(frames=frames.permute(0, 3, 1, 2).contiguous()),                      # uint8 frames must be channel-last
        dict(frames=frames.float()),                                               # float frames must be planar
        dict(K=K[None]),                                                           # one [3,3] matrix
        dict(K=K.long()),
        dict(poses=poses[:, :3]),                                                  # [T,3,4]
        dict(poses=poses.long()),
        dict(task="flow"),
    ]
    for change in bad:
        a = dict(frames=frames, K=K, poses=poses, **kw)
        a.update(change)
        f, k, p = a.pop("frames"), a.pop("K"), a.pop("poses")
        with pytest.raises(ValueError):
            infer_depth_sequence(m, f, k, p, padding_factor=16, **a)
    with pytest.raises(ValueError):
        DepthSequenceRunner(m, (32, 48), 2, "cpu", K[None], **kw)
    with pytest.raises(ValueError):
        DepthSequenceRunner(m, (32, 48), 2, "cpu", K, task="stereo", **kw)
    with pytest.raises(ValueError):
        m.encode_frames(frames.permute(0, 3, 1, 2).float(), task="segmentation")
    with pytest.raises(ValueError):
        m.forward_encoded([None], [None], task="stereo", **kw)


@pytest.mark.parametrize("size,bidir", [(None, True), ((48, 80), False)])
def test_infer_depth_sequence_host_logic_cpu(size, bidir):
    refops.register_cpu_kernels()
    m, kw = synthetic_model(_WL, "cpu"), workload_call(_WL, drop=("task", "min_depth", "max_depth", "num_depth_candidates"))
    frames, K, poses = synthetic_posed_sequence(3, 40, 60, seed=7)
    got = infer_depth_sequence(m, frames, K, poses, padding_factor=16, inference_size=size, pred_bidir_depth=bidir, **kw)
    norm = refops_depth.normalize_frames(frames, IMAGENET_MEAN, IMAGENET_STD)
    rel = torch.from_numpy(np.stack(_ref_relative(poses.numpy(), False)))
    ref = infer_depth(m, norm[:-1], norm[1:], K[None].repeat(2, 1, 1), rel, padding_factor=16, inference_size=size,
                      pred_bidir_depth=bidir, **kw)
    assert set(got) == set(ref) == ({"depth", "depth_bwd"} if bidir else {"depth"})
    for k in ref:
        assert got[k].shape == ref[k].shape == (2, 40, 60)
        assert (got[k] - ref[k]).abs().max().item() <= 1e-4 * ref[k].abs().max().item(), k
