"""Video inference on the device: the colouring kernel against the reference's pictures, the frame-upload kernel against the
resize kernel (bit for bit), `infer_flow_video` against `infer_flow` on the same pairs, and the streaming `VideoFlowRunner`
(carried frame across steps, short tail, graph / eager, frame + flow pictures).

The flows are compared within 1e-4 of the largest flow component, not bit for bit: the encoder works per image, but
um_conv2d_tc sums the K chunks of a tile in an order rotated by the CTA that owns it, and which CTA owns a tile depends on the
launch's tile count, i.e. on how many frames are encoded together (see UniMatch.encode_frames)."""
import os

import numpy as np
import pytest
import torch

from oracle import flow_viz as OV
from unimatch_b200.inference import VideoFlowRunner, flow_to_image, infer_flow, infer_flow_video
from unimatch_b200.spec import WORKLOADS
from unimatch_b200.synthetic import synthetic_model, synthetic_video, workload_call

pytestmark = pytest.mark.gpu
GOLD_VIS = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_vis.pt"))
_OPS = torch.ops.unimatch_sm100


def _vis_close(got, ref, what):
    """every byte within 1 of the reference and at most 0.1 % of the bytes different (fp64 atan2 vs numpy's)"""
    d = (got.astype(np.int16) - ref.astype(np.int16))
    frac = float((d != 0).mean())
    print("%s: %.4f %% of bytes differ, max |diff| %d" % (what, 100 * frac, int(np.abs(d).max())))
    assert np.abs(d).max() <= 1 and frac <= 1e-3, (what, frac)


def test_flow_to_image_kernel_matches_reference_golden():
    for name, g in sorted(GOLD_VIS.items()):
        flow = g["flow"]
        got = flow_to_image(flow.cuda()).cpu().numpy()
        ref = g["image"].numpy()
        _vis_close(got, ref, name)
        u, v = flow[:, 0].numpy(), flow[:, 1].numpy()
        unknown = (np.abs(u) > 1e7) | (np.abs(v) > 1e7)
        zero = (u == 0) & (v == 0) & ~unknown
        rad = np.where(unknown, 0, np.sqrt(u * u + v * v))
        top = rad == rad.reshape(rad.shape[0], -1).max(1)[:, None, None]
        for mask, what in ((unknown, "unknown"), (zero, "zero"), (top & ~zero, "max radius")):
            assert np.array_equal(got[mask], ref[mask]), (name, what)


def test_flow_to_image_full_size_batch():
    g = torch.Generator().manual_seed(17)
    smooth = torch.randn((4, 2, 15, 26), generator=g) * 30
    flow = torch.nn.functional.interpolate(smooth, size=(480, 832), mode="bilinear", align_corners=True)
    flow = flow + torch.randn(flow.shape, generator=g)
    got = flow_to_image(flow.cuda())
    torch.cuda.synchronize()
    _vis_close(got.cpu().numpy(), OV.flow_to_image_batch(flow.numpy()), "480x832 x4")
    # HBM throughput of the two passes (flow read by both, picture written once)
    fd = flow.cuda()
    out = torch.empty((4, 480, 832, 3), dtype=torch.uint8, device="cuda")
    for _ in range(3):
        flow_to_image(fd, out)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20):
        flow_to_image(fd, out)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 20
    print("flow_to_image 4x480x832: %.3f ms, %.0f GB/s (flow once + picture)" % (ms, (fd.numel() * 4 + out.numel()) / ms / 1e6))


def test_flow_to_image_strided_output():
    flow = GOLD_VIS["odd_37x53"]["flow"].cuda()
    big = torch.zeros((4, 37, 2 * 53, 3), dtype=torch.uint8, device="cuda")
    flow_to_image(flow, big[:, :, 53:])
    assert torch.equal(big[:, :, 53:], flow_to_image(flow)) and not big[:, :, :53].any()


@pytest.mark.parametrize("hw,size,transpose", [((48, 80), (48, 80), False), ((37, 53), (64, 96), False),
                                               ((80, 48), (48, 80), True), ((90, 60), (64, 96), True)])
def test_frames_to_planar_equals_resize(hw, size, transpose):
    frames = synthetic_video(3, *hw, seed=5).cuda()
    got = _OPS.frames_to_planar(frames, size[0], size[1], transpose)
    x = frames.permute(0, 3, 1, 2).float()
    if transpose:
        x = x.transpose(-2, -1)
    ref = _OPS.resize_bilinear(x.contiguous(), size[0], size[1], None, False)
    assert torch.equal(got, ref)
    if tuple(size) == tuple(x.shape[-2:]):
        assert torch.equal(got, x)


def _close(got, ref, what, rel=1e-4):
    err = (got.float() - ref.float()).abs().max().item()
    assert err <= rel * max(1.0, ref.abs().max().item()), (what, err)


def test_encoder_is_per_frame():
    """a frame's pyramid does not depend on the batch it is encoded in (up to summation order); same batch: bit for bit"""
    m = synthetic_model("gmflow-scale2")
    frames = synthetic_video(5, 64, 96, seed=2).cuda().permute(0, 3, 1, 2).float().contiguous()
    full = m.encode_frames(frames)
    assert all(torch.equal(a, b) for a, b in zip(full, m.encode_frames(frames)))
    for t in (0, 3):
        alone = m.encode_frames(frames[t:t + 1])
        for a, f in zip(alone, full):
            _close(a[0], f[t], "frame %d" % t, rel=1e-5)


@pytest.mark.parametrize("workload,bidir,bwd", [("gmflow-scale1", False, False), ("gmflow-scale2-regrefine6", False, False),
                                                ("gmflow-scale1", True, False), ("gmflow-scale2-regrefine6", False, True)])
def test_infer_flow_video_equals_pairwise(workload, bidir, bwd):
    m, call = synthetic_model(workload), workload_call(workload, drop=("task",))
    pad = WORKLOADS[workload]["pad"]
    frames = synthetic_video(7, 128, 192, seed=11).cuda()
    got = infer_flow_video(m, frames, padding_factor=pad, pred_bidir_flow=bidir, pred_bwd_flow=bwd,
                           fwd_bwd_consistency_check=bidir, **call)
    planar = frames.permute(0, 3, 1, 2).float()
    a, b = (planar[1:], planar[:-1]) if bwd else (planar[:-1], planar[1:])
    ref = infer_flow(m, a, b, padding_factor=pad, pred_bidir_flow=bidir, fwd_bwd_consistency_check=bidir, **call)
    assert set(got) == set(ref)
    for k in ("flow", "flow_bwd"):
        if k in ref:
            assert got[k].shape == ref[k].shape
            _close(got[k], ref[k], k)
    for k in ("fwd_occ", "bwd_occ"):
        if k in ref:
            assert (got[k] != ref[k]).float().mean().item() < 0.01, k


def test_infer_flow_video_portrait_resized_equals_pairwise():
    m, call = synthetic_model("gmflow-scale1"), workload_call("gmflow-scale1", drop=("task",))
    pad = WORKLOADS["gmflow-scale1"]["pad"]
    frames = synthetic_video(4, 100, 70, seed=12).cuda()
    got = infer_flow_video(m, frames, padding_factor=pad, inference_size=(64, 112), **call)
    planar = frames.permute(0, 3, 1, 2).float()
    ref = infer_flow(m, planar[:-1], planar[1:], padding_factor=pad, inference_size=(64, 112), **call)
    assert got["flow"].shape == ref["flow"].shape == (3, 2, 100, 70)
    _close(got["flow"], ref["flow"], "flow")


@pytest.mark.parametrize("use_graph", [False, True])
def test_video_flow_runner_matches_infer_flow_video(use_graph):
    """11 frames, batch 4: frame 0 primes the carried pyramid, then three steps of 4 / 4 / 2 (+2 repeats) new frames."""
    m, call = synthetic_model("gmflow-scale1"), workload_call("gmflow-scale1", drop=("task",))
    pad = WORKLOADS["gmflow-scale1"]["pad"]
    frames = synthetic_video(11, 96, 160, seed=21)
    runner = VideoFlowRunner(m, (96, 160), 4, "cuda", padding_factor=pad, use_graph=use_graph, visualize=True,
                             pred_bidir_flow=True, **call)
    res = [{k: v.clone() for k, v in r.items()} for r in runner.run(f.numpy() for f in frames)]
    ref = infer_flow_video(m, frames.cuda(), padding_factor=pad, pred_bidir_flow=True, **call)
    assert len(res) == 10
    for t, r in enumerate(res):
        assert set(r) == {"flow", "flow_bwd", "vis"}
        _close(r["flow"], ref["flow"][t].cpu(), "flow %d" % t)
        _close(r["flow_bwd"], ref["flow_bwd"][t].cpu(), "flow_bwd %d" % t)
    flows = torch.stack([r["flow"] for r in res]).cuda()
    assert torch.equal(torch.stack([r["vis"] for r in res]), flow_to_image(flows).cpu())


@pytest.mark.parametrize("hw,return_flow", [((64, 96), True), ((96, 64), True), ((64, 96), False)])
def test_video_flow_runner_concat_layout(hw, return_flow):
    """concat_flow_img (evaluate_flow.py:818-825): frame above its picture when H < W, beside it otherwise."""
    m, call = synthetic_model("gmflow-scale1"), workload_call("gmflow-scale1", drop=("task",))
    pad = WORKLOADS["gmflow-scale1"]["pad"]
    h, w = hw
    frames = synthetic_video(6, h, w, seed=4)
    runner = VideoFlowRunner(m, hw, 4, "cuda", padding_factor=pad, visualize=True, concat_frame=True, return_flow=return_flow,
                             **call)
    res = [{k: v.clone() for k, v in r.items()} for r in runner.run(list(frames))]
    assert len(res) == 5
    axis = 0 if h < w else 1
    for t, r in enumerate(res):
        assert set(r) == ({"vis", "flow"} if return_flow else {"vis"})
        assert tuple(r["vis"].shape) == ((2 * h, w, 3) if axis == 0 else (h, 2 * w, 3))
        frame_half, pic_half = r["vis"].split(h if axis == 0 else w, dim=axis)
        assert torch.equal(frame_half, frames[t]), t
        if return_flow:
            assert torch.equal(pic_half, flow_to_image(r["flow"][None].cuda())[0].cpu()), t
