"""Stereo scene flow on the device: `um_warp_disparity` and `um_scene_flow_stats` against the numpy statement
(tests/refops_sceneflow.py); `infer_scene_flow` against the stereo and flow paths it is built from; `SceneFlowRunner`
against `infer_scene_flow`, across graph replay and against its own pictures; `validate_scene_flow` and
`create_scene_flow_submission` against the statement and the submission oracle applied to `infer_scene_flow`'s outputs.

The kernels are compared bit for bit (warp) and count for count (statistics): both evaluate the statement's fp32
expressions in the header's order, which numpy float32 evaluates correctly rounded as well."""
import os

import numpy as np
import pytest
import torch

import refops_sceneflow as R
from oracle import submission_io as S
from unimatch_b200 import ops
from unimatch_b200.evaluation import scene_flow_results, validate_scene_flow
from unimatch_b200.inference import (SceneFlowRunner, _flow_outputs, _frame_geometry, _frames_to_model, _stereo_from_frames,
                                     disparity_to_image, flow_to_image, infer_scene_flow, warp_disparity)
from unimatch_b200.submission import create_scene_flow_submission
from unimatch_b200.synthetic import synthetic_model, synthetic_stereo_video, workload_call

pytestmark = pytest.mark.gpu
_OPS = torch.ops.unimatch_sm100
_STEREO, _FLOW = "gmstereo-scale2", "gmflow-scale2"
SIZES = [(48, 160), (37, 301)]                           # 37 x 301: neither a multiple of 32 nor of the 256-thread block


@pytest.fixture(scope="module")
def models():
    return synthetic_model(_STEREO), synthetic_model(_FLOW)


def _kw():
    """the scale-2 networks' windows need the inference size at a multiple of 32"""
    return dict(stereo_kwargs=workload_call(_STEREO), flow_kwargs=workload_call(_FLOW), stereo_padding_factor=32,
                flow_padding_factor=32)


# ---- um_warp_disparity --------------------------------------------------------------------------------------------------
def _warp_inputs(b, h, w, seed):
    g = np.random.default_rng(seed)
    ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    disp = (20 + 10 * np.sin(xs / 7.0) + 5 * np.cos(ys / 5.0) + g.standard_normal((b, h, w))).astype(np.float32)
    flow = (g.standard_normal((b, 2, h, w)) * 6).astype(np.float32)
    flow[:, 0, :, :3] -= 10.0                            # leaves on the left
    flow[:, 1, -3:] += 10.0                              # leaves at the bottom
    flow[0, 0, 0, 0], flow[0, 1, 1, 1] = np.nan, np.nan
    flow[1 % b, :, 2, 2] = np.inf
    flow[0, 0, 3, :] = (w - 1) - np.arange(w)            # lands exactly on the last column
    flow[0, 1, 3, :] = 0.0
    flow[0, 0, 4, :] = -np.arange(w)                     # exactly on the first column
    flow[0, 1, 4, :] = 0.0
    return disp, flow


@pytest.mark.parametrize("b,h,w", [(3, 37, 301), (2, 64, 128), (1, 1, 5)])
def test_warp_disparity_matches_statement(b, h, w):
    if h < 5:
        disp = np.arange(b * h * w, dtype=np.float32).reshape(b, h, w)
        flow = np.zeros((b, 2, h, w), np.float32)
        flow[:, 0] = [[-1.5, 0.25, 9.0, np.nan, 1.0]]
    else:
        disp, flow = _warp_inputs(b, h, w, seed=h + w)
    out = warp_disparity(torch.from_numpy(disp).cuda(), torch.from_numpy(flow).cuda())
    d1, inside = out["disp_1"].cpu().numpy(), out["in_frame"].cpu().numpy()
    emu, emu_in = R.warp_disparity(disp, flow, np.float32)
    assert np.array_equal(d1, emu) and np.array_equal(inside.astype(bool), emu_in)
    ref, _ = R.warp_disparity(disp, flow)
    # fp32: the coordinate x + u rounds by half an ulp of |q| <= w + max|u|, moved along a slope of at most the largest
    # neighbour difference; the bilinear's six roundings add a few ulps of max|disp|
    lip = max(np.abs(np.diff(disp, axis=1)).max(initial=0), np.abs(np.diff(disp, axis=2)).max(initial=0))
    tol = 2.0 ** -23 * (w + h) * lip * 2 + 8 * 2.0 ** -24 * np.abs(disp).max()
    assert np.abs(d1 - ref).max() <= tol
    if h >= 5:
        assert inside[0, 3].all() and inside[0, 4].all() and not inside[0, 0, 0] and not inside[0, 1, 1]


# ---- um_scene_flow_stats -----------------------------------------------------------------------------------------------
def _stats_inputs(b, h, w, seed):
    g = np.random.default_rng(seed)

    def near(x):                                         # errors on both sides of 3 px and 5 %
        kind = g.integers(0, 5, x.shape)
        size = np.choose(kind, [np.full(x.shape, 2.9), np.full(x.shape, 3.0), np.full(x.shape, 3.1), 0.05 * np.abs(x),
                                np.full(x.shape, 6.0)])
        return (x + g.choice([0, 1, -1], x.shape) * size * (g.random(x.shape) < 0.7)).astype(np.float32)
    gt = {}
    for key in ("occ", "noc"):
        d0 = (g.random((b, h, w)) * 80).astype(np.float32)
        d0[g.random((b, h, w)) < 0.2] = 0
        d1 = (g.random((b, h, w)) * 80).astype(np.float32)
        d1[g.random((b, h, w)) < 0.2] = 0
        f = (g.standard_normal((b, 2, h, w)) * 30).astype(np.float32)
        v = (g.random((b, h, w)) < 0.8).astype(np.float32)
        gt[key] = {"disp0": d0, "disp1": d1, "flow": f, "flow_valid": v}
    occ = gt["occ"]
    pred = (near(occ["disp0"]), near(occ["disp1"]), near(occ["flow"]))
    obj = (g.random((b, h, w)) < 0.3).astype(np.float32) * g.choice([1.0, 2.0, -1.0], (b, h, w)).astype(np.float32)
    return pred, gt, obj


@pytest.mark.parametrize("with_noc,with_obj", [(False, False), (True, False), (True, True), (False, True)])
def test_scene_flow_stats_count_for_count(with_noc, with_obj):
    b, h, w = 3, 37, 301
    pred, gt, obj = _stats_inputs(b, h, w, seed=7 + 2 * with_noc + with_obj)
    cuda = [torch.from_numpy(x).cuda() for x in pred]
    occ = [torch.from_numpy(gt["occ"][k]).cuda() for k in ("disp0", "disp1", "flow", "flow_valid")]
    noc = [torch.from_numpy(gt["noc"][k]).cuda() if with_noc else None for k in ("disp0", "disp1", "flow", "flow_valid")]
    table = _OPS.scene_flow_stats(*cuda, *occ, *noc, torch.from_numpy(obj).cuda() if with_obj else None).cpu().numpy()
    ref = R.scene_flow_counts(*pred, gt["occ"], gt["noc"] if with_noc else None, obj if with_obj else None)
    assert np.array_equal(table, ref.astype(np.float64))
    assert ref[:, [R.sf_col(0, 0, m, 1) for m in range(4)]].min() > 0       # every outlier kind occurs
    again = _OPS.scene_flow_stats(*cuda, *occ, *noc, torch.from_numpy(obj).cuda() if with_obj else None)
    assert torch.equal(again.cpu(), torch.from_numpy(table))


# ---- infer_scene_flow -------------------------------------------------------------------------------------------------
def _quadruples(T, h, w, seed):
    left, right = synthetic_stereo_video(T, h, w, seed=seed)
    return left.cuda(), right.cuda()


@pytest.mark.parametrize("h,w", SIZES)
def test_infer_scene_flow_is_its_parts(models, h, w):
    sm, fm = models
    left, right = _quadruples(4, h, w, seed=h)
    l0, r0, l1, r1 = left[:-1], right[:-1], left[1:], right[1:]
    out = infer_scene_flow(sm, fm, l0, r0, l1, r1, **_kw())
    b = l0.shape[0]
    disp = _stereo_from_frames(sm, torch.cat((l0, l1, r0, r1)), padding_factor=32, **workload_call(_STEREO))["disp"]
    assert torch.equal(out["disp_0"], disp[:b])
    transposed, ori, size = _frame_geometry(h, w, 32, None, "flow")
    planes = _frames_to_model(torch.cat((l0, l1)), "flow", transposed, size)
    flow = fm(planes[:b], planes[b:], **workload_call(_FLOW))["flow_preds"][-1]
    flow = _flow_outputs(flow, ori, size, transposed, False, False)["flow"]
    assert torch.equal(out["flow"], flow)
    warped = warp_disparity(disp[b:], flow)
    assert torch.equal(out["disp_1"], warped["disp_1"]) and torch.equal(out["in_frame"], warped["in_frame"])
    assert out["disp_0"].shape == (b, h, w) and out["flow"].shape == (b, 2, h, w) and out["in_frame"].dtype == torch.uint8


# ---- SceneFlowRunner --------------------------------------------------------------------------------------------------
def _run(runner, left, right):
    return [{k: v.clone() for k, v in r.items()} for r in runner.run(list(zip(left, right)))]


def test_runner_matches_quadruples_and_graph_replay(models):
    """7 frames at batch 3: two full steps and a short one; pairs 3 and 6 take their disp_0 and flow pyramid from the
    previous step's carry.  Against `infer_scene_flow` on the 6 consecutive quadruples the
    runner differs only by the batch composition: its stereo runs 3 pairs per step (and the first frame alone), its flow
    encoder the new frames of a step, so convolution and encoder sums run in another order; 1e-5 of the largest value is
    the encoder summation-order tolerance the video runners use."""
    sm, fm = models
    h, w = SIZES[1]
    left, right = synthetic_stereo_video(7, h, w, seed=5)
    ref = infer_scene_flow(sm, fm, left[:-1].cuda(), right[:-1].cuda(), left[1:].cuda(), right[1:].cuda(), **_kw())
    kw = _kw()                                           # the runner takes infer_scene_flow's keywords
    eager = _run(SceneFlowRunner(sm, fm, (h, w), 3, "cuda", use_graph=False, **kw), left, right)
    graph_runner = SceneFlowRunner(sm, fm, (h, w), 3, "cuda", visualize=True, **kw)
    graphed = _run(graph_runner, left, right)
    again = _run(graph_runner, left, right)              # a second run restarts from its own first frame
    assert len(eager) == len(graphed) == len(again) == 6
    for t in range(6):
        for k in ("disp_0", "flow"):
            r = ref[k][t].cpu()
            assert torch.allclose(eager[t][k], r, rtol=0, atol=1e-5 * r.abs().max().item()), (t, k)
        # disp_1 samples frame t+1's disparity where the flow points: the flows' difference moves the sample along the
        # disparity's slope (at most its largest neighbour difference L per pixel)
        nxt = ref["disp_1"][t].cpu()
        d_next = ref["disp_0"][t + 1].cpu() if t < 5 else eager[t]["disp_1"]
        lip = max(d_next.diff(dim=0).abs().max().item(), d_next.diff(dim=1).abs().max().item())
        dflow = (eager[t]["flow"] - ref["flow"][t].cpu()).abs().max().item()
        assert (eager[t]["disp_1"] - nxt).abs().max().item() <= 1e-5 * nxt.abs().max().item() + 2 * lip * dflow, t
        if t < 5:                                        # the warp of the runner's own disparity of frame t+1
            own = warp_disparity(eager[t + 1]["disp_0"][None].cuda(), eager[t]["flow"][None].cuda())["disp_1"][0].cpu()
            assert torch.equal(eager[t]["disp_1"], own), t
        # in_frame thresholds x + u at the frame edge: equal wherever the flows agree that far from the edge
        assert (eager[t]["in_frame"] != ref["in_frame"][t].cpu()).float().mean() < 1e-3
        for k in ("disp_0", "disp_1", "flow", "in_frame"):
            assert torch.equal(graphed[t][k], eager[t][k]), (t, k)
            assert torch.equal(again[t][k], graphed[t][k]), (t, k)
        assert torch.equal(graphed[t]["vis_disp_0"], disparity_to_image(graphed[t]["disp_0"].cuda()).cpu())
        assert torch.equal(graphed[t]["vis_disp_1"], disparity_to_image(graphed[t]["disp_1"].cuda()).cpu())
        assert torch.equal(graphed[t]["vis_flow"], flow_to_image(graphed[t]["flow"][None].cuda())[0].cpu())


# ---- validate_scene_flow and the submission ----------------------------------------------------------------------------
def _dataset(models, n=5, seed=11):
    """n samples alternating between the two SIZES, their predictions by `infer_scene_flow` at the batch composition
    `validate_scene_flow(batch=2)` forms (sizes interleaved: batches [0, 2], [1, 3], [4]), and ground truth around them"""
    sm, fm = models
    g = np.random.default_rng(seed)
    samples = []
    for i in range(n):
        h, w = SIZES[i % 2]
        left, right = synthetic_stereo_video(2, h, w, seed=seed + i)
        samples.append({"left0": left[0], "right0": right[0], "left1": left[1], "right1": right[1]})
    preds = {}
    for group in ([0, 2], [1, 3], [4]):
        v = [torch.stack([samples[i][k] for i in group]).cuda() for k in ("left0", "right0", "left1", "right1")]
        out = infer_scene_flow(sm, fm, *v, **_kw())
        for j, i in enumerate(group):
            preds[i] = {k: out[k][j].cpu().numpy() for k in ("disp_0", "disp_1", "flow")}
    for i, s in enumerate(samples):
        p = preds[i]
        h, w = p["disp_0"].shape

        def around(x):
            return (x + g.choice([0.0, 2.0, 5.0, -8.0], x.shape)).astype(np.float32)
        for suffix in ("", "_noc"):
            s["disp0" + suffix] = torch.from_numpy(np.maximum(around(p["disp_0"]), 0) * (g.random((h, w)) < 0.9))
            s["disp1" + suffix] = torch.from_numpy(np.maximum(around(p["disp_1"]), 0) * (g.random((h, w)) < 0.9))
            s["flow" + suffix] = torch.from_numpy(around(p["flow"]))
        s["flow_valid"] = torch.from_numpy((g.random((h, w)) < 0.9).astype(np.float32))
        s["flow_noc_valid"] = s["flow_valid"] * torch.from_numpy((g.random((h, w)) < 0.8).astype(np.float32))
        s["obj_map"] = torch.from_numpy((g.random((h, w)) < 0.3).astype(np.uint8))
    return samples, preds


def test_validate_scene_flow_counts(models):
    samples, preds = _dataset(models)
    res = validate_scene_flow(*models, samples, batch=2, **_kw())
    counts = np.zeros(R.SF_COLS, np.int64)
    for i, s in enumerate(samples):
        occ = {k: s[k].numpy()[None] for k in ("disp0", "disp1", "flow", "flow_valid")}
        noc = {k: s[k + ("_noc" if k != "flow_valid" else "")].numpy()[None] for k in ("disp0", "disp1", "flow")}
        noc["flow_valid"] = s["flow_noc_valid"].numpy()[None]
        p = preds[i]
        counts += R.scene_flow_counts(p["disp_0"][None], p["disp_1"][None], p["flow"][None], occ, noc,
                                      s["obj_map"].numpy()[None])[0]
    expect = scene_flow_results(counts.astype(np.float64), noc=True)
    assert res.keys() == expect.keys() and len(res) == 24
    for k in expect:
        assert res[k] == expect[k] or (np.isnan(res[k]) and np.isnan(expect[k])), k
    print({k: round(v, 3) for k, v in res.items() if k.endswith("_all")})
    plain = [{k: v for k, v in s.items() if not k.endswith("noc") and k != "flow_noc_valid" and k != "obj_map"}
             for s in samples]
    res2 = validate_scene_flow(*models, plain, batch=2, **_kw())
    assert len(res2) == 12 and np.isnan(res2["kitti_sf_occ_sf_fg"])
    # obj_map without the noc maps
    obj_only = [dict(p, obj_map=s["obj_map"]) for p, s in zip(plain, samples)]
    res3 = validate_scene_flow(*models, obj_only, batch=2, **_kw())
    counts = np.zeros(R.SF_COLS, np.int64)
    for i, s in enumerate(samples):
        occ = {k: s[k].numpy()[None] for k in ("disp0", "disp1", "flow", "flow_valid")}
        p = preds[i]
        counts += R.scene_flow_counts(p["disp_0"][None], p["disp_1"][None], p["flow"][None], occ, None,
                                      s["obj_map"].numpy()[None])[0]
    expect = scene_flow_results(counts.astype(np.float64), noc=False)
    assert res3.keys() == expect.keys() and len(res3) == 12
    for k in expect:
        assert res3[k] == expect[k] or (np.isnan(res3[k]) and np.isnan(expect[k])), k
    assert not np.isnan(res3["kitti_sf_occ_d1_fg"])
    for k in res3:                                       # bg + fg = all: the obj_map split the occ set's pixels
        if k.startswith("kitti_sf_occ"):
            assert res3[k] == res[k] or (np.isnan(res3[k]) and np.isnan(res[k])), k


def _read(path):
    with open(path, "rb") as f:
        return f.read()


def test_submission_files(models, tmp_path):
    samples, preds = _dataset(models, seed=23)
    samples[3]["name"] = "000042_10"
    stats = create_scene_flow_submission(*models, samples, output_path=str(tmp_path), batch=2, writers=3, **_kw())
    assert stats["samples"] == 5 and stats["batches"] == 3
    names = ["%06d_10" % i for i in range(5)]
    names[3] = "000042_10"
    for d in ("disp_0", "disp_1", "flow"):
        assert sorted(os.listdir(tmp_path / d)) == sorted(n + ".png" for n in names)
    for i, name in enumerate(names):
        p = preds[i]
        assert np.array_equal(S.decode_png(_read(tmp_path / "disp_0" / (name + ".png"))), S.kitti_disp_pixels(p["disp_0"]))
        assert np.array_equal(S.decode_png(_read(tmp_path / "disp_1" / (name + ".png"))), S.kitti_disp_pixels(p["disp_1"]))
        assert np.array_equal(S.decode_png(_read(tmp_path / "flow" / (name + ".png"))), S.kitti_flow_pixels(p["flow"]))
