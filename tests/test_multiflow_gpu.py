"""Multi-flow dense point tracks on the device: `um_fb_consistency_error` and `um_multi_flow_tracks` against the statement
(tests/refops_multiflow.py), and `MultiFlowTrackRunner` against `multi_flow_tracks` on its own flows, across graph replay,
batch sizes and runs, and on `infer_flow`'s flows of the same pairs.

Tolerances.  Both kernels evaluate the statement's expression in fp32 in the order the header fixes, so they equal the
statement evaluated in numpy float32 bit for bit.  Against the float64 statement, each frame is evaluated from the kernel's
own states of its source frames: a candidate's position is within `refops_tracks.step_rounding` of the float64 one, and
its sigma2 within a few roundings of the largest sigma2 and e^2.  Where two candidates' sigma2 lie within that of each
other, or a candidate's validity test lies within rounding of a threshold (`refops_tracks.near_threshold`), the choice may
fall either way; such pixels are counted and bounded, and every other pixel must agree."""
import numpy as np
import pytest
import torch

import refops_multiflow as RM
import refops_tracks as RT
from test_multiflow_cpu import _occluder, _random_case, occluder_checks
from unimatch_b200.inference import (MultiFlowTrackRunner, chain_tracks, infer_flow, multi_flow_sources,
                                     multi_flow_tracks)
from unimatch_b200.spec import WORKLOADS
from unimatch_b200.synthetic import synthetic_model, synthetic_video, workload_call

_WL = "gmflow-scale1"

pytestmark = pytest.mark.gpu
_OPS = torch.ops.unimatch_sm100


@pytest.mark.parametrize("b,hw", [(3, (37, 53)), (2, (61, 40)), (1, (480, 832))])
def test_fb_consistency_error(b, hw):
    h, w = hw
    flows = RT.smooth_flows(2 * b, h, w, 5.0, seed=b + h, drift=(2.0, -1.0))
    fwd, bwd = flows[:b], -0.8 * flows[b:]
    fd, bd = torch.from_numpy(fwd).cuda(), torch.from_numpy(np.ascontiguousarray(bwd)).cuda()
    occ, bocc, err = _OPS.fb_consistency_error(fd, bd, 0.01, 0.5)
    ref_occ, ref_bocc = _OPS.fb_consistency(fd, bd, 0.01, 0.5)
    assert torch.equal(occ, ref_occ) and torch.equal(bocc, ref_bocc)
    o32, e32 = RM.fb_residual(fwd, bwd, dtype=np.float32)
    assert np.array_equal(err.cpu().numpy(), e32) and np.array_equal(occ.cpu().numpy(), o32)
    # float64: a few roundings of the largest flow, plus the sampling position's rounding through the normalise /
    # un-normalise of bilinear_sample (a few units in the last place of the frame size) times the backward flow's slope
    _, e64 = RM.fb_residual(fwd, bwd)
    scale = np.abs(fwd).max() + np.abs(bwd).max() + 1.0
    tol = 2.0 ** -24 * (64 * scale + 8 * max(h, w) * (1 + 2 * RT.lipschitz(bwd)))
    assert np.abs(err.cpu().numpy() - e64).max() <= tol
    assert 0 < o32.mean() < 1


def _kernel_in_steps(flows, occ, err, gaps, anchor, batch):
    """um_multi_flow_tracks over the clip in launches of `batch` frames, the states in a ring of max(gaps) + batch + 1
    slots (frame 0 in slot 0), as the runner keeps them"""
    n, k, _, h, w = flows.shape
    slots = max(gaps, default=0) + batch + 1
    ring = lambda f: 0 if f == 0 else 1 + (f - 1) % (slots - 1)
    pos = torch.empty((slots, h, w, 2), device="cuda")
    sig = torch.empty((slots, h, w), device="cuda")
    vis = torch.empty((slots, h, w), device="cuda", dtype=torch.uint8)
    pos[0] = torch.from_numpy(RT.track_start(h, w, np.float32)[0]).cuda()
    sig[0], vis[0] = 0, 1
    fd, od, ed = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (flows, occ, err))
    outs = []
    for t0 in range(1, n + 1, batch):
        ts = range(t0, min(t0 + batch, n + 1))
        src = torch.tensor([[ring(s) if s >= 0 else -1 for s in multi_flow_sources(t, gaps, anchor)] for t in ts],
                           dtype=torch.int32).cuda()
        dst = torch.tensor([ring(t) for t in ts], dtype=torch.int32).cuda()
        sl = slice(t0 - 1, t0 - 1 + len(ts))
        outs.append(_OPS.multi_flow_tracks(fd[sl], od[sl], ed[sl], src, dst, pos, sig, vis))
    return [torch.cat([o[i] for o in outs]).cpu().numpy() for i in range(3)]


def _check_float64(tracks, visible, sigma, flows, occ, err, gaps, anchor):
    """each frame from the kernel's own source states, against the float64 statement: agreement but for pixels where the
    choice is within rounding, which are counted and bounded"""
    n, k, _, h, w = flows.shape
    states = {t + 1: (tracks[t], sigma[t], visible[t].astype(bool)) for t in range(n)}
    ref = RM.multi_flow_tracks(flows, occ, err, gaps, anchor, states=states)
    eps = RT.step_rounding(ref["tracks"], flows.reshape(-1, 2, h, w))
    emax = float(np.nanmax(np.abs(err)))
    tol_s = 2.0 ** -20 * (float(np.nanmax(np.abs(sigma))) + emax * emax + 1.0)
    start = RT.track_start(h, w, np.float64)[0]
    unsure = np.zeros((n, h, w), bool)
    for t, cands in enumerate(ref["candidates"]):
        src = multi_flow_sources(t + 1, gaps, anchor)
        for j, x, s2, _ in cands:
            p = start if src[j] == 0 else states[src[j]][0].astype(np.float64)
            o = RT.bilinear(occ[t, j][None].astype(np.float64), p[..., 0], p[..., 1])[0]
            unsure[t] |= RT.near_threshold(x[None], o[None], h, w, eps, 2 * eps + 1e-6)[0]
            for j2, x2, s22, _ in cands:
                if j2 > j:
                    unsure[t] |= (np.abs(s2 - s22) <= tol_s) & (np.abs(x - x2).max(-1) > eps)
    agree = ((np.abs(tracks - ref["tracks"]).max(-1) <= eps) & (visible.astype(bool) == ref["visible"]) &
             (np.abs(sigma - ref["uncertainty"]) <= tol_s))
    bad = ~agree & ~unsure
    print("%dx%d n=%d gaps %s anchor %s: %d pixels within rounding of a choice, %d disagree outside them"
          % (h, w, n, gaps, anchor, int(unsure.sum()), int(bad.sum())))
    assert bad.sum() == 0 and unsure.mean() <= 0.01


@pytest.mark.parametrize("gaps,anchor,batch,n,hw", [((1, 2, 4), True, 2, 11, (37, 53)), ((1, 2, 4, 8), False, 3, 14, (29, 41)),
                                                     ((), True, 4, 6, (33, 31)), ((1, 3), True, 1, 9, (61, 40)),
                                                     ((1, 2, 4, 8, 16, 32), True, 4, 40, (24, 36))])
def test_kernel_matches_statement(gaps, anchor, batch, n, hw):
    """bit for bit against the float32 statement, in launches of `batch` frames over a state ring that wraps around
    (n > max(gaps) + batch), and the float64 statement within rounding"""
    h, w = hw
    flows, occ, err = _random_case(n, h, w, gaps, anchor, seed=n * 5 + h)
    tracks, visible, sigma = _kernel_in_steps(flows, occ, err, gaps, anchor, batch)
    emu = RM.multi_flow_tracks(flows, occ, err, gaps, anchor, dtype=np.float32)
    assert np.array_equal(tracks, emu["tracks"], equal_nan=True)
    assert np.array_equal(visible.astype(bool), emu["visible"])
    assert np.array_equal(sigma, emu["uncertainty"], equal_nan=True)
    assert visible.any() and not visible.all()
    whole = multi_flow_tracks(torch.from_numpy(flows).cuda(), torch.from_numpy(flows).cuda(), gaps, anchor)
    assert whole["tracks"].shape == (n, h, w, 2) and whole["visible"].dtype == torch.uint8
    _check_float64(tracks, visible, sigma, flows, occ, err, gaps, anchor)


def test_gap_one_is_chain_tracks_on_the_device():
    n, h, w = 7, 45, 67
    flows = RT.smooth_flows(n, h, w, 3.0, seed=3, drift=(1.5, -0.5))[:, None]
    bwd = -0.9 * flows
    fd, bd = torch.from_numpy(flows).cuda(), torch.from_numpy(np.ascontiguousarray(bwd)).cuda()
    got = multi_flow_tracks(fd, bd, gaps=(1,), anchor=False)
    occ, _ = _OPS.fb_consistency(fd[:, 0].contiguous(), bd[:, 0].contiguous(), 0.01, 0.5)
    ref = chain_tracks(fd[:, 0], occ)
    assert torch.equal(got["tracks"], ref["tracks"]) and torch.equal(got["visible"], ref["visible"])
    assert 0 < got["visible"].float().mean() < 1


@pytest.mark.parametrize("gaps,anchor", [((1, 2, 4, 8, 16, 32), True), ((1,), False)])
def test_occluder_clip_on_the_device(gaps, anchor):
    clip, fwd, bwd, occ, err = _occluder(gaps, anchor)
    got = multi_flow_tracks(torch.from_numpy(fwd).cuda(), torch.from_numpy(bwd).cuda(), gaps, anchor)
    tracks, visible = got["tracks"].cpu().numpy(), got["visible"].cpu().numpy()
    emu = RM.multi_flow_tracks(fwd, occ, err, gaps, anchor, dtype=np.float32)
    assert np.array_equal(tracks, emu["tracks"], equal_nan=True) and np.array_equal(visible.astype(bool), emu["visible"])
    if anchor:
        chain = RT.chain_tracks(fwd[:, 0], occ[:, 0], dtype=np.float32)
        occluder_checks(clip, tracks, visible, chain["visible"])
    else:
        pos, covered, _, background = clip.truth()
        passed = background & covered.any(axis=0)
        first = np.argmax(covered, axis=0)
        later = (np.arange(clip.frames)[:, None, None] >= first[None]) & passed[None]
        assert not visible.astype(bool)[later[1:]].any()


def _run(runner, frames):
    return [{k: v.clone() for k, v in r.items()} for r in runner.run(list(frames.numpy()))]


def _stack(res, key):
    return torch.stack([r[key] for r in res])


@pytest.mark.parametrize("batch,use_graph", [(1, True), (3, True), (3, False)])
def test_runner_equals_multi_flow_tracks_on_its_flows(batch, use_graph):
    """12 frames (11 new: steps of 1, or 3 / 3 / 3 / 2 + a repeat), gaps (1, 2, 4) and the anchor: ring of 4 + batch + 1
    slots, wrapped.  The runner's tracks are `multi_flow_tracks` on its own flows bit for bit, and a second run repeats
    the first"""
    m, call = synthetic_model(_WL), workload_call(_WL, drop=("task",))
    pad = WORKLOADS[_WL]["pad"]
    gaps = (1, 2, 4)
    frames = synthetic_video(12, 64, 96, seed=17)
    runner = MultiFlowTrackRunner(m, (64, 96), batch, "cuda", gaps=gaps, padding_factor=pad, use_graph=use_graph,
                                  return_flow=True, **call)
    res = _run(runner, frames)
    assert len(res) == 11
    assert all(set(r) == {"tracks", "visible", "uncertainty", "flow", "flow_bwd", "sources"} for r in res)
    assert [r["sources"].tolist() for r in res] == [multi_flow_sources(t, gaps, True) for t in range(1, 12)]
    ref = multi_flow_tracks(_stack(res, "flow").cuda(), _stack(res, "flow_bwd").cuda(), gaps, True)
    for k in ("tracks", "visible", "uncertainty"):
        assert torch.equal(_stack(res, k), ref[k].cpu()), k
    again = _run(runner, frames)
    for a, b in zip(res, again):
        for k in a:
            assert torch.equal(a[k], b[k]), k
    plain = _run(MultiFlowTrackRunner(m, (64, 96), batch, "cuda", gaps=gaps, padding_factor=pad, use_graph=use_graph,
                                      **call), frames)
    assert all(set(r) == {"tracks", "visible", "uncertainty"} for r in plain)
    for a, b in zip(res, plain):
        assert torch.equal(a["tracks"], b["tracks"]) and torch.equal(a["uncertainty"], b["uncertainty"])


def test_runner_against_infer_flow_pairs():
    """against `multi_flow_tracks` on `infer_flow`'s flows of the same pairs: the flows agree within the encoder's
    summation order (as in test_tracks_gpu.py), and the tracks agree but for the pixels where that difference moves a
    mask or a choice"""
    m, call = synthetic_model(_WL), workload_call(_WL, drop=("task",))
    pad = WORKLOADS[_WL]["pad"]
    gaps, h, w, T = (1, 2, 4), 64, 96, 9
    frames = synthetic_video(T, h, w, seed=23)
    res = _run(MultiFlowTrackRunner(m, (h, w), 2, "cuda", gaps=gaps, padding_factor=pad, return_flow=True, **call), frames)
    img = frames.permute(0, 3, 1, 2).float().cuda()
    k = len(gaps) + 1
    fwd = torch.zeros((T - 1, k, 2, h, w), device="cuda")
    bwd = torch.zeros_like(fwd)
    for t in range(1, T):
        src = multi_flow_sources(t, gaps, True)
        idx = [j for j, s in enumerate(src) if s >= 0]
        out = infer_flow(m, img[[src[j] for j in idx]], img[t].expand(len(idx), 3, h, w), padding_factor=pad,
                         pred_bidir_flow=True, **call)
        fwd[t - 1, idx], bwd[t - 1, idx] = out["flow"], out["flow_bwd"]
    present = torch.tensor([[s >= 0 for s in multi_flow_sources(t, gaps, True)] for t in range(1, T)])
    own = _stack(res, "flow").cuda()
    dflow = float((own - fwd)[present].abs().max())
    assert dflow <= 1e-4 * max(1.0, float(fwd.abs().max()))
    ref = multi_flow_tracks(fwd, bwd, gaps, True)
    d = (_stack(res, "tracks").cuda() - ref["tracks"]).abs().amax(-1)
    vis = (_stack(res, "visible").cuda() != ref["visible"]).float().mean().item()
    far = (d > 1e-2).float().mean().item()
    print("flows differ by %.2e px; tracks differ by more than 0.01 px on %.4f %% and visibility on %.4f %% of pixels"
          % (dflow, 100 * far, 100 * vis))
    assert far <= 0.01 and vis <= 0.01
