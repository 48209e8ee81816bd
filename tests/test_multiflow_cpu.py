"""Multi-flow dense point tracks without a device: the source schedule, the refusals of the C entries, `multi_flow_tracks`
and `MultiFlowTrackRunner` before any device work, the statement (tests/refops_multiflow.py) pinned to `chain_tracks` and
to the direct flow from frame 0, and the analytic occluder clip, where the multi-flow tracks bring back every point that
`chain_tracks` loses behind the square."""
import ctypes

import numpy as np
import pytest
import torch

import refops_multiflow as RM
import refops_tracks as RT
from unimatch_b200 import ops
from unimatch_b200.inference import MULTI_FLOW_GAPS, MultiFlowTrackRunner, multi_flow_sources, multi_flow_tracks


def test_sources_schedule():
    assert MULTI_FLOW_GAPS == (1, 2, 4, 8, 16, 32)
    assert multi_flow_sources(1) == [0, -1, -1, -1, -1, -1, 0]
    assert multi_flow_sources(2) == [1, 0, -1, -1, -1, -1, 0]
    assert multi_flow_sources(5) == [4, 3, 1, -1, -1, -1, 0]
    assert multi_flow_sources(32) == [31, 30, 28, 24, 16, 0, 0]          # frame 0 twice: as gap 32 and as the anchor
    assert multi_flow_sources(1000) == [999, 998, 996, 992, 984, 968, 0]
    assert multi_flow_sources(7, (4, 1), anchor=False) == [6, 3]          # gaps in increasing order
    assert multi_flow_sources(3, (), anchor=True) == [0]
    assert multi_flow_sources(1, (1,), anchor=False) == [0]
    assert multi_flow_sources(2, (8, 2), anchor=False) == [0, -1]


@pytest.mark.parametrize("gaps,anchor,t", [((0, 1), True, 3), ((-2,), True, 3), ((1, 1), True, 3), ((2, 4), False, 1),
                                           ((), False, 3), ((1.5,), True, 3), ((1,), True, 0)])
def test_sources_refusals(gaps, anchor, t):
    with pytest.raises(ValueError):
        multi_flow_sources(t, gaps, anchor)


def test_c_entries_refuse_before_any_cuda_call():
    L = ops.LIB
    one = ctypes.c_void_p(256)
    assert L.um_fb_consistency_error(one, one, 0.01, 0.5, one, one, None, 1, 4, 4, None) == -22
    assert L.um_fb_consistency_error(one, one, 0.01, 0.5, one, one, one, 1, 1, 4, None) == -22
    assert b"um_fb_consistency_error" in L.um_last_error()

    def call(**kw):
        a = dict(flow=256, occ=1 << 20, err=2 << 20, src=3 << 20, dst=4 << 20, n=2, k=3, h=4, w=5, r=4, pos=5 << 20,
                 sig=6 << 20, vis=7 << 20, tracks=8 << 20, visible=9 << 20, sigma=10 << 20)
        a.update(kw)
        p = {k: (ctypes.c_void_p(v) if v else None) for k, v in a.items() if k not in ("n", "k", "h", "w", "r")}
        return L.um_multi_flow_tracks(p["flow"], p["occ"], p["err"], p["src"], p["dst"], a["n"], a["k"], a["h"], a["w"],
                                      a["r"], p["pos"], p["sig"], p["vis"], p["tracks"], p["visible"], p["sigma"], None)
    for bad in (dict(err=0), dict(dst=0), dict(n=0), dict(k=0), dict(r=0), dict(h=1), dict(pos=(5 << 20) + 4),
                dict(sig=(6 << 20) + 2), dict(tracks=(5 << 20) + 8), dict(sigma=256 + 16)):
        assert call(**bad) == -22, bad
        assert b"um_multi_flow_tracks" in L.um_last_error()


def test_wrapper_and_runner_refusals():
    f = torch.zeros((3, 7, 2, 8, 8))
    with pytest.raises(ValueError, match="K = len"):
        multi_flow_tracks(f[:, :6], f[:, :6])                            # 6 candidates for the default 7
    with pytest.raises(ValueError, match="flows_bwd"):
        multi_flow_tracks(f, f[:2])
    with pytest.raises(ValueError, match="positive"):
        multi_flow_tracks(f[:, :2], f[:, :2], gaps=(1, 0), anchor=False)
    with pytest.raises(ValueError, match="no source"):
        multi_flow_tracks(f[:, :0], f[:, :0], gaps=(), anchor=False)
    with pytest.raises(ValueError, match="4 candidates|K = len"):
        multi_flow_tracks(f[..., 0, :, :], f[..., 0, :, :])
    for k in ("pred_bwd_flow", "visualize", "concat_frame", "visualize_bwd"):
        with pytest.raises(ValueError, match=k):
            MultiFlowTrackRunner(None, (32, 32), 1, "cpu", **{k: True})
    with pytest.raises(ValueError, match="always on"):
        MultiFlowTrackRunner(None, (32, 32), 1, "cpu", pred_bidir_flow=False)
    with pytest.raises(ValueError, match="distinct"):
        MultiFlowTrackRunner(None, (32, 32), 1, "cpu", gaps=(2, 2))
    with pytest.raises(ValueError, match="flow task"):
        MultiFlowTrackRunner(None, (32, 32), 1, "cpu", task="stereo")


def _random_case(n, h, w, gaps, anchor, seed):
    k = len(gaps) + anchor
    flows = RT.smooth_flows(n * k, h, w, 2.0, seed=seed, drift=(0.7, -0.4)).reshape(n, k, 2, h, w)
    rng = np.random.default_rng(seed + 1)
    occ = (rng.random((n, k, h, w)) < 0.15).astype(np.float32)
    err = (rng.random((n, k, h, w)) * 2).astype(np.float32)
    return flows, occ, err


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_gap_one_is_chain_tracks(dtype):
    """gaps=(1,), no anchor: one candidate per frame, the chain_tracks step, bit for bit"""
    flows, occ, err = _random_case(6, 23, 31, (1,), False, seed=4)
    got = RM.multi_flow_tracks(flows, occ, err, (1,), False, dtype=dtype)
    ref = RT.chain_tracks(flows[:, 0], occ[:, 0], dtype=dtype)
    assert np.array_equal(got["tracks"], ref["tracks"], equal_nan=True)
    assert np.array_equal(got["visible"], ref["visible"])


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_anchor_only_is_the_direct_flow(dtype):
    """gaps=(), anchor: x_t = p + F_{0->t}(p) at the integer pixel, visible from the direct pair alone"""
    n, h, w = 5, 21, 29
    flows, occ, err = _random_case(n, h, w, (), True, seed=9)
    got = RM.multi_flow_tracks(flows, occ, err, (), True, dtype=dtype)
    p, _ = RT.track_start(h, w, dtype)
    for t in range(n):
        f = flows[t, 0].astype(dtype)
        x = np.stack((p[..., 0] + f[0], p[..., 1] + f[1]), -1)
        inside = (x[..., 0] >= 0) & (x[..., 0] <= w - 1) & (x[..., 1] >= 0) & (x[..., 1] <= h - 1)
        assert np.array_equal(got["tracks"][t], x)
        assert np.array_equal(got["visible"][t], (occ[t, 0] < 0.5) & inside)
        assert np.array_equal(got["uncertainty"][t], err[t, 0].astype(dtype) ** 2)


def test_choice_rule():
    """the valid candidate of smallest sigma2 wins, the first on ties; with none valid the smallest of all, invisible"""
    h, w, gaps = 6, 7, (1, 2)
    flows = np.zeros((2, 3, 2, h, w), np.float32)
    flows[1, 0, 0], flows[1, 1, 0], flows[1, 2, 0] = 1.0, 2.0, 3.0         # frame 2 from frames 1, 0 and 0 (anchor)
    occ = np.zeros((2, 3, h, w), np.float32)
    err = np.zeros((2, 3, h, w), np.float32)
    err[1, 0], err[1, 1], err[1, 2] = 3.0, 1.0, 1.0
    got = RM.multi_flow_tracks(flows, occ, err, gaps, True)
    x = got["tracks"][1, ..., 0] - np.arange(w)
    assert np.all(x[:, :w - 2] == 2.0) and np.all(got["uncertainty"][1, :, :w - 2] == 1.0)   # gap 2 beats the tie
    occ[1, 1] = 1.0
    got = RM.multi_flow_tracks(flows, occ, err, gaps, True)
    assert np.all(got["tracks"][1, :, :w - 3, 0] - np.arange(w - 3) == 3.0) and got["visible"][1, :, :w - 3].all()
    occ[1] = 1.0
    got = RM.multi_flow_tracks(flows, occ, err, gaps, True)
    assert not got["visible"][1].any() and np.all(got["tracks"][1, ..., 0] - np.arange(w) == 2.0)


def test_fp32_residual_is_the_float64_one_within_rounding():
    """the float32 evaluation of the residual (the kernel's order) within a few roundings of the float64 statement, and its
    masks equal wherever the residual is not within that of the threshold"""
    flows = RT.smooth_flows(6, 33, 47, 4.0, seed=12, drift=(1.5, 0.5))
    fwd, bwd = flows[:3], -flows[3:] * 0.9
    o64, e64 = RM.fb_residual(fwd, bwd)
    o32, e32 = RM.fb_residual(fwd, bwd, dtype=np.float32)
    assert e32.dtype == np.float32
    scale = np.abs(fwd).max() + np.abs(bwd).max() + 1.0
    tol = 64 * 2.0 ** -24 * scale
    assert np.abs(e32 - e64).max() <= tol
    thr = 0.01 * (np.hypot(fwd[:, 0], fwd[:, 1]) + np.hypot(bwd[:, 0], bwd[:, 1])) + 0.5
    sure = np.abs(e64 - thr) > 2 * tol
    assert np.array_equal(o32[sure], o64[sure]) and sure.mean() > 0.99 and 0 < o64.mean() < 1


def _occluder(gaps, anchor):
    clip = RM.OccluderClip()
    n, h, w = clip.frames - 1, clip.h, clip.w
    fwd, bwd = RM.pair_flows(clip.flows, n, gaps, anchor, h, w)
    occ = np.full(fwd.shape[:2] + (h, w), np.nan, np.float32)
    err = occ.copy()
    for t in range(n):
        ok = ~np.isnan(fwd[t, :, 0, 0, 0])
        occ[t, ok], err[t, ok] = RM.fb_residual(fwd[t, ok], bwd[t, ok], dtype=np.float32)
    return clip, fwd, bwd, occ, err


def occluder_checks(clip, tracks, visible, chain_visible=None, first_frame=1):
    """What the clip shows: background points the square passes over are visible, at their exact positions, in every frame
    t >= first_frame where they are uncovered and inside (and invisible where covered); chain_tracks loses each of them
    for good from its first covered frame.  Returns how many such points there are."""
    pos, covered, inside, background = clip.truth()
    passed = background & covered.any(axis=0)
    assert passed.sum() > 50
    t = np.arange(1, clip.frames)[:, None, None]
    shown = ~covered[1:] & inside[1:] & passed[None] & (t >= first_frame)
    assert np.array_equal(visible.astype(bool)[shown], np.ones(int(shown.sum()), bool))
    assert not visible.astype(bool)[covered[1:] & passed[None]].any()
    assert np.array_equal(tracks[shown], pos[1:][shown])
    if chain_visible is not None:
        first = np.argmax(covered, axis=0)
        later = (np.arange(clip.frames)[:, None, None] >= first[None]) & passed[None]
        assert not chain_visible[later[1:]].any()
        assert (shown & ~chain_visible.astype(bool)).sum() > 0.3 * shown.sum()      # what the multi-flow tracks bring back
    return int(passed.sum())


def test_occluder_clip_chain_loses_points_multi_flow_brings_them_back():
    clip, fwd, bwd, occ, err = _occluder((1,), False)
    chain = RT.chain_tracks(fwd[:, 0], occ[:, 0], dtype=np.float32)
    clip, fwd, bwd, occ, err = _occluder(MULTI_FLOW_GAPS, True)
    got = RM.multi_flow_tracks(fwd, occ, err, MULTI_FLOW_GAPS, True, dtype=np.float32)
    occluder_checks(clip, got["tracks"], got["visible"], chain["visible"])


def test_occluder_clip_long_gap_without_anchor():
    """no anchor: the consecutive chain and one gap longer than any point stays covered (10 px square, 3 px per frame
    relative speed: at most 4 frames).  A point reappears through the long flow once that flow reaches back before its
    occlusion, i.e. from frame 8 on for every point covered at frame 7 or later"""
    gaps = (1, 8)
    clip, fwd, bwd, occ, err = _occluder(gaps, False)
    got = RM.multi_flow_tracks(fwd, occ, err, gaps, False, dtype=np.float32)
    pos, covered, _, background = clip.truth()
    late = covered[:8].sum(axis=0) == 0                 # not covered before frame 8
    assert (background & covered.any(axis=0) & late).sum() > 30
    # the points covered earlier stand in with their truth, so the checks below speak of the late ones only
    vis = np.where(late[None], got["visible"], ~covered[1:])
    trk = np.where(late[None, ..., None], got["tracks"], pos[1:])
    occluder_checks(clip, trk, vis, first_frame=8)
