"""Query point tracks without a device: the statement (tests/refops_points.py) against the reference's own `flow_warp` and
`forward_backward_consistency_check` iterated forward and backward from the query frame, the fp32 order of operations
against the statement within its rounding bound, both directions against the dense statement, the refusals of
`um_track_points_forward` / `um_track_points_backward`, `track_points` and `PointTrackRunner` before any device work, and
`tapvid_metrics` on hand-computed cases."""
import ctypes
import importlib.util
import os

import numpy as np
import pytest
import torch

import refops_points as RP
import refops_tracks as RT
from unimatch_b200 import ops
from unimatch_b200.evaluation import tapvid_metrics
from unimatch_b200.inference import PointTrackRunner, track_points

REFERENCE = os.environ.get("UNIMATCH_REFERENCE", "/root/reference")
needs_reference = pytest.mark.skipif(not os.path.isfile(os.path.join(REFERENCE, "unimatch", "geometry.py")),
                                     reason="the reference tree is not available (set UNIMATCH_REFERENCE)")


def _reference_geometry():
    spec = importlib.util.spec_from_file_location("reference_geometry", os.path.join(REFERENCE, "unimatch", "geometry.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _bidir(n, h, w, seed, drift=(2.5, -1.5)):
    """seeded forward flows, backward flows near their negation, and binary masks of a fifth of the pixels"""
    fwd = RT.smooth_flows(n, h, w, 3.0, seed=seed, drift=drift)
    bwd = (-fwd + RT.smooth_flows(n, h, w, 0.5, seed=seed + 50)).astype(np.float32)
    rng = np.random.default_rng(seed + 1)
    occ = [(rng.random((n, h, w)) < 0.2).astype(np.float32) for _ in range(2)]
    return fwd, bwd, occ[0], occ[1]


@needs_reference
@pytest.mark.parametrize("n,hw,tq,offset", [(4, (23, 31), 2, (0.25, 0.6)), (5, (40, 28), 0, (0.0, 0.0)),
                                            (5, (30, 30), 5, (0.5, 0.125)), (6, (26, 35), 3, (0.0, 0.0))])
def test_statement_equals_reference_iterated(n, hw, tq, offset):
    """every pixel (+ a fractional offset) queried at frame tq: p_t = p + flow_warp(F, p - grid) forward through the
    forward flows from pair tq, backward through the backward flows from pair tq-1 down to 0, with the masks of the
    reference's forward_backward_consistency_check, all in float64"""
    G = _reference_geometry()
    h, w = hw
    fwd = torch.from_numpy(RT.smooth_flows(n, h, w, 1.0, seed=n + h, drift=(1.5, 0.5))).double()
    bwd = -fwd + torch.from_numpy(RT.smooth_flows(n, h, w, 0.3, seed=n + 100)).double()
    occs = [G.forward_backward_consistency_check(fwd[t:t + 1], bwd[t:t + 1]) for t in range(n)]
    focc = torch.cat([o[0] for o in occs]).double()
    bocc = torch.cat([o[1] for o in occs]).double()
    assert 0 < focc.mean() < 1 and 0 < bocc.mean() < 1
    grid = G.coords_grid(1, h, w).double()
    start = grid + torch.tensor(offset, dtype=torch.float64)[None, :, None, None]      # (dx, dy)
    keep = ((start[0, 0] <= w - 1) & (start[0, 1] <= h - 1)).numpy()
    ref_p = np.empty((h, w, n + 1, 2))
    ref_v = np.empty((h, w, n + 1), bool)
    ref_p[:, :, tq], ref_v[:, :, tq] = start[0].permute(1, 2, 0).numpy(), True
    for pairs, flows, masks, frame in ((range(tq, n), fwd, focc, 1), (range(tq - 1, -1, -1), bwd, bocc, 0)):
        p, vis = start.clone(), torch.ones((1, h, w), dtype=torch.bool)
        for j in pairs:
            d = G.flow_warp(flows[j:j + 1], p - grid)
            o = G.flow_warp(masks[j:j + 1, None], p - grid)[:, 0]
            p = p + d
            vis = vis & (o < 0.5) & (p[:, 0] >= 0) & (p[:, 0] <= w - 1) & (p[:, 1] >= 0) & (p[:, 1] <= h - 1)
            ref_p[:, :, j + frame] = p[0].permute(1, 2, 0).numpy()
            ref_v[:, :, j + frame] = vis[0].numpy()
    ys, xs = np.nonzero(keep)
    s = start[0].numpy()
    queries = np.stack((np.full(len(ys), tq, np.float64), s[1][ys, xs], s[0][ys, xs]), axis=-1)
    got = RP.track_points(fwd.numpy(), bwd.numpy(), focc.numpy(), bocc.numpy(), queries)
    assert np.abs(got["tracks"] - ref_p[ys, xs]).max() <= 1e-9
    assert got["visible"].any() and not got["visible"].all()      # some tracks leave or get occluded, some stay
    total, unexplained = RP.visibility_mismatches(ref_v[ys, xs], got, queries, h, w, 1e-9, 1e-9)
    assert unexplained == 0 and total <= 1, total


@pytest.mark.parametrize("n,hw,frames", [(3, (37, 53), None), (8, (61, 40), [0, 4, 8]), (8, (96, 160), None)])
def test_fp32_order_within_rounding_of_statement(n, hw, frames):
    """float32 (the kernels' expression) within `chain_tolerance` of the float64 statement at every frame reached by a
    path that stays in the frame, |t - t_q| steps away from the query"""
    h, w = hw
    fwd, bwd, focc, bocc = _bidir(n, h, w, seed=11)
    q = RP.random_queries(300, n + 1, h, w, seed=12, frames=frames)
    ref = RP.track_points(fwd, bwd, focc, bocc, q)
    got = RP.track_points(fwd, bwd, focc, bocc, q, dtype=np.float32)
    tol = RT.chain_tolerance(ref["tracks"], np.concatenate((fwd, bwd)))
    tq = q[:, 0].astype(int)
    x, y = ref["tracks"][..., 0], ref["tracks"][..., 1]
    inside = (x >= 0) & (x <= w - 1) & (y >= 0) & (y <= h - 1)
    worst = 0.0
    for i in range(len(q)):
        for frames_out in (range(tq[i] + 1, n + 1), range(tq[i] - 1, -1, -1)):
            for k, t in enumerate(frames_out):
                if not inside[i, t]:
                    break
                err = float(np.abs(got["tracks"][i, t] - ref["tracks"][i, t]).max())
                worst = max(worst, err)
                assert err <= tol[k], (i, t, err, tol[k])
        assert np.array_equal(got["tracks"][i, tq[i]], q[i, [2, 1]]) and got["visible"][i, tq[i]]
    total, unexplained = RP.visibility_mismatches(got["visible"], ref, q, h, w, tol[n - 1], 2 * tol[n - 1] + 1e-6)
    assert unexplained == 0 and total <= 3, total


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_both_directions_equal_the_dense_statement(dtype):
    """a query at an integer pixel: forward = refops_tracks.chain_tracks(flows[t_q:], fwd_occ[t_q:]) and backward =
    refops_tracks.chain_tracks(flows_bwd[t_q-1::-1], bwd_occ[t_q-1::-1]) at that pixel, exactly"""
    n, h, w = 7, 29, 41
    fwd, bwd, focc, bocc = _bidir(n, h, w, seed=21)
    ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    for tq in (0, 3, n):
        q = np.stack((np.full(h * w, tq), ys.ravel(), xs.ravel()), -1).astype(np.float32)
        got = RP.track_points(fwd, bwd, focc, bocc, q, dtype=dtype)
        tracks, visible = got["tracks"].reshape(h, w, n + 1, 2), got["visible"].reshape(h, w, n + 1)
        if tq < n:
            dense = RT.chain_tracks(fwd[tq:], focc[tq:], dtype=dtype)
            assert np.array_equal(tracks[:, :, tq + 1:].transpose(2, 0, 1, 3), dense["tracks"])
            assert np.array_equal(visible[:, :, tq + 1:].transpose(2, 0, 1), dense["visible"])
        if tq > 0:
            dense = RT.chain_tracks(bwd[tq - 1::-1], bocc[tq - 1::-1], dtype=dtype)
            assert np.array_equal(tracks[:, :, tq - 1::-1].transpose(2, 0, 1, 3), dense["tracks"])
            assert np.array_equal(visible[:, :, tq - 1::-1].transpose(2, 0, 1), dense["visible"])


def test_statement_without_masks():
    """masks None: only the frame decides; zero flow keeps every query where it is in every frame"""
    n, h, w = 4, 9, 13
    zero = np.zeros((n, 2, h, w), np.float32)
    q = np.array([[0, 2.5, 3.25], [4, 8, 12], [2, 0, 0]], np.float32)
    got = RP.track_points(zero, zero, None, None, q)
    assert np.array_equal(got["tracks"], np.broadcast_to(q[:, None, [2, 1]], (3, n + 1, 2))) and got["visible"].all()


def _ptr(k):
    return ctypes.c_void_p(k << 20)


def test_c_abi_refusals_without_a_gpu():
    """um_track_points_forward / um_track_points_backward check their arguments before any CUDA call"""
    fwd = dict(flow=_ptr(1), occ=None, n=2, h=8, w=8, t0=0, queries=_ptr(2), nq=4, nt=5, pos=_ptr(3), vis=_ptr(4),
               tracks=_ptr(5), visible=_ptr(6))
    bad = [dict(flow=None), dict(queries=None), dict(pos=None), dict(vis=None), dict(tracks=None), dict(visible=None),
           dict(n=0), dict(h=1), dict(w=0), dict(nq=0), dict(h=1 << 16, w=1 << 16), dict(t0=-1), dict(t0=3),
           dict(n=5), dict(nt=2), dict(flow=ctypes.c_void_p((1 << 20) + 2)), dict(pos=ctypes.c_void_p((3 << 20) + 4)),
           dict(tracks=ctypes.c_void_p((5 << 20) + 4)), dict(visible=ctypes.c_void_p((5 << 20) + 8)),
           dict(pos=ctypes.c_void_p((2 << 20) + 8)), dict(tracks=ctypes.c_void_p((1 << 20) + 64))]
    for change in bad:
        a = dict(fwd, **change)
        rc = ops.LIB.um_track_points_forward(a["flow"], a["occ"], a["n"], a["h"], a["w"], a["t0"], a["queries"], a["nq"],
                                             a["nt"], a["pos"], a["vis"], a["tracks"], a["visible"], None)
        assert rc == -22, change
        assert b"um_track_points_forward" in ops.LIB.um_last_error(), change
    bwd = dict(flow=_ptr(1), occ=_ptr(7), n=2, h=8, w=8, queries=_ptr(2), nq=4, nt=5, tracks=_ptr(5), visible=_ptr(6))
    bad = [dict(flow=None), dict(queries=None), dict(tracks=None), dict(visible=None), dict(n=-1), dict(h=1), dict(nq=0),
           dict(nt=1, n=0), dict(n=5), dict(h=1 << 16, w=1 << 16), dict(occ=ctypes.c_void_p((7 << 20) + 1)),
           dict(tracks=ctypes.c_void_p((5 << 20) + 4)), dict(visible=ctypes.c_void_p((5 << 20) + 16)),
           dict(tracks=ctypes.c_void_p((7 << 20) + 128)), dict(visible=ctypes.c_void_p((2 << 20) + 4))]
    for change in bad:
        a = dict(bwd, **change)
        rc = ops.LIB.um_track_points_backward(a["flow"], a["occ"], a["n"], a["h"], a["w"], a["queries"], a["nq"], a["nt"],
                                              a["tracks"], a["visible"], None)
        assert rc == -22, change
        assert b"um_track_points_backward" in ops.LIB.um_last_error(), change


BAD_QUERIES = [np.zeros((4, 2)), np.zeros((0, 3)), np.zeros((2, 3, 1)), [[0, float("nan"), 1]], [[0, 1, float("inf")]],
               [[1.5, 2, 2]], [[-1, 2, 2]], [[0, -0.5, 2]], [[0, 2, 12.01]], [[0, 6, 2]]]


@pytest.mark.parametrize("queries", BAD_QUERIES)
def test_track_points_refuses_queries(queries):
    """6x13 frames, 3 pairs: queries must be [N,3], finite, at a non-negative integer frame and inside the frame"""
    flow = torch.zeros((3, 2, 6, 13))
    with pytest.raises(ValueError):
        track_points(flow, flow, None, None, queries)


def test_track_points_refusals():
    flow = torch.zeros((3, 2, 6, 7))
    ok = np.array([[1, 2, 3]], np.float32)
    for args in [(torch.zeros((3, 3, 6, 7)), flow, None, None, ok), (torch.zeros((0, 2, 6, 7)),) * 2 + (None, None, ok),
                 (flow, torch.zeros((2, 2, 6, 7)), None, None, ok), (flow, flow, torch.zeros((3, 6, 6)), None, ok),
                 (flow, flow, None, torch.zeros((2, 6, 7)), ok)]:
        with pytest.raises(ValueError):
            track_points(*args)
    with pytest.raises(ValueError, match="query 1 is given at frame 4 of a clip of 4 frames"):
        track_points(flow, flow, None, None, [[3, 2, 3], [4, 2, 3]])
    with pytest.raises(RuntimeError):                                 # no CPU kernel: the op refuses host tensors
        track_points(flow, flow, None, None, ok)


@pytest.mark.parametrize("flag", [dict(pred_bwd_flow=True), dict(visualize=True), dict(concat_frame=True),
                                  dict(visualize_bwd=True), dict(pred_bidir_flow=False),
                                  dict(fwd_bwd_consistency_check=False)])
def test_runner_refused_flags(flag):
    with pytest.raises(ValueError):
        PointTrackRunner(None, (32, 48), 2, "cuda", **flag)


def test_runner_track_refusals_before_device_work():
    """queries and clips of fewer than two frames are refused before the runner touches the device (here: a runner
    without device state, so any device work would fail differently)"""
    r = object.__new__(PointTrackRunner)
    r.h, r.w = 6, 13
    frames = [np.zeros((6, 13, 3), np.uint8)] * 3
    for q in BAD_QUERIES:
        with pytest.raises(ValueError):
            r.track(frames, q)
    for clip in ([], frames[:1], iter(frames[:1])):
        with pytest.raises(ValueError, match="at least two frames"):
            r.track(clip, [[0, 1, 1]])


# ---- tapvid_metrics ----------------------------------------------------------------------------------------------------
def _case(b=1, n=2, t=4):
    qp = np.zeros((b, n, 3))
    occ = np.zeros((b, n, t), bool)
    gt = np.zeros((b, n, t, 2))
    return qp, occ, gt


def test_tapvid_metrics_perfect_prediction():
    qp, occ, gt = _case(b=2)
    occ[0, 1, 2] = True
    for mode in ("first", "strided"):
        m = tapvid_metrics(qp, occ, gt, occ.copy(), gt.copy(), mode)
        for k, v in m.items():
            assert v.shape == (2,) and np.array_equal(v, [1.0, 1.0]), k


def test_tapvid_metrics_all_predicted_occluded():
    qp, occ, gt = _case()
    m = tapvid_metrics(qp, occ, gt, np.ones_like(occ), gt, "first")
    assert m["occlusion_accuracy"][0] == 0.0                          # every evaluation point is visible in truth
    assert m["pts_within_1"][0] == 1.0                                # positions are scored on true visibility only
    assert m["jaccard_1"][0] == 0.0 and m["average_jaccard"][0] == 0.0


def test_tapvid_metrics_known_counts():
    """one video, two tracks of 5 frames queried at frame 0 ('first': 8 evaluation points)"""
    qp, occ, gt = _case(n=2, t=5)
    pred = gt.copy()
    pred_occ = occ.copy()
    occ[0, 0, 4] = True                      # truth: point (0, 4) occluded -> 7 visible evaluation points
    pred_occ[0, 1, 3] = True                 # predicted occluded where visible: occlusion disagrees at (1, 3) and (0, 4)
    pred[0, 0, 1] = (1.5, 0)                 # 1.5 px off: within 2, 4, 8, 16, not 1
    pred[0, 0, 2] = (0, 3)                   # 3 px off: within 4, 8, 16
    pred[0, 1, 1] = (10, 0)                  # 10 px off: within 16
    m = tapvid_metrics(qp, occ, gt, pred_occ, pred, "first")
    assert m["occlusion_accuracy"][0] == 6 / 8
    # visible evaluation points: (0,1) (0,2) (0,3) (1,1) (1,2) (1,3) (1,4); within d: 1: (0,3) (1,2) (1,3) (1,4) = 4
    assert [m["pts_within_%d" % d][0] for d in (1, 2, 4, 8, 16)] == [4 / 7, 5 / 7, 6 / 7, 6 / 7, 7 / 7]
    # predicted visible: all but (1,3); (0,4) is predicted visible but truly occluded -> FP at every d
    # d=1: TP = (0,3) (1,2) (1,4) = 3, FP = (0,1) (0,2) (1,1) (0,4) = 4 -> 3 / (7 + 4)
    # d=2: TP 4, FP 3 -> 4 / 10;  d=4, 8: TP 5, FP 2 -> 5 / 9;  d=16: TP 6, FP 1 -> 6 / 8
    want = [3 / 11, 4 / 10, 5 / 9, 5 / 9, 6 / 8]
    assert np.allclose([m["jaccard_%d" % d][0] for d in (1, 2, 4, 8, 16)], want, rtol=0, atol=1e-15)
    assert np.isclose(m["average_jaccard"][0], np.mean(want)) and np.isclose(m["average_pts_within_thresh"][0],
                                                                             np.mean([4, 5, 6, 6, 7]) / 7)


def test_tapvid_metrics_first_against_strided_and_query_frame_excluded():
    """a track queried at frame 2 of 4: 'first' scores frame 3 only, 'strided' frames 0, 1 and 3; frame 2 never counts"""
    qp, occ, gt = _case(n=1, t=4)
    qp[0, 0, 0] = 2
    pred = gt.copy()
    pred[0, 0, 0] = (100, 0)                 # wrong before the query frame
    pred[0, 0, 2] = (100, 0)                 # wrong AT the query frame: excluded in both modes
    pred_occ = occ.copy()
    pred_occ[0, 0, 2] = True
    first = tapvid_metrics(qp, occ, gt, pred_occ, pred, "first")
    strided = tapvid_metrics(qp, occ, gt, pred_occ, pred, "strided")
    assert first["occlusion_accuracy"][0] == 1.0 and first["pts_within_16"][0] == 1.0 and first["jaccard_1"][0] == 1.0
    assert strided["occlusion_accuracy"][0] == 1.0 and strided["pts_within_16"][0] == 2 / 3
    assert strided["jaccard_16"][0] == 2 / 4                  # TP 2, 3 visible + FP 1
    qp[0, 0, 0] = 3                                          # queried at the last frame: nothing to score with 'first'
    m = tapvid_metrics(qp, occ, gt, occ, gt, "first")
    assert np.isnan(m["occlusion_accuracy"][0]) and np.isnan(m["pts_within_1"][0]) and np.isnan(m["average_jaccard"][0])
    with pytest.raises(ValueError):
        tapvid_metrics(qp, occ, gt, occ, gt, "last")
