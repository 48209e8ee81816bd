"""Query point tracks on the device: `um_track_points_forward` / `um_track_points_backward` (through `track_points`) bit for
bit against the float32 statement (tests/refops_points.py), the identities with `um_chain_tracks`, forward chains split
across launches, and `PointTrackRunner` against `track_points` on its own flows, against `VideoFlowRunner`, and across
calls.  The kernels evaluate the statement's expression in fp32 in the order the header fixes, so every comparison here is
exact; how far fp32 lies from the float64 statement is tests/test_points_cpu.py's subject."""
import numpy as np
import pytest
import torch

import refops_points as RP
import refops_tracks as RT
from unimatch_b200.inference import (PointTrackRunner, VideoFlowRunner, chain_tracks, infer_flow_video, track_points)
from unimatch_b200.spec import WORKLOADS
from unimatch_b200.synthetic import synthetic_model, synthetic_video, workload_call

_WL = "gmflow-scale1"

pytestmark = pytest.mark.gpu
_OPS = torch.ops.unimatch_sm100


def _inputs(n, h, w, occ_kind, seed):
    """forward flows drifting out of the frame, backward flows drifting the other way, masks binary / soft / absent"""
    fwd = RT.smooth_flows(n, h, w, 3.0, seed=seed, drift=(2.5, -1.5))
    bwd = RT.smooth_flows(n, h, w, 3.0, seed=seed + 7, drift=(-2.0, 1.5))
    rng = np.random.default_rng(seed + 1)
    masks = {"none": (None, None),
             "binary": tuple((rng.random((n, h, w)) < 0.2).astype(np.float32) for _ in range(2)),
             "soft": tuple(rng.random((n, h, w)).astype(np.float32) for _ in range(2))}[occ_kind]
    return fwd, bwd, masks[0], masks[1]


def _cuda(*arrays):
    return [None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]


def _host(out):
    return out["tracks"].cpu().numpy(), out["visible"].cpu().numpy()


@pytest.mark.parametrize("n,hw,occ_kind", [(3, (37, 53), "binary"), (5, (61, 40), "soft"), (4, (37, 53), "none"),
                                           (8, (480, 832), "binary")])
def test_kernels_match_statement(n, hw, occ_kind):
    """fractional queries, queries on the edges and corners, at the first, middle and last frames"""
    h, w = hw
    fwd, bwd, focc, bocc = _inputs(n, h, w, occ_kind, seed=n * 5 + h)
    q = RP.random_queries(600, n + 1, h, w, seed=n + w)
    q[-3:, 0] = (0, n // 2, n)
    assert {0, n // 2, n} <= set(q[:, 0].astype(int).tolist())
    tracks, visible = _host(track_points(*_cuda(fwd, bwd, focc, bocc), q))
    assert tracks.shape == (600, n + 1, 2) and visible.dtype == np.uint8 and set(np.unique(visible)) <= {0, 1}
    emu = RP.track_points(fwd, bwd, focc, bocc, q, dtype=np.float32)
    assert np.array_equal(tracks, emu["tracks"]) and np.array_equal(visible.astype(bool), emu["visible"])
    x, y = emu["tracks"][..., 0], emu["tracks"][..., 1]
    gone = (x < 0) | (x > w - 1) | (y < 0) | (y > h - 1)
    assert gone.any() and not visible[gone].any()                     # tracks that leave the frame are invisible
    assert visible.all(axis=1).any() or occ_kind != "none"
    print("%dx%d n=%d %s: %.1f %% of entries visible, %.1f %% outside the frame"
          % (h, w, n, occ_kind, 100 * visible.mean(), 100 * gone.mean()))


def test_identities_with_chain_tracks():
    """a query at an integer pixel: forward = chain_tracks(flows[t_q:], fwd_occ[t_q:]) and backward =
    chain_tracks(flows_bwd[t_q-1::-1], bwd_occ[t_q-1::-1]) at that pixel, bit for bit"""
    n, h, w = 6, 45, 67
    fwd, bwd, focc, bocc = _cuda(*_inputs(n, h, w, "binary", seed=3))
    ys, xs = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    for tq in (0, 2, n):
        q = torch.stack((torch.full((h * w,), tq), ys.reshape(-1), xs.reshape(-1)), -1).float()
        out = track_points(fwd, bwd, focc, bocc, q)
        tracks, visible = out["tracks"].reshape(h, w, n + 1, 2), out["visible"].reshape(h, w, n + 1)
        if tq < n:
            dense = chain_tracks(fwd[tq:], focc[tq:])
            assert torch.equal(tracks[:, :, tq + 1:].permute(2, 0, 1, 3), dense["tracks"])
            assert torch.equal(visible[:, :, tq + 1:].permute(2, 0, 1), dense["visible"])
        if tq > 0:
            dense = chain_tracks(bwd[:tq].flip(0), bocc[:tq].flip(0))
            assert torch.equal(tracks[:, :, :tq].flip(2).permute(2, 0, 1, 3), dense["tracks"])
            assert torch.equal(visible[:, :, :tq].flip(2).permute(2, 0, 1), dense["visible"])


def test_forward_split_across_launches():
    """forward launches over pairs (0..2), (3), (4..7) equal one launch over (0..7); the backward launch serves queries up
    to its n stored pairs and gives the others a NaN, invisible row"""
    n, h, w = 8, 40, 56
    fwd, bwd, focc, bocc = _cuda(*_inputs(n, h, w, "soft", seed=9))
    qd = torch.from_numpy(RP.random_queries(300, n + 1, h, w, seed=10)).cuda()
    tables = []
    for cuts in ([(0, 8)], [(0, 3), (3, 4), (4, 8)], [(t, t + 1) for t in range(8)]):
        tracks = torch.zeros((300, n + 1, 2), device="cuda")
        visible = torch.zeros((300, n + 1), device="cuda", dtype=torch.uint8)
        pos = torch.empty((300, 2), device="cuda")
        vis = torch.empty((300,), device="cuda", dtype=torch.uint8)
        for a, b in cuts:
            _OPS.track_points_forward(fwd[a:b], focc[a:b], a, qd, pos, vis, tracks, visible)
        tables.append((tracks, visible))
    for tracks, visible in tables[1:]:
        assert torch.equal(tracks, tables[0][0]) and torch.equal(visible, tables[0][1])
    tracks, visible = tables[0]
    _OPS.track_points_backward(bwd[:4], bocc[:4], qd, tracks, visible)
    served = qd[:, 0] <= 4
    assert 0 < served.sum() < 300
    assert torch.isnan(tracks[~served]).all() and not visible[~served].any()
    ref = track_points(fwd, bwd, focc, bocc, qd)
    assert torch.equal(tracks[served], ref["tracks"][served]) and torch.equal(visible[served], ref["visible"][served])


def test_track_points_on_infer_flow_video():
    m, call = synthetic_model(_WL), workload_call(_WL, drop=("task",))
    pad = WORKLOADS[_WL]["pad"]
    frames = synthetic_video(7, 64, 96, seed=12)
    ifv = infer_flow_video(m, frames.cuda(), padding_factor=pad, pred_bidir_flow=True, fwd_bwd_consistency_check=True,
                           **call)
    q = RP.random_queries(200, 7, 64, 96, seed=13)
    tracks, visible = _host(track_points(ifv["flow"], ifv["flow_bwd"], ifv["fwd_occ"], ifv["bwd_occ"], q))
    host = {k: v.cpu().numpy() for k, v in ifv.items()}
    emu = RP.track_points(host["flow"], host["flow_bwd"], host["fwd_occ"], host["bwd_occ"], q, dtype=np.float32)
    assert np.array_equal(tracks, emu["tracks"]) and np.array_equal(visible.astype(bool), emu["visible"])


@pytest.mark.parametrize("batch,hw,use_graph,stream", [(1, (64, 96), True, False), (3, (64, 96), False, True),
                                                       (3, (80, 48), True, False), (8, (64, 96), True, True),
                                                       (8, (64, 96), False, False)])
def test_runner(batch, hw, use_graph, stream):
    """11 frames (10 pairs: steps of 1, of 3 + 3 + 3 + 1, of 8 + 2), landscape and portrait, graph and eager, a list or a
    generator of frames (the tables then grow as the stream goes).  The tracks are `track_points` on the runner's own flows
    bit for bit; the flows are VideoFlowRunner's bit for bit; a second call with other queries is independent of the
    first; return_flow=False returns the same tracks only; a query past the clip's end is refused, naming it"""
    m, call = synthetic_model(_WL), workload_call(_WL, drop=("task",))
    pad = WORKLOADS[_WL]["pad"]
    h, w = hw
    frames = list(synthetic_video(11, h, w, seed=31).numpy())
    clip = (lambda: (f for f in frames)) if stream else (lambda: frames)
    q1 = RP.random_queries(256, 11, h, w, seed=batch + h)
    q1[:3, 0] = (0, 5, 10)
    q2 = RP.random_queries(100, 11, h, w, seed=99, frames=[0, 1, 7])
    runner = PointTrackRunner(m, hw, batch, "cuda", padding_factor=pad, use_graph=use_graph, return_flow=True, **call)
    first = runner.track(clip(), q1)
    assert set(first) == {"tracks", "visible", "flow", "flow_bwd", "fwd_occ", "bwd_occ"}
    assert first["tracks"].shape == (256, 11, 2) and first["flow"].shape == (10, 2, h, w)
    own = track_points(*[first[k].cuda() for k in ("flow", "flow_bwd", "fwd_occ", "bwd_occ")], q1)
    assert torch.equal(first["tracks"], own["tracks"].cpu()) and torch.equal(first["visible"], own["visible"].cpu())

    fr = VideoFlowRunner(m, hw, batch, "cuda", padding_factor=pad, use_graph=use_graph, pred_bidir_flow=True,
                         fwd_bwd_consistency_check=True, **call)
    pairs = [{k: v.clone() for k, v in r.items()} for r in fr.run(frames)]
    assert len(pairs) == 10 and set(pairs[0]) == {"flow", "flow_bwd", "fwd_occ", "bwd_occ"}
    for k in pairs[0]:
        assert torch.equal(first[k], torch.stack([p[k] for p in pairs])), k

    second = runner.track(clip(), q2)
    own = track_points(*[second[k].cuda() for k in ("flow", "flow_bwd", "fwd_occ", "bwd_occ")], q2)
    assert torch.equal(second["tracks"], own["tracks"].cpu()) and torch.equal(second["visible"], own["visible"].cpu())
    again = runner.track(clip(), q1)
    assert torch.equal(again["tracks"], first["tracks"]) and torch.equal(again["visible"], first["visible"])

    slim = PointTrackRunner(m, hw, batch, "cuda", padding_factor=pad, use_graph=use_graph, **call).track(clip(), q1)
    assert set(slim) == {"tracks", "visible"}
    assert torch.equal(slim["tracks"], first["tracks"]) and torch.equal(slim["visible"], first["visible"])
    late = q2.copy()
    late[42, 0] = 11
    with pytest.raises(ValueError, match="query 42 is given at frame 11 of a clip of 11 frames"):
        runner.track(clip(), late)
    print("batch %d %dx%d graph %s: %.1f %% of entries visible" % (batch, h, w, use_graph,
                                                                   100 * first["visible"].float().mean()))
