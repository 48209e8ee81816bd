"""Dense point tracks on the device: `um_chain_tracks` against the statement (tests/refops_tracks.py), and `VideoTrackRunner`
against the statement applied to `infer_flow_video`'s flows and masks, to its own flows, across graph replay and against
`VideoFlowRunner`.

Tolerances.  The kernel evaluates the statement's expression in fp32 in the order the header fixes, so it equals the
statement evaluated with numpy float32 bit for bit.  Against the float64 statement a step adds at most half a unit in the
last place of the largest |p| plus ten roundings relative to the largest |F| (`refops_tracks.step_rounding`: 3.1e-5 px at
480x832); over a chain that error grows by at most (1 + 2 L) per step inside the frame, L the flows' largest neighbour
difference (`refops_tracks.chain_tolerance`).  A visibility test within that distance of a frame edge, or within twice it of
o = 0.5 (a mask in [0, 1] changes by at most 1 per pixel along each axis), may fall either way: such tracks are counted and
bounded, and every other track must agree."""
import numpy as np
import pytest
import torch

import refops_tracks as RT
from unimatch_b200.inference import VideoFlowRunner, VideoTrackRunner, chain_tracks, infer_flow_video
from unimatch_b200.spec import WORKLOADS
from unimatch_b200.synthetic import synthetic_model, synthetic_video, workload_call

_WL = "gmflow-scale1"

pytestmark = pytest.mark.gpu
_OPS = torch.ops.unimatch_sm100


def _inputs(n, h, w, occ_kind, seed):
    flow = RT.smooth_flows(n, h, w, 3.0, seed=seed, drift=(2.5, -1.5))
    rng = np.random.default_rng(seed + 1)
    occ = {"none": None, "binary": (rng.random((n, h, w)) < 0.2).astype(np.float32),
           "soft": rng.random((n, h, w)).astype(np.float32)}[occ_kind]
    return flow, occ


def _check_against_statement(tracks, visible, flow, occ, start=None):
    """bit for bit against the float32 evaluation; within rounding of the float64 statement (each step from the kernel's
    own previous positions, and the whole chain on tracks that stay in the frame); visibility equal but for tracks within
    rounding of a threshold, which are counted and bounded"""
    n, _, h, w = flow.shape
    emu = RT.chain_tracks(flow, occ, state=start, dtype=np.float32)
    assert np.array_equal(tracks, emu["tracks"], equal_nan=True)
    assert np.array_equal(visible.astype(bool), emu["visible"])
    ref = RT.chain_tracks(flow, occ, state=start)
    eps = RT.step_rounding(ref["tracks"], flow)
    prev = RT.track_start(h, w, np.float32) if start is None else start
    for t in range(n):
        one = RT.chain_tracks(flow[t:t + 1], None if occ is None else occ[t:t + 1], state=prev)["tracks"][0]
        assert np.abs(tracks[t] - one).max() <= eps, t
        prev = (tracks[t], visible[t])
    tol = RT.chain_tolerance(ref["tracks"], flow)
    inside = np.ones((h, w), bool)
    worst = 0.0
    for t in range(n):
        x, y = ref["tracks"][t, ..., 0], ref["tracks"][t, ..., 1]
        inside &= (x >= 0) & (x <= w - 1) & (y >= 0) & (y <= h - 1)
        err = np.abs(tracks[t] - ref["tracks"][t])[inside].max(initial=0)
        worst = max(worst, err)
        assert err <= tol[t], (t, err, tol[t])
    total, unexplained = RT.visibility_mismatches(visible, ref, h, w, tol[-1], 2 * tol[-1] + 1e-6)
    print("%dx%d n=%d: step bound %.2e px, chain %.2e px (bound %.2e), visibility differs on %d tracks (all near a "
          "threshold: %s)" % (h, w, n, eps, worst, tol[-1], total, unexplained == 0))
    assert unexplained == 0 and total <= 1e-3 * h * w
    return ref


@pytest.mark.parametrize("n,hw,occ_kind", [(1, (37, 53), "binary"), (3, (37, 53), "none"), (3, (61, 40), "soft"),
                                           (8, (61, 40), "binary"), (8, (37, 53), "none"), (8, (480, 832), "binary")])
def test_kernel_matches_statement(n, hw, occ_kind):
    h, w = hw
    flow, occ = _inputs(n, h, w, occ_kind, seed=n * 7 + h)
    out = chain_tracks(torch.from_numpy(flow).cuda(), None if occ is None else torch.from_numpy(occ).cuda())
    tracks, visible = out["tracks"].cpu().numpy(), out["visible"].cpu().numpy()
    assert tracks.shape == (n, h, w, 2) and visible.dtype == np.uint8 and set(np.unique(visible)) <= {0, 1}
    ref = _check_against_statement(tracks, visible, flow, occ)
    x, y = ref["tracks"][-1, ..., 0], ref["tracks"][-1, ..., 1]
    gone = (x < 0) | (x > w - 1) | (y < 0) | (y > h - 1)
    assert gone.any() and not visible[-1][gone].any()                # tracks that leave the frame stay invisible
    if n > 1:
        assert visible[-1].any()


def test_state_is_carried_in_place():
    """a chain split over calls equals one call bit for bit; the state holds the last step"""
    h, w = 45, 67
    flow, occ = _inputs(8, h, w, "binary", seed=3)
    fd, od = torch.from_numpy(flow).cuda(), torch.from_numpy(occ).cuda()
    whole = chain_tracks(fd, od)
    ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32), indexing="ij")
    pos, vis = torch.stack((xs, ys), -1).cuda(), torch.ones((h, w), dtype=torch.uint8, device="cuda")
    parts = [chain_tracks(fd[a:b], od[a:b], (pos, vis)) for a, b in ((0, 3), (3, 4), (4, 8))]
    assert torch.equal(torch.cat([p["tracks"] for p in parts]), whole["tracks"])
    assert torch.equal(torch.cat([p["visible"] for p in parts]), whole["visible"])
    assert torch.equal(pos, whole["tracks"][-1]) and torch.equal(vis, whole["visible"][-1])


def test_kernel_in_cuda_graph():
    """one launch, no host synchronisation: captured once, replayed on a reset state, it equals the eager call"""
    h, w, n = 64, 96, 4
    flow, occ = _inputs(n, h, w, "binary", seed=5)
    fd, od = torch.from_numpy(flow).cuda(), torch.from_numpy(occ).cuda()
    ref = chain_tracks(fd, od)
    ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32), indexing="ij")
    start = torch.stack((xs, ys), -1).cuda()
    pos, vis = start.clone(), torch.ones((h, w), dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _OPS.chain_tracks(fd, od, pos, vis)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = _OPS.chain_tracks(fd, od, pos, vis)
    for _ in range(2):
        pos.copy_(start)
        vis.fill_(1)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out[0], ref["tracks"]) and torch.equal(out[1], ref["visible"])


def _run(runner, frames):
    return [{k: v.clone() for k, v in r.items()} for r in runner.run(list(frames.numpy()))]


@pytest.mark.parametrize("batch,hw", [(1, (96, 160)), (4, (96, 160)), (3, (80, 48))])
def test_runner_matches_statement(batch, hw):
    """10 frames: 9 steps of one pair, or steps of 4 / 4 / 1 (+3 repeats), or a portrait clip in steps of 3.  The tracks are
    the statement on the runner's own flows and masks bit for bit (fp32), and agree with the float64 statement on
    `infer_flow_video`'s flows and masks within the flows' difference (the encoder's summation order) carried along"""
    m, call = synthetic_model(_WL), workload_call(_WL, drop=("task",))
    pad = WORKLOADS[_WL]["pad"]
    h, w = hw
    frames = synthetic_video(10, h, w, seed=31)
    runner = VideoTrackRunner(m, hw, batch, "cuda", padding_factor=pad, return_flow=True, **call)
    res = _run(runner, frames)
    assert len(res) == 9
    assert all(set(r) == {"flow", "flow_bwd", "fwd_occ", "bwd_occ", "tracks", "visible"} for r in res)
    tracks = torch.stack([r["tracks"] for r in res]).numpy()
    visible = torch.stack([r["visible"] for r in res]).numpy()
    own_flow = torch.stack([r["flow"] for r in res]).numpy()
    own_occ = torch.stack([r["fwd_occ"] for r in res]).numpy()
    emu = RT.chain_tracks(own_flow, own_occ, dtype=np.float32)
    assert np.array_equal(tracks, emu["tracks"], equal_nan=True) and np.array_equal(visible.astype(bool), emu["visible"])

    ifv = infer_flow_video(m, frames.cuda(), padding_factor=pad, pred_bidir_flow=True, fwd_bwd_consistency_check=True, **call)
    flow, occ = ifv["flow"].cpu().numpy(), ifv["fwd_occ"].cpu().numpy()
    ref = RT.chain_tracks(flow, occ)
    dflow = float(np.abs(own_flow - flow).max())
    assert dflow <= 1e-4 * max(1.0, float(np.abs(flow).max()))
    grow = 1.0 + 2.0 * RT.lipschitz(flow)
    eps = RT.step_rounding(ref["tracks"], flow) + dflow
    inside = np.ones((h, w), bool)
    for t in range(9):
        x, y = ref["tracks"][t, ..., 0], ref["tracks"][t, ..., 1]
        inside &= (x >= 0) & (x <= w - 1) & (y >= 0) & (y <= h - 1)
        tol = eps * sum(grow ** k for k in range(t + 1))
        err = np.abs(tracks[t] - ref["tracks"][t])[inside].max(initial=0)
        assert err <= tol, (t, err, tol)
    differ = (visible.astype(bool) != ref["visible"]).any(axis=0).mean()
    masks = float((own_occ != occ).mean())
    print("batch %d %dx%d: flows differ by %.2e px, masks on %.4f %% of pixels, visibility on %.4f %% of tracks; "
          "%.1f %% visible at the end" % (batch, h, w, dflow, 100 * masks, 100 * differ, 100 * ref["visible"][-1].mean()))
    assert differ <= 0.01 + 36 * masks                  # a track reads 4 mask pixels per step for 9 steps


def test_runner_graph_replay_and_reset():
    """tracks with and without graph replay; a second run starts again from the first frame; return_flow=False sends back
    the tracks only"""
    m, call = synthetic_model(_WL), workload_call(_WL, drop=("task",))
    pad = WORKLOADS[_WL]["pad"]
    frames = synthetic_video(7, 64, 96, seed=8)
    out = {}
    for use_graph in (False, True):
        runner = VideoTrackRunner(m, (64, 96), 4, "cuda", padding_factor=pad, use_graph=use_graph, **call)
        out[use_graph] = _run(runner, frames)
        again = _run(runner, frames)
        assert all(set(r) == {"tracks", "visible"} for r in out[use_graph])
        for a, b in zip(out[use_graph], again):
            assert torch.equal(a["tracks"], b["tracks"]) and torch.equal(a["visible"], b["visible"])
    eager, graph = out[False], out[True]
    assert len(eager) == len(graph) == 6
    same = all(torch.equal(a["tracks"], b["tracks"]) and torch.equal(a["visible"], b["visible"]) for a, b in zip(eager, graph))
    diff = max((a["tracks"] - b["tracks"]).abs().max().item() for a, b in zip(eager, graph))
    vis = max((a["visible"] != b["visible"]).float().mean().item() for a, b in zip(eager, graph))
    print("graph vs eager: bit-identical %s, largest track difference %.2e px, visibility on %.4f %% of tracks"
          % (same, diff, 100 * vis))
    assert diff <= 1e-2 and vis <= 0.01


@pytest.mark.parametrize("use_graph", [False, True])
def test_runner_flows_equal_video_flow_runner(use_graph):
    """VideoTrackRunner(return_flow=True) returns what VideoFlowRunner(pred_bidir_flow=True, fwd_bwd_consistency_check=True)
    returns, bit for bit"""
    m, call = synthetic_model(_WL), workload_call(_WL, drop=("task",))
    pad = WORKLOADS[_WL]["pad"]
    frames = synthetic_video(8, 64, 96, seed=9)
    tr = _run(VideoTrackRunner(m, (64, 96), 3, "cuda", padding_factor=pad, use_graph=use_graph, return_flow=True, **call),
              frames)
    fr = _run(VideoFlowRunner(m, (64, 96), 3, "cuda", padding_factor=pad, use_graph=use_graph, pred_bidir_flow=True,
                              fwd_bwd_consistency_check=True, **call), frames)
    assert len(tr) == len(fr) == 7
    for a, b in zip(tr, fr):
        assert set(a) - {"tracks", "visible"} == set(b)
        for k in b:
            assert torch.equal(a[k], b[k]), k
