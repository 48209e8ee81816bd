"""Dense point tracks without a device: the statement (tests/refops_tracks.py) against the reference's own `flow_warp` and
`forward_backward_consistency_check` iterated over a few steps, the fp32 order of operations against the statement within
its rounding bound, and the refusals of `um_chain_tracks`, `chain_tracks` and `VideoTrackRunner` before any device work."""
import ctypes
import importlib.util
import os

import numpy as np
import pytest
import torch

import refops_tracks as RT
from unimatch_b200 import ops
from unimatch_b200.inference import VideoTrackRunner, chain_tracks

REFERENCE = os.environ.get("UNIMATCH_REFERENCE", "/root/reference")
needs_reference = pytest.mark.skipif(not os.path.isfile(os.path.join(REFERENCE, "unimatch", "geometry.py")),
                                     reason="the reference tree is not available (set UNIMATCH_REFERENCE)")


def _reference_geometry():
    spec = importlib.util.spec_from_file_location("reference_geometry", os.path.join(REFERENCE, "unimatch", "geometry.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@needs_reference
@pytest.mark.parametrize("n,hw,drift", [(3, (23, 31), (1.5, 0.5)), (5, (40, 28), (-2.0, 3.0)), (4, (30, 30), (0.0, 0.0))])
def test_statement_equals_reference_iterated(n, hw, drift):
    """p_t = p_{t-1} + flow_warp(F, p_{t-1} - grid), o = flow_warp(fwd_occ, p_{t-1} - grid) with the reference's functions in
    float64, fwd_occ from its forward_backward_consistency_check on a forward and a backward flow per step"""
    G = _reference_geometry()
    h, w = hw
    fwd = torch.from_numpy(RT.smooth_flows(n, h, w, 1.0, seed=n, drift=drift)).double()
    bwd = -fwd + torch.from_numpy(RT.smooth_flows(n, h, w, 0.3, seed=n + 100)).double()
    occ = torch.cat([G.forward_backward_consistency_check(fwd[t:t + 1], bwd[t:t + 1])[0] for t in range(n)]).double()
    assert 0 < occ.mean() < 1
    grid = G.coords_grid(1, h, w).double()
    p, vis = grid.clone(), torch.ones((1, h, w), dtype=torch.bool)
    ref_p, ref_v = [], []
    for t in range(n):
        d = G.flow_warp(fwd[t:t + 1], p - grid)
        o = G.flow_warp(occ[t:t + 1, None], p - grid)[:, 0]
        p = p + d
        vis = vis & (o < 0.5) & (p[:, 0] >= 0) & (p[:, 0] <= w - 1) & (p[:, 1] >= 0) & (p[:, 1] <= h - 1)
        ref_p.append(p[0].permute(1, 2, 0).numpy())
        ref_v.append(vis[0].numpy())
    got = RT.chain_tracks(fwd.numpy(), occ.numpy())
    ref_p = np.stack(ref_p)
    assert np.abs(got["tracks"] - ref_p).max() <= 1e-9
    left = ~got["visible"][-1] & ref_v[0]
    assert left.any() and got["visible"][-1].any()                   # some tracks leave or get occluded, some stay
    total, unexplained = RT.visibility_mismatches(np.stack(ref_v), got, h, w, 1e-9, 1e-9)
    assert unexplained == 0 and total <= 1, total


def test_statement_without_occlusion_and_start():
    """occ None: only the frame decides; zero flow keeps every track where it started"""
    h, w = 9, 13
    got = RT.chain_tracks(np.zeros((2, 2, h, w), np.float32))
    start, _ = RT.track_start(h, w)
    assert np.array_equal(got["tracks"][1], start) and got["visible"].all()
    shift = np.zeros((1, 2, h, w), np.float32)
    shift[:, 0] = 2.25
    got = RT.chain_tracks(shift)
    assert np.array_equal(got["tracks"][0][..., 0], start[..., 0] + 2.25)
    assert np.array_equal(got["visible"][0], start[..., 0] + 2.25 <= w - 1)


@pytest.mark.parametrize("n,hw", [(1, (37, 53)), (3, (61, 40)), (8, (37, 53)), (8, (96, 160))])
def test_fp32_order_within_rounding_of_statement(n, hw):
    """The kernel's fp32 expression (refops_tracks with float32) stays within the rounding bound of the float64 statement:
    every step from the same start, and the whole chain for tracks whose path stays inside the frame"""
    h, w = hw
    flow = RT.smooth_flows(n, h, w, 3.0, seed=7, drift=(2.5, -1.5))
    occ = (np.random.default_rng(8).random((n, h, w)) < 0.2).astype(np.float32)
    ref = RT.chain_tracks(flow, occ)
    got = RT.chain_tracks(flow, occ, dtype=np.float32)
    prev = RT.track_start(h, w, np.float32)
    eps = RT.step_rounding(ref["tracks"], flow)
    for t in range(n):
        one = RT.chain_tracks(flow[t:t + 1], occ[t:t + 1], state=prev)["tracks"][0]
        assert np.abs(got["tracks"][t] - one).max() <= eps, t
        prev = (got["tracks"][t], got["visible"][t])
    tol = RT.chain_tolerance(ref["tracks"], flow)
    inside = np.ones((h, w), bool)
    for t in range(n):
        x, y = ref["tracks"][t, ..., 0], ref["tracks"][t, ..., 1]
        inside &= (x >= 0) & (x <= w - 1) & (y >= 0) & (y <= h - 1)
        assert np.abs(got["tracks"][t] - ref["tracks"][t])[inside].max(initial=0) <= tol[t], t
    total, unexplained = RT.visibility_mismatches(got["visible"], ref, h, w, tol[-1], 2 * tol[-1] + 1e-6)
    assert unexplained == 0 and total <= 1e-3 * h * w, total


def test_c_abi_refusals_without_a_gpu():
    """um_chain_tracks checks its arguments before any CUDA call"""
    a, b, c, d, e = (ctypes.c_void_p(1 << 20), ctypes.c_void_p(2 << 20), ctypes.c_void_p(3 << 20), ctypes.c_void_p(4 << 20),
                     ctypes.c_void_p(5 << 20))
    ok = dict(flow=a, occ=None, n=2, h=8, w=8, pos=b, vis=c, pos_out=d, vis_out=e)
    bad = [dict(flow=None), dict(pos=None), dict(vis=None), dict(pos_out=None), dict(vis_out=None), dict(n=0), dict(n=-1),
           dict(h=1), dict(w=0), dict(h=1 << 16, w=1 << 16), dict(pos=ctypes.c_void_p((2 << 20) + 4)),
           dict(pos_out=ctypes.c_void_p((2 << 20) + 8)), dict(vis=ctypes.c_void_p((2 << 20) + 16))]
    for change in bad:
        args = dict(ok, **change)
        rc = ops.LIB.um_chain_tracks(args["flow"], args["occ"], args["n"], args["h"], args["w"], args["pos"], args["vis"],
                                     args["pos_out"], args["vis_out"], None)
        assert rc == -22, change
        assert b"um_chain_tracks" in ops.LIB.um_last_error(), change


def test_chain_tracks_shape_refusals():
    flow = torch.zeros((2, 2, 6, 7))
    for args in [(torch.zeros((2, 3, 6, 7)),), (torch.zeros((0, 2, 6, 7)),), (torch.zeros((2, 6, 7)),),
                 (flow, torch.zeros((2, 6, 6))), (flow, torch.zeros((1, 6, 7))),
                 (flow, None, (torch.zeros((6, 7, 2)), torch.ones((7, 6), dtype=torch.uint8))),
                 (flow, None, (torch.zeros((7, 6, 2)), torch.ones((6, 7), dtype=torch.uint8)))]:
        with pytest.raises(ValueError):
            chain_tracks(*args)
    with pytest.raises(RuntimeError):                                 # no CPU kernel: the op refuses host tensors
        chain_tracks(flow)


@pytest.mark.parametrize("flag", [dict(pred_bwd_flow=True), dict(visualize=True), dict(concat_frame=True),
                                  dict(visualize_bwd=True), dict(pred_bidir_flow=False),
                                  dict(fwd_bwd_consistency_check=False)])
def test_runner_refused_flags(flag):
    with pytest.raises(ValueError):
        VideoTrackRunner(None, (32, 48), 2, "cuda", **flag)
