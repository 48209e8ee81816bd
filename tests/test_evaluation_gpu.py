"""Validation on the device: `um_eval_stats` against its CPU statement (tests/refops_eval.py) on edge cases, odd and large
sizes and strided views, bit-reproducible and graph-capturable; the golden protocols through the CUDA op; the drivers around
the real module against the reference loop restated at batch 1 (tests/refloop_eval.py); and no host synchronisation in the flow and stereo drivers."""
import math

import pytest
import torch

import eval_samples as E
import refloop_eval
import refops_eval
from test_evaluation_cpu import GOLDEN, check_results, run_case
from unimatch_b200 import UniMatch, evaluation, ops
from unimatch_b200.spec import WORKLOADS
from unimatch_b200.synthetic import BENCH_WEIGHTS, synthetic_state_dict

pytestmark = pytest.mark.gpu
OPS = torch.ops.unimatch_sm100
COUNT_COLS = {"n", "1px", "2px", "3px", "5px", "outlier", "d1", "a1", "a2", "a3", "s0_10_n", "s10_40_n", "s40_n", "matched_n",
              "unmatched_n"}


def _flow_case(g, b, h, w, scale=6.0):
    """pred on a 1/8 grid (exact epe on thresholds where pred - gt is (1, 0), (0, 3), (3, 4)), zero-magnitude GT, bin edges."""
    gt = torch.randn((b, 2, h, w), generator=g) * scale
    delta = torch.randn((b, 2, h, w), generator=g) * 2.0
    kind = torch.randint(0, 5, (b, h, w), generator=g)
    for k, (du, dv) in ((1, (1.0, 0.0)), (2, (0.0, 3.0)), (3, (3.0, 4.0))):
        delta[:, 0][kind == k], delta[:, 1][kind == k] = du, dv
    gt = torch.round(gt * 8) / 8
    gt[:, :, : max(h // 5, 1), : max(w // 7, 1)] = 0.0
    if h > 2:
        gt[:, 0, 1], gt[:, 1, 1] = 10.0, 0.0
        gt[:, 0, 2], gt[:, 1, 2] = 24.0, 32.0                          # magnitude exactly 40
    pred = gt + delta
    valid = (torch.rand((b, h, w), generator=g) < 0.7).float()
    noc = (torch.rand((b, h, w), generator=g) < 0.8).float()
    return pred, gt, valid, noc


def _compare(task, pred, gt, valid, noc, mask_mode=0, max_val=0.0, emin=0.0, emax=0.0, pad=None):
    ref = refops_eval.eval_stats(pred, gt, valid, noc, task, mask_mode, max_val, emin, emax)
    dpred = pred.cuda()
    if pad is not None:                                  # the same values as an unpadded view of a larger buffer
        big = torch.full(pred.shape[:-2] + (pred.shape[-2] + 2 * pad, pred.shape[-1] + 3 * pad), float("nan"), device="cuda")
        big[..., pad:pad + pred.shape[-2], pad:pad + pred.shape[-1]] = dpred
        dpred = big[..., pad:pad + pred.shape[-2], pad:pad + pred.shape[-1]]
        assert not dpred.is_contiguous()
    c = lambda t: None if t is None else t.cuda()  # noqa: E731
    got = OPS.eval_stats(dpred, gt.cuda(), c(valid), c(noc), task, mask_mode, max_val, emin, emax)
    again = OPS.eval_stats(dpred, gt.cuda(), c(valid), c(noc), task, mask_mode, max_val, emin, emax)
    assert torch.equal(got, again), "two launches differ"
    got = got.cpu()
    for j, name in enumerate(ops.EVAL_COLS[task]):
        if name in COUNT_COLS:
            assert torch.equal(got[:, j], ref[:, j]), (name, got[:, j], ref[:, j])
        else:
            # log_sq: logf and numpy's float32 log may differ by 1 ulp per pixel
            rtol = 1e-6 if name == "log_sq" else 1e-12
            assert torch.allclose(got[:, j], ref[:, j], rtol=rtol, atol=0.0), (name, got[:, j], ref[:, j])
    return got


@pytest.mark.parametrize("b,h,w", [(3, 37, 53), (1, 1, 1), (2, 64, 96), (4, 75, 130)])
@pytest.mark.parametrize("mask_mode", [ops.EVAL_MASK_ALL, ops.EVAL_MASK_VALID, ops.EVAL_MASK_VALID_MAX])
def test_flow_stats_match_cpu_statement(b, h, w, mask_mode):
    g = torch.Generator().manual_seed(b * 1000 + h * 10 + mask_mode)
    pred, gt, valid, noc = _flow_case(g, b, h, w)
    valid[0] = 0.0 if b > 1 else valid[0]                 # an empty mask
    _compare(ops.EVAL_FLOW, pred, gt, valid if mask_mode else None, noc, mask_mode, 8.0, pad=3)
    _compare(ops.EVAL_FLOW, pred, gt, valid if mask_mode else None, None, mask_mode, 8.0)


def test_stereo_and_depth_stats_match_cpu_statement():
    g = torch.Generator().manual_seed(7)
    b, h, w = 3, 45, 77
    pred = torch.floor(torch.rand((b, h, w), generator=g) * 80)
    gt = pred + torch.randint(-4, 5, (b, h, w), generator=g).float()
    gt[:, 0, :] = 60.0                                     # e / gt exactly 0.05 where pred = 57 / 63
    gt[:, 1, :] = 0.0
    gt[1] = -1.0                                           # empty mask
    for max_val in (0.0, 50.0):
        _compare(ops.EVAL_STEREO, pred, gt, None, None, 0, max_val, pad=2)
    dpred = 1.0 + torch.floor(torch.rand((b, h, w), generator=g) * 16) * 0.25
    dgt = dpred * torch.tensor([1.0, 1.25, 1.5625, 1.953125, 0.8, 2.0])[torch.randint(0, 6, (b, h, w), generator=g)]
    dgt[:, 0, :], dgt[:, 1, :] = 0.5, 10.0                 # on the range bounds
    valid = (torch.rand((b, h, w), generator=g) < 0.9).float()
    _compare(ops.EVAL_DEPTH, dpred, dgt, valid, None, 0, 0.0, 0.5, 10.0, pad=1)
    _compare(ops.EVAL_DEPTH, dpred, dgt, None, None, 0, 0.0, 0.5, 10.0)


def test_large_batch_many_ctas():
    g = torch.Generator().manual_seed(11)
    pred, gt, valid, noc = _flow_case(g, 8, 1080, 1920, scale=20.0)
    _compare(ops.EVAL_FLOW, pred, gt, valid, noc, ops.EVAL_MASK_VALID_MAX, 50.0)


def test_graph_capture_matches_eager():
    g = torch.Generator().manual_seed(5)
    pred, gt, valid, noc = [t.cuda() for t in _flow_case(g, 4, 240, 320)]
    args = (ops.EVAL_FLOW, ops.EVAL_MASK_VALID, 0.0, 0.0, 0.0)
    eager = OPS.eval_stats(pred, gt, valid, noc, *args)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        OPS.eval_stats(pred, gt, valid, noc, *args)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = OPS.eval_stats(pred, gt, valid, noc, *args)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(captured, eager)


@pytest.mark.parametrize("case", GOLDEN, ids=[c["name"] for c in GOLDEN])
def test_golden_protocols_on_device(case):
    build = {name: b for name, _, _, b in E.CASES}[case["name"]]
    samples = build()
    got = run_case(case, samples, batch=3, device="cuda")
    check_results(got, case["results"])


# ------------------------------------------------------------------------------------------------ end to end, real module
def _model(name):
    cfg = WORKLOADS[name]
    m = UniMatch(**cfg["model"]).eval()
    m.load_state_dict(synthetic_state_dict(seed=326, **BENCH_WEIGHTS, **cfg["model"]), strict=True)
    kw = {k: v for k, v in cfg["call"].items() if k not in ("min_depth", "max_depth")}
    return m.cuda(), kw


def _e2e(task, workload, samples, opts):
    """The driver at batch 3 (short batches, two shapes) against the reference loop restated at batch 1 around the same module
    (tests/refloop_eval.py).  Batch composition changes `um_conv2d_tc`'s summation order, hence the tolerances."""
    model, kw = _model(workload)
    want = refloop_eval.LOOPS[task](model, samples, **opts, **kw)
    driver = {"flow": evaluation.validate_flow, "stereo": evaluation.validate_stereo, "depth": evaluation.validate_depth}[task]
    got = driver(model, samples, batch=3, device="cuda", **opts, **kw)
    check_results(got, want, sum_rtol=1e-4, ratio_atol=1e-3)
    return got


def test_validate_flow_end_to_end():
    sintel = E.flow_samples(51, [(96, 128), (80, 112)], 7, noc=True)
    _e2e("flow", "gmflow-scale2-regrefine6", sintel,
         dict(protocol="sintel", padding_factor=32, with_speed_metric=True, evaluate_matched_unmatched=True))
    kitti = E.flow_samples(52, [(96, 128), (88, 120)], 7, sparse=True)
    _e2e("flow", "gmflow-scale2-regrefine6", kitti, dict(protocol="kitti", padding_factor=32, with_speed_metric=True))


@pytest.mark.parametrize("inference_size", [None, (96, 160)])
def test_validate_stereo_end_to_end(inference_size):
    samples = E.stereo_samples(53, [(96, 128), (80, 144)], 7)
    _e2e("stereo", "gmstereo-scale2", samples,
         dict(protocol="kitti15", padding_factor=32, inference_size=inference_size))


@pytest.mark.parametrize("inference_size", [None, (96, 160)])
def test_validate_depth_end_to_end(inference_size):
    samples = E.depth_samples(54, [(96, 128), (88, 120)], 7)          # 88x120 is padded: 'kitti' mode puts all 8 rows below
    _e2e("depth", "gmdepth-scale1-regrefine1", samples,
         dict(protocol="scannet", padding_factor=16, inference_size=inference_size))


def test_flow_and_stereo_drivers_do_not_synchronise():
    flow_model, flow_kw = _model("gmflow-scale2-regrefine6")
    stereo_model, stereo_kw = _model("gmstereo-scale2")
    flow = E.flow_samples(55, [(96, 128), (80, 112)], 5, sparse=True)
    stereo = E.stereo_samples(56, [(96, 128)], 4)
    runs = [lambda: evaluation.validate_flow(flow_model, flow, protocol="kitti", padding_factor=32, batch=3, **flow_kw),
            lambda: evaluation.validate_stereo(stereo_model, stereo, protocol="kitti15", padding_factor=32, batch=3,
                                               inference_size=(96, 160), **stereo_kw)]
    for run in runs:
        want = run()                                     # warm-up: module caches are built outside the checked run
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            got = run()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        assert got == want or all(math.isclose(got[k], want[k], rel_tol=1e-12) for k in want)
