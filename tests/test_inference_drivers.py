"""The callers' side of the boundary (SURVEY.md section 8f rows 3-4): `infer_flow`, `infer_stereo` (incl. the hflip trick for
right / bidirectional disparity), `infer_depth`, the resize kernel and the batched, graph-replayed runner, against the oracle's
restatements of the reference drivers (evaluate_flow.py:711-792, evaluate_stereo.py:776-836, evaluate_depth.py:360-400).
CPU variants check the host logic through the oracle-backed kernels of tests/refops.py; `-m gpu` variants run the product."""
import pytest
import torch

import cases
import refops
from cases import O
from unimatch_b200.inference import BatchedFlowRunner, infer_depth, infer_flow, infer_stereo
from unimatch_b200.spec import WORKLOADS
from unimatch_b200.synthetic import BENCH_WEIGHTS, synthetic_batch, synthetic_model, synthetic_state_dict, workload_call


def _setup(workload, b, h, w, dev):
    cfg = WORKLOADS[workload]
    sd = synthetic_state_dict(seed=326, **BENCH_WEIGHTS, **cfg["model"])
    data = synthetic_batch(cfg["model"]["task"], b, h, w)
    mk = {k: cfg["model"][k] for k in ("num_scales", "upsample_factor", "reg_refine")}
    call = workload_call(workload, drop=("task",))
    return synthetic_model(workload, dev), sd, {k: v.to(dev) for k, v in data.items()}, data, mk, call


def _stereo_check(dev, bidir, right, size):
    m, sd, d, data, mk, call = _setup("gmstereo-scale2", 1, 100, 150, dev)
    got = infer_stereo(m, d["img0"], d["img1"], padding_factor=32, inference_size=size, pred_bidir_disp=bidir,
                       pred_right_disp=right, **call)
    ref = O.infer_stereo(lambda a, b: O.forward(sd, a, b, task="stereo", **mk, **call)["flow_preds"][-1], data["img0"],
                         data["img1"], 32, size, bidir, right)
    assert set(got) == set(ref)
    for k in ref:
        assert tuple(got[k].shape) == tuple(ref[k].shape) == (1, 100, 150)
        err = (got[k].cpu() - ref[k]).abs()
        assert err.mean().item() <= 2e-2 and err.max().item() <= 2e-1, (k, err.mean().item(), err.max().item())


def _depth_check(dev, bidir):
    m, sd, d, data, mk, call = _setup("gmdepth-scale1-regrefine1", 1, 90, 120, dev)
    kw = {k: v for k, v in call.items() if k not in ("min_depth", "max_depth", "num_depth_candidates")}
    got = infer_depth(m, d["img0"], d["img1"], d["intrinsics"], d["pose"], padding_factor=16, min_depth=0.5, max_depth=10.0,
                      num_depth_candidates=64, pred_bidir_depth=bidir, **kw)

    def fwd(a, b):
        return O.forward(sd, a, b, task="depth", intrinsics=data["intrinsics"], pose=data["pose"], min_depth=1 / 10.0, max_depth=1 / 0.5,
                         num_depth_candidates=64, pred_bidir_depth=bidir, **mk, **kw)["flow_preds"][-1]

    ref = O.infer_depth(fwd, data["img0"], data["img1"], 16, None, bidir)
    assert set(got) == set(ref)
    for k in ref:
        assert tuple(got[k].shape) == tuple(ref[k].shape) == (1, 90, 120)
        err = (got[k].cpu() - ref[k]).abs()
        assert err.mean().item() <= 1e-4 and err.max().item() <= 1e-3, (k, err.mean().item(), err.max().item())


@pytest.mark.parametrize("bidir,right,size", [(False, False, None), (True, False, None), (False, True, (96, 160))])
def test_infer_stereo_host_logic_cpu(bidir, right, size):
    refops.register_cpu_kernels()
    _stereo_check(torch.device("cpu"), bidir, right, size)


@pytest.mark.parametrize("bidir", [False, True])
def test_infer_depth_host_logic_cpu(bidir):
    refops.register_cpu_kernels()
    _depth_check(torch.device("cpu"), bidir)


@pytest.mark.gpu
@pytest.mark.parametrize("bidir,right,size", [(False, False, None), (True, False, None), (False, True, (96, 160))])
def test_infer_stereo_gpu(bidir, right, size):
    _stereo_check(torch.device("cuda", 0), bidir, right, size)


@pytest.mark.gpu
@pytest.mark.parametrize("bidir", [False, True])
def test_infer_depth_gpu(bidir):
    _depth_check(torch.device("cuda", 0), bidir)


@pytest.mark.gpu
@pytest.mark.parametrize("hw,size", [((60, 90), None), ((90, 60), None), ((64, 96), (64, 128))])
def test_infer_flow_gpu(hw, size):
    dev = torch.device("cuda", 0)
    m, sd, d, data, mk, call = _setup("gmflow-scale1", 1, *hw, dev)
    got = infer_flow(m, d["img0"], d["img1"], padding_factor=16, inference_size=size, pred_bidir_flow=True,
                     fwd_bwd_consistency_check=True, **call)
    ref = O.infer_flow(lambda a, b, bd: O.forward(sd, a, b, pred_bidir_flow=bd, task="flow", **mk, **call)["flow_preds"][-1],
                       data["img0"], data["img1"], 16, inference_size=size, pred_bidir_flow=True, fwd_bwd_consistency_check=True)
    for k in ("flow", "flow_bwd"):
        assert tuple(got[k].shape) == tuple(ref[k].shape) == (1, 2, *hw)
        mean, mx = cases.epe(got[k].cpu(), ref[k])
        assert mean <= 1e-2 and mx <= 1e-1, (k, mean, mx)
    for k in ("fwd_occ", "bwd_occ"):
        assert (got[k].cpu() != ref[k]).float().mean().item() < 0.01, k


@pytest.mark.gpu
@pytest.mark.parametrize("shape,out,scale,flip", [((2, 2, 37, 53), (64, 96), [1.5, 0.5], False), ((1, 3, 60, 90), (64, 96), None, False),
                                                  ((2, 1, 48, 80), (48, 80), None, True), ((1, 1, 64, 96), (37, 53), [0.55], True)])
def test_resize_bilinear_kernel(shape, out, scale, flip):
    x = torch.randn(shape, generator=torch.Generator().manual_seed(11)) * 20
    got = torch.ops.unimatch_sm100.resize_bilinear(x.cuda(), out[0], out[1], scale, flip).cpu()
    ref = refops.resize_bilinear(x, out[0], out[1], scale, flip)
    assert got.shape == ref.shape
    assert (got - ref).abs().max().item() <= 1e-5 * max(1.0, ref.abs().max().item())


@pytest.mark.gpu
@pytest.mark.parametrize("use_graph", [False, True])
def test_batched_flow_runner_matches_per_pair_inference(use_graph):
    """5 host pairs of 100x150 through a batch-2 runner (padded to 128x160; the short last batch is filled up): every flow
    equals the module's own output on the padded pair, un-padded."""
    dev = torch.device("cuda", 0)
    m, sd, _, _, mk, call = _setup("gmflow-scale2", 1, 64, 64, dev)
    pairs = []
    for i in range(5):
        p = synthetic_batch("flow", 1, 100, 150, first_index=10 + i)
        pairs.append((p["img0"][0], p["img1"][0]))
    runner = BatchedFlowRunner(m, (100, 150), 2, dev, padding_factor=32, use_graph=use_graph, **call)
    flows = [f.clone() for f in runner.run(pairs)]
    assert len(flows) == 5 and all(tuple(f.shape) == (2, 100, 150) for f in flows)
    for (a, b), f in zip(pairs, flows):
        pa, pb = runner.padder.pad(a[None].cuda(), b[None].cuda())
        ref = runner.padder.unpad(m(pa, pb, task="flow", **call)["flow_preds"][-1])[0].cpu()
        assert (f - ref).abs().max().item() <= 1e-4 * max(1.0, ref.abs().max().item())
