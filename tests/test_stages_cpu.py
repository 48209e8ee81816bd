"""The teacher-forced stage harness (tests/stage_checks.py) on the CPU at small shapes, with the oracle-backed CPU kernels of
tests/refops*.py standing in for the CUDA ops: checks the harness itself and the host orchestration of every
`UniMatch._stage_*` method, for every workload and both bidirectional modes.  The CUDA kernels take the same harness at the
bench resolutions in tests/test_stages_gpu.py.

The defect tests give the harness its teeth: each injects one plausible host-side mistake (a sign, an operand order, a
channel offset, a factor, a stream order) by wrapping the op table the module calls, and shows that the check of the stage
it belongs to fails -- and names that stage -- while every stage before it still passes, as teacher forcing promises."""
import functools

import pytest
import torch

import refops
import stage_checks
import unimatch_b200.unimatch as um
from unimatch_b200 import UniMatch
from unimatch_b200.spec import WORKLOADS


def small_shape(workload, bidir):
    return (96, 128) if bidir and workload.startswith("gmdepth") else (128, 192)


def run_small(workload, bidir):
    refops.register_cpu_kernels()
    res = stage_checks.run(torch.device("cpu"), workload, *small_shape(workload, bidir), bidir, report=lambda *_: None)
    assert "e2e" in res and all(v <= 1 for v in res.values())


def test_stage_harness_small_shape_on_cpu():
    run_small("gmflow-scale2-regrefine6", False)


@pytest.mark.parametrize("workload,bidir", [c for c in stage_checks.CASES if c != ("gmflow-scale2-regrefine6", False)])
def test_stage_harness_every_workload_small_shape_on_cpu(workload, bidir):
    run_small(workload, bidir)


def test_end_to_end_tolerance_of_every_workload_is_bench_tolerance():
    tol = {wl: stage_checks.e2e_tol(wl)[:2] for wl in WORKLOADS}
    assert tol["gmflow-scale2-regrefine6"] == tol["gmflow-scale1"] == (stage_checks.E2E_MEAN, stage_checks.E2E_MAX)
    assert tol["gmflow-scale2"] == tol["gmflow-scale1"]                      # not in the bench: the flow task's tolerance
    assert tol["gmstereo-scale2-regrefine3"] == tol["gmstereo-scale2"] == (2e-2, 2e-1)
    assert tol["gmdepth-scale1"] == tol["gmdepth-scale1-regrefine1"] == (1e-4, 1e-3)


# ---- defects, injected by wrapping the op table the module (and the harness) calls ---------------------------------------
class OpDefect:
    """Delegates to the op table `real`, except for op `name`, which becomes `hook(real_op, *args)`."""

    def __init__(self, real, name, hook):
        self.real, self.name, self.hook = real, name, hook

    def __getattr__(self, name):
        fn = getattr(self.real, name)
        return functools.partial(self.hook, fn) if name == self.name else fn


def _warp_disp_negated(fn, f, flow, h, w):
    return fn(f, -flow if flow.shape[-1] == 1 else flow, h, w)


def _corr_volume_disp_negated(fn, f0, f1, flow, h, w, r):
    return fn(f0, f1, -flow if flow.shape[-1] == 1 else flow, h, w, r)


def _depth_K_Kinv_swapped(fn, f0, f1, K, K_inv, pose, *rest):
    return fn(f0, f1, K_inv, K, pose, *rest)


def _depth_halves_swapped(fn, *a):
    out = fn(*a)
    n = out.shape[0] // 2
    return torch.cat((out[n:], out[:n]), 0)


def _upsampler_flow_at_0(fn, src, dst, off):
    """the flow channels of the learned upsampler's [feature | flow] planes written over the feature's first channels"""
    return fn(src, dst, 0 if off == 128 and dst.shape[-1] == 192 else off)


def _convex_mult_1(fn, flow, mask, factor, mult):
    return fn(flow, mask, factor, 1.0)


def _ops(name, hook):
    return lambda mp: mp.setattr(um, "_OPS", OpDefect(um._OPS, name, hook))


def _rigid_flow_pose_inverted(mp):
    rigid = UniMatch._rigid_flow
    mp.setattr(UniMatch, "_rigid_flow", staticmethod(
        lambda inv_depth, K, K_inv, pose, h, w: rigid(inv_depth, K, K_inv, torch.inverse(pose), h, w)))


# name -> (workload, bidir, stage that must fail, a stage before it that must pass, patch(monkeypatch))
DEFECTS = {
    "stereo_warp_disparity_sign": ("gmstereo-scale2", False, "s1.warp", "s0.propagation",
                                   _ops("flow_warp", _warp_disp_negated)),
    "stereo_refine_corr_disparity_sign": ("gmstereo-scale2-regrefine3", False, "refine0", "s1.propagation",
                                          _ops("local_corr_volume", _corr_volume_disp_negated)),
    "depth_corr_K_Kinv_swapped": ("gmdepth-scale1", False, "s0.correlation", "s0.transformer.view1",
                                  _ops("depth_corr_softmax", _depth_K_Kinv_swapped)),
    "rigid_flow_pose_inverted": ("gmdepth-scale1-regrefine1", False, "rigid_flow0", "s0.propagation",
                                 _rigid_flow_pose_inverted),
    "upsampler_flow_at_offset_0": ("gmdepth-scale1", False, "upsample", "s0.propagation",
                                   _ops("split_planes", _upsampler_flow_at_0)),
    "upsampler_mult_1": ("gmflow-scale1", False, "upsample", "s0.propagation", _ops("convex_upsample", _convex_mult_1)),
    "bidir_depth_halves_swapped": ("gmdepth-scale1-regrefine1", True, "s0.correlation", "s0.transformer.view1",
                                   _ops("depth_corr_softmax", _depth_halves_swapped)),
}


@pytest.mark.parametrize("defect", sorted(DEFECTS))
def test_stage_check_catches_defect_at_its_stage(monkeypatch, defect):
    workload, bidir, stage, before, patch = DEFECTS[defect]
    refops.register_cpu_kernels()
    patch(monkeypatch)
    res = {}
    with pytest.raises(AssertionError) as e:
        stage_checks.run(torch.device("cpu"), workload, *small_shape(workload, bidir), bidir, report=lambda *_: None, res=res)
    print("%s rejected: %s" % (defect, e.value))
    assert str(e.value).startswith(stage + ":"), str(e.value)
    assert list(res)[-1] == stage and res[stage] > 1
    assert before in res and all(v <= 1 for k, v in res.items() if k != stage)
