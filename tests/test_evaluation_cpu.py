"""Validation drivers without a device: every protocol and option of tests/golden/golden_eval.pt (the reference's own
validate_* loops on seeded samples with a stub model) is reproduced through the CPU statement of `eval_stats`, at several
batch sizes; the C entry rejects bad arguments before touching a device."""
import ctypes
import math
import os

import pytest
import torch

import eval_samples as E
import refloop_eval
import refops
from unimatch_b200 import evaluation, ops

GOLDEN = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_eval.pt"), weights_only=False)
RATIOS = ("_1px", "_2px", "_3px", "_5px", "_d1", "_f1", "a1", "a2", "a3")
DRIVERS = {"flow": evaluation.validate_flow, "stereo": evaluation.validate_stereo, "depth": evaluation.validate_depth}


def check_results(got, want, sum_rtol=1e-6, ratio_atol=0.0):
    """Ratios of counts exactly (or within `ratio_atol`), sums within `sum_rtol` relative (the reference sums in float32)."""
    assert sorted(got) == sorted(want)
    for k, v in want.items():
        if k.endswith(RATIOS):
            assert abs(got[k] - v) <= ratio_atol, (k, got[k], v)
        else:
            assert math.isclose(got[k], v, rel_tol=sum_rtol, abs_tol=0.0), (k, got[k], v)


def run_case(case, samples, **kw):
    return DRIVERS[case["task"]](E.STUB, samples, **case["options"], **kw)


@pytest.fixture(scope="module", autouse=True)
def _cpu_kernels():
    refops.register_cpu_kernels()


@pytest.mark.parametrize("case", GOLDEN, ids=[c["name"] for c in GOLDEN])
def test_golden_protocols_on_cpu(case):
    build = {name: b for name, _, _, b in E.CASES}[case["name"]]
    samples = build()
    assert E.digest(samples) == case["digest"], "eval_samples.py no longer builds the golden samples"
    results = [run_case(case, samples, batch=b, device="cpu") for b in (1, 3, 8)]
    check_results(results[0], case["results"])
    assert results[0] == results[1] == results[2]


@pytest.mark.parametrize("case", GOLDEN, ids=[c["name"] for c in GOLDEN])
def test_restated_reference_loops_reproduce_golden(case):
    """tests/refloop_eval.py, which the device tests and tools/eval_bench.py compare the drivers against, IS the reference loop:
    with the stub model it gives the reference's results dicts to the last bit."""
    build = {name: b for name, _, _, b in E.CASES}[case["name"]]
    got = refloop_eval.LOOPS[case["task"]](E.STUB, build(), device="cpu", **case["options"])
    assert sorted(got) == sorted(case["results"])
    for k, v in case["results"].items():
        assert math.isclose(got[k], v, rel_tol=1e-12), (k, got[k], v)


def test_driver_arguments():
    with pytest.raises(ValueError):
        evaluation.validate_flow(E.STUB, [], protocol="spring", device="cpu")
    with pytest.raises(ValueError):
        evaluation.validate_stereo(E.STUB, [], protocol="kitti", device="cpu")
    with pytest.raises(ValueError):
        evaluation.validate_depth(E.STUB, [], protocol="scannet", batch=0, device="cpu")
    with pytest.raises(ValueError):
        evaluation.validate_flow(E.STUB, E.flow_samples(1, [(16, 24)], 1), protocol="sintel",
                                 evaluate_matched_unmatched=True, device="cpu")


def _stats(**kw):
    one = ctypes.c_void_p(1024)                    # any non-null address: validation never dereferences it
    a = dict(pred=one, sb=2 * 8 * 16, sc=8 * 16, sy=16, sx=1, gt=one, valid=one, noc=None, task=ops.EVAL_FLOW,
             mask=ops.EVAL_MASK_VALID, b=2, h=8, w=16, scratch=one, out=one)
    a.update(kw)
    return ops.LIB.um_eval_stats(a["pred"], a["sb"], a["sc"], a["sy"], a["sx"], a["gt"], a["valid"], a["noc"], a["task"],
                                 a["mask"], 400.0, 0.5, 10.0, a["b"], a["h"], a["w"], a["scratch"], a["out"], None)


def test_eval_stats_validation_without_a_gpu():
    """um_eval_stats rejects bad arguments with -EINVAL and a message before touching the device."""
    bad = [dict(pred=None), dict(gt=None), dict(scratch=None), dict(out=None),      # null pointers
           dict(task=3), dict(task=-1), dict(mask=3), dict(valid=None),              # bad task / mask mode, missing mask
           dict(task=ops.EVAL_STEREO, noc=ctypes.c_void_p(1024)),                   # noc_valid is flow-only
           dict(b=0), dict(h=0), dict(w=-1), dict(b=70000), dict(h=50000, w=50000),  # bad sizes
           dict(sx=0), dict(sx=-1), dict(sy=15), dict(sc=16), dict(sb=8 * 16)]       # bad strides (overlapping views)
    for kw in bad:
        assert _stats(**kw) == -22, kw
        assert b"um_eval_stats" in ops.LIB.um_last_error(), kw
