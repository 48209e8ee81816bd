"""Host-logic tests (no GPU): the drop-in module's orchestration, run on CPU by installing the oracle-backed
CPU kernels of tests/refops.py for the custom ops, must reproduce the REFERENCE outputs stored in
tests/golden/golden.pt for every workload (flow / stereo / depth, 1-2 scales, refinement, bidirectional).
This checks everything the CUDA kernels do not: layouts, stream pairing (kv_shift), the static attention
dispatch, hoisted refinement work, sign conventions, output shapes."""
import os
import subprocess
import sys

import pytest
import torch

import cases
import refops
from unimatch_b200 import UniMatch, param_spec
from unimatch_b200.spec import WORKLOADS

GOLD = torch.load(os.path.join(os.path.dirname(__file__), "golden", "golden.pt"))["vectors"]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_state_dict_layout_matches_spec():
    for wl in WORKLOADS.values():
        m = UniMatch(**wl["model"])
        spec = param_spec(**wl["model"])
        sd = m.state_dict()
        assert list(sd.keys()) == list(spec.keys())
        assert all(tuple(sd[k].shape) == tuple(spec[k]) for k in spec)


def test_param_counts_match_reference():
    # SURVEY.md §8b (measured on the reference): flow s1 / stereo s2 / flow s2 rr / depth rr
    count = lambda **kw: sum(torch.Size(s).numel() for s in param_spec(**kw).values())
    assert count() == 4680288
    assert count(num_scales=2, upsample_factor=4, task="stereo") == 4716720
    assert count(num_scales=2, upsample_factor=4, reg_refine=True) == 7360688
    assert count(num_scales=1, upsample_factor=8, reg_refine=True, task="depth") == 7322592


def test_inference_only():
    m = UniMatch()
    assert not m.training
    with pytest.raises(NotImplementedError):
        m.train()
    m.eval()


def test_no_cpu_fallback_in_product():
    """Outside the test harness the ops have no CPU kernel: a CPU call must fail loudly."""
    code = ("import torch, unimatch_b200.ops\n"
            "try:\n"
            "    torch.ops.unimatch_sm100.upsample2x(torch.zeros(1,2,2,2), 2.0)\n"
            "except NotImplementedError as e:\n"
            "    print('LOUD')\n")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=300)
    assert "LOUD" in r.stdout, r.stdout + r.stderr


@pytest.mark.parametrize("name", sorted(cases.E2E_CASES))
def test_module_matches_reference_on_cpu(name):
    refops.register_cpu_kernels()
    cfg, sd, batch, call = cases.e2e_setup(name)
    m = UniMatch(**cfg["model"]).eval()
    res = m.load_state_dict(sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    out = m(batch["img0"], batch["img1"], intrinsics=batch.get("intrinsics"), pose=batch.get("pose"), **call)
    assert isinstance(out, dict) and list(out) == ["flow_preds"] and len(out["flow_preds"]) == 1
    got, ref = out["flow_preds"][-1], GOLD[name]
    assert got.shape == ref.shape and got.dtype == torch.float32
    mean, mx = cases.epe(got, ref)
    assert mean <= cases.e2e_tolerance(name), (mean, mx)



def test_cpu_statements_are_named_after_defined_ops():
    """Every CPU statement of the registry is installed under the name of an op that unimatch_b200/ops.py defines, so a
    misspelt or removed name fails here rather than only in a test that happens to call that op."""
    from unimatch_b200 import ops  # noqa: F401  defines the unimatch_sm100 ops
    unknown = [name for name in refops.cpu_statements() if not hasattr(torch.ops.unimatch_sm100, name)]
    assert not unknown, unknown
