"""Without a GPU: the driver size table (tests/driver_sizes.py) against the drivers' own size rule and the model's
divisibility rules, the launch replay's closed op table, its signatures and dedupe, and its copy of the inputs before the
call (tests/launch_replay.py), on the CPU statements of the ops (tests/refops.py)."""
import os
import re

import pytest
import torch

import driver_sizes
import launch_replay as LR
import refops
from unimatch_b200 import ops
from unimatch_b200.inference import _inference_size
from unimatch_b200.spec import WORKLOADS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- the size table ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", driver_sizes.CASES, ids=driver_sizes.case_id)
def test_driver_size_is_the_drivers_inference_size(case):
    assert _inference_size(case.raw, case.padding, case.inference_size) == (case.H, case.W), case.origin
    assert case.origin


@pytest.mark.parametrize("case", driver_sizes.CASES, ids=driver_sizes.case_id)
def test_driver_size_obeys_the_model_divisibility_rules(case):
    """scale s works at 1/8 / 2^s of the input; its map must split into attn_splits_list[s] windows both ways"""
    cfg = WORKLOADS[case.workload]
    assert case.bidir is False or cfg["model"]["task"] in ("flow", "depth")
    for s, splits in enumerate(cfg["call"]["attn_splits_list"]):
        f = 8 // 2 ** s
        assert case.H % f == 0 and case.W % f == 0, (case, f)
        assert (case.H // f) % splits == 0 and (case.W // f) % splits == 0, (case, s, splits)


def test_driver_sizes_cover_every_workload_and_mode_named_by_the_drivers():
    have = {(c.workload, c.H, c.W, c.bidir) for c in driver_sizes.CASES}
    for need in [("gmflow-scale2-regrefine6", 416, 1024, False), ("gmflow-scale2-regrefine6", 352, 1216, False),
                 ("gmflow-scale2-regrefine6", 384, 1248, False), ("gmflow-scale1", 448, 1024, False),
                 ("gmstereo-scale2-regrefine3", 352, 1216, False), ("gmstereo-scale2-regrefine3", 1024, 1536, False),
                 ("gmstereo-scale2-regrefine3", 512, 768, False), ("gmstereo-scale2", 384, 1248, False),
                 ("gmdepth-scale1", 480, 640, False), ("gmdepth-scale1-regrefine1", 480, 640, False),
                 ("gmdepth-scale1-regrefine1", 480, 640, True)]:
        assert need in have, need
    assert any(c.workload == "gmflow-scale2-regrefine6" and c.bidir for c in driver_sizes.CASES)


# ---- the closed op table -------------------------------------------------------------------------------------------
def test_every_op_the_module_calls_is_replayed_or_has_no_numerics():
    src = open(os.path.join(ROOT, "unimatch_b200", "unimatch.py")).read()
    called = set(re.findall(r"\b_OPS\.(\w+)", src))
    assert len(called) >= 15, called
    missing = called - set(LR.CHECKS) - set(LR.NO_NUMERICS)
    assert not missing, "ops the module calls with no float64 check in tests/launch_replay.py: %s" % sorted(missing)
    assert all(isinstance(why, str) and why.strip() for why in LR.NO_NUMERICS.values())
    assert not set(LR.CHECKS) & set(LR.NO_NUMERICS)


def test_every_replay_check_binds_to_an_op():
    for name in LR.CHECKS:
        assert hasattr(ops, "_" + name) and hasattr(torch.ops.unimatch_sm100, name), name


# ---- signatures, dedupe and the copy before the call ---------------------------------------------------------------
class _Counting:
    """An op table that counts the calls of each op and may run a hook after the real op."""

    def __init__(self, after=None):
        refops.register_cpu_kernels()
        self.real, self.calls, self.after = torch.ops.unimatch_sm100, {}, after

    def __getattr__(self, name):
        fn = getattr(self.real, name)

        def call(*a, **kw):
            self.calls[name] = self.calls.get(name, 0) + 1
            out = fn(*a, **kw)
            if self.after:
                self.after(name, a, out)
            return out
        return call


def _flow(shape, seed=0):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed)) * 4


def test_signature_holds_op_scalars_shapes_and_strides():
    f = _flow((2, 6, 8, 2))
    base = LR.signature("upsample2x", {"flow": f, "mult": 2.0})
    assert base == ("upsample2x", ("flow", ("tensor", (2, 6, 8, 2), (96, 16, 2, 1), "torch.float32")), ("mult", 2.0))
    assert LR.signature("upsample2x", {"flow": f, "mult": 4.0}) != base
    assert LR.signature("upsample2x", {"flow": _flow((2, 6, 9, 2)), "mult": 2.0}) != base
    strided = torch.zeros((2, 6, 8, 4))[..., :2]
    assert strided.shape == f.shape and LR.signature("upsample2x", {"flow": strided, "mult": 2.0}) != base
    assert LR.signature("upsample2x", {"flow": _flow((2, 6, 8, 2), 1), "mult": 2.0}) == base      # values do not count
    assert LR.signature("conv2d_tc", {"win_geom": [4, 6, 2, 2, 1, 1, 1]})[1] == ("win_geom", (4, 6, 2, 2, 1, 1, 1))


def test_replay_checks_each_signature_once():
    table = _Counting()
    rp = LR.Replay(table)
    for seed in range(3):                                             # refinement iterations: one check
        rp.upsample2x(_flow((2, 6, 8, 2), seed), 2.0)
    rp.upsample2x(flow=_flow((2, 6, 8, 2)), mult=2.0)                 # keywords bind to the same signature
    rp.upsample2x(_flow((2, 6, 8, 2)), 4.0)
    rp.upsample2x(_flow((1, 5, 7, 1)), 2.0)
    assert table.calls["upsample2x"] == 6
    assert [sig[-1][1] for sig, _ in rp.checked] == [2.0, 4.0, 2.0] and len(rp.seen) == 3
    assert all(0 <= r <= 1 for _, r in rp.checked)
    assert rp.upsample2x.__name__ == "wrapped"
    assert LR.Replay(table, only={"add_position"}).upsample2x.__name__ == "call"          # not checked: runs as it is


def test_replay_copies_inputs_before_the_call():
    """An op that overwrites its input after computing passes (the check reads the copy taken before the call), and the
    check of an op whose output is wrong fails, naming the op and the signature."""
    def scribble(name, a, out):
        if name == "upsample2x":
            a[0].mul_(-3.0).add_(1.0)
    rp = LR.Replay(_Counting(scribble))
    f = _flow((2, 6, 8, 2))
    orig = f.clone()
    rp.upsample2x(f, 2.0)
    assert not torch.equal(f, orig) and len(rp.checked) == 1

    def wrong(name, a, out):
        if name == "upsample2x":
            out[:, -1, -1, 0] += 1e-3 * out.abs().max()
    rp = LR.Replay(_Counting(wrong))
    with pytest.raises(AssertionError) as e:
        rp.upsample2x(_flow((2, 6, 8, 2)), 2.0)
    assert str(e.value).startswith("upsample2x:") and "signature: upsample2x(flow=((2, 6, 8, 2)" in str(e.value)


def test_replay_reads_planes_as_hi_plus_lo():
    """split_planes writes (hi, lo) in place: the replay checks it bit for bit, and planes_value reads back the fp32 value
    to within the split's 22 bits."""
    rp = LR.Replay(_Counting())
    x = _flow((3, 5, 7, 40)) + 8.0
    dst = torch.zeros((2, 3, 5, 7, 128), dtype=torch.float16)
    rp.split_planes(x, dst, 64)
    assert len(rp.checked) == 1 and dst[..., :64].abs().max() == 0
    assert ((LR.planes_value(dst)[..., 64:104] - x).abs() <= 2.0 ** -22 * x.abs()).all()


def test_subsets_hold_every_row_of_the_last_tiles():
    g = torch.Generator().manual_seed(0)
    rows = LR.token_rows(6688, g)                                     # KITTI 1/8: last query tile of 32 rows
    assert set(range(6656, 6688)) <= set(rows.tolist()) and set(range(64)) <= set(rows.tolist())
    tok = LR.attention_rows(44, 152, 2, 2, 11, 38, g)                 # 1/8 windows of 1672 tokens, tail 8
    t_all, _ = __import__("ref64").window_layout(44, 152, 2, 2, 11, 38)
    for wi in range(4):
        assert set(t_all[wi, 1664:].tolist()) <= set(tok.tolist())
