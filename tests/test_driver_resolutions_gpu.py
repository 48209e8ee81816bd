"""The model at the sizes the drivers run it at (tests/driver_sizes.py: the reference's submission and evaluation sizes), not
only at the bench resolutions:

  * every distinct launch of one synthetic forward against float64 (tests/launch_replay.py), with its `max err/bound`;
  * the teacher-forced stage parity against the oracle (tests/stage_checks.py, its tolerances unchanged);
  * the launch census: every dispatch key these sizes reach must have an edge case in tests/test_kernel_edges_gpu.py or
    tests/test_matching_edges_gpu.py;
  * and the replay's teeth: a lo plane dropped from a convolution input, the last ragged query tile of the window attention
    off by 2^-12, and the last ragged key tile dropped from the global correlation, each at a driver size, must fail the
    check, naming the op and its signature.

Each test prints its wall time and the part of it spent on the host (oracle forward, float64 references, copies)."""
import math
import time

import pytest
import torch

import launch_replay as LR
import ref64
import stage_checks
import test_kernel_edges_gpu as K
import unimatch_b200.unimatch as um
from driver_sizes import CASES, case_id
from unimatch_b200 import ops
from unimatch_b200.spec import WORKLOADS
from unimatch_b200.synthetic import synthetic_batch, synthetic_model, workload_call

pytestmark = pytest.mark.gpu


def _forward(case, model=None):
    task = WORKLOADS[case.workload]["model"]["task"]
    call = workload_call(case.workload)
    if case.bidir:
        call["pred_bidir_flow" if task == "flow" else "pred_bidir_depth"] = True
    model = model or synthetic_model(case.workload)
    inp = {k: v.cuda() for k, v in synthetic_batch(task, 1, case.H, case.W).items()}
    with torch.no_grad():
        out = model(inp["img0"], inp["img1"], intrinsics=inp.get("intrinsics"), pose=inp.get("pose"), **call)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_every_launch_against_float64(monkeypatch, case):
    model = synthetic_model(case.workload)
    replay = LR.Replay(um._OPS)
    monkeypatch.setattr(um, "_OPS", replay)
    t0 = time.perf_counter()
    _forward(case, model)
    wall = time.perf_counter() - t0
    print("%s: %d signatures checked, worst max err/bound %.3f; wall %.1f s, host (copies, float64) %.1f s, device and "
          "launch %.1f s" % (case_id(case), len(replay.checked), max(r for _, r in replay.checked), wall, replay.host_s,
                             wall - replay.host_s))
    ops_seen = {sig[0] for sig, _ in replay.checked}
    assert {"conv2d_tc", "conv7x7_small", "instance_norm_stats", "instance_norm_apply", "split_planes", "add_position",
            "window_attention" if ops_seen.isdisjoint({"window_attention_planes"}) else "window_attention_planes"} <= ops_seen


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_teacher_forced_stages(case):
    lines = []
    t0 = time.perf_counter()
    try:
        stage_checks.run(torch.device("cuda", 0), case.workload, case.H, case.W, case.bidir, report=lines.append)
    finally:
        print("\n%s (%s)\n%s\nwall %.1f s" % (case_id(case), case.origin, "\n".join(lines), time.perf_counter() - t0))


def test_launch_census_at_driver_sizes(monkeypatch):
    census = K._Census(um._OPS)
    monkeypatch.setattr(um, "_OPS", census)
    for case in CASES:
        _forward(case)
        print("census: ran", case_id(case))
    for key in sorted(census.keys, key=str):
        print("census:", key)
    missing = census.keys - K.covered_keys()
    assert not missing, "launch configurations without an edge case: %s" % sorted(missing, key=str)


# ---- the replay rejects defects -----------------------------------------------------------------------------------------
class _Defect:
    """The op table `real`, with op `name` replaced by hook(real_op, *args, **kwargs)."""

    def __init__(self, real, name, hook):
        self.real, self.name, self.hook = real, name, hook

    def __getattr__(self, name):
        fn = getattr(self.real, name)
        return (lambda *a, **kw: self.hook(fn, *a, **kw)) if name == self.name else fn


def _conv_lo_plane_dropped(fn, *a, **kw):
    """the first source's lo plane read as zeros"""
    src0 = kw.pop("src0") if "src0" in kw else a[0]
    src0 = src0.clone()
    src0[1].zero_()
    return fn(src0, *a[1:], **kw) if a else fn(src0=src0, **kw)


def _attention_last_query_tile_off(fn, qp, kp, vp, n, kvs, h, w, kh, kw, sh, sw, mask, out_f32, out_split):
    """every row of the last (ragged) query tile of every window written 2^-12 too large"""
    fn(qp, kp, vp, n, kvs, h, w, kh, kw, sh, sw, mask, out_f32, out_split)
    tok, _ = ref64.window_layout(h, w, kh, kw, sh, sw)
    tail = tok[:, LR.tail_rows(tok.shape[1], LR.TILE_Q)].reshape(-1)
    rows = (torch.arange(n)[:, None] * h * w + tail).reshape(-1).to(out_split.device)
    x = (out_split[0, rows].float() + out_split[1, rows].float()) * (1 + 2.0 ** -12)
    hi = x.half()
    out_split[0, rows], out_split[1, rows] = hi, (x - hi.float()).half()


def _expectation_last_key_tile_dropped(fn, q, k, values, ns, kvs, vdim, vm, post, h, w, kh, kw, mask):
    """the global correlation (softmax over every key, expected key coordinates minus the query's) without the keys of its
    last (ragged) key tile, in float64 on the device"""
    if vm != ops.VALUE_COORDS:
        return fn(q, k, values, ns, kvs, vdim, vm, post, h, w, kh, kw, mask)
    L = q.shape[1]
    keep = (L - 1) // LR.TILE_K * LR.TILE_K
    t = torch.arange(L, device=q.device)
    xy = torch.stack((t % w, t // w), -1).double()
    outs = []
    for s in range(ns):
        kk = k[(s + kvs) % q.shape[0], :keep].double()
        p = torch.softmax(q[s].double() @ kk.T / math.sqrt(128), -1)
        outs.append(p @ xy[:keep] - xy)
    return torch.stack(outs).float()


DEFECTS = {
    "conv_lo_plane_dropped": ("conv2d_tc", _conv_lo_plane_dropped),
    "attention_last_query_tile_2^-12": ("window_attention_planes", _attention_last_query_tile_off),
    "expectation_last_key_tile_dropped": ("softmax_expectation", _expectation_last_key_tile_dropped),
}


@pytest.mark.parametrize("defect", sorted(DEFECTS))
def test_replay_rejects_defect_at_driver_size(monkeypatch, defect):
    """KITTI flow submission size, 352x1216: 6688 correlation tokens (last key tile: 32 keys), 1/8 windows of 1672 tokens
    (last query tile: 8 rows).  Only the defective op is checked."""
    name, hook = DEFECTS[defect]
    case = [c for c in CASES if (c.workload, c.H, c.W, c.bidir) == ("gmflow-scale2-regrefine6", 352, 1216, False)][0]
    model = synthetic_model(case.workload)
    monkeypatch.setattr(um, "_OPS", LR.Replay(_Defect(um._OPS, name, hook), only={name}))
    with pytest.raises(AssertionError) as e:
        _forward(case, model)
    msg = str(e.value)
    print("%s rejected: %s" % (defect, msg))
    assert msg.startswith(name + ":") and ("signature: %s(" % name) in msg, msg
