"""Batches of pairs on the host side (no GPU): the table of batched launches the module issues, with their stream arguments
written relative to the batch B; the census that checks every launch of every workload against that table; the batch-3
cases (bidirectional modes, a distinct camera per pair) run through the module's host logic with the oracle-backed CPU
kernels of tests/refops.py and compared pair by pair with the reference; and the defects these checks must catch, injected
by wrapping the op table the module calls.  tests/test_batch_gpu.py runs the same table, census and cases on the device."""
import functools
import types

import pytest
import torch

import cases
import refops
from unimatch_b200 import UniMatch, ops
from unimatch_b200.spec import WORKLOADS

# ---- the batched launches of the module ------------------------------------------------------------------------------
# B pairs = 2B streams (all first views, then all second views); stream b pairs with stream B + b.  Each row: name, stream
# pattern (op, stream arguments relative to B, then what selects the variant), feature map (h, w), parameters.
ATTN, PLANES, EXP = "window_attention", "window_attention_planes", "softmax_expectation"
VC, VX, VT = ops.VALUE_COORDS, ops.VALUE_XCOORD, ops.VALUE_TENSOR
BATCH_TABLE = [
    # attention: (op, streams, kv_shift); kernel window (kh, kw) and Swin shift
    ("attn_swin2d_s8_self", (PLANES, "2B", "0"), (60, 104), dict(k=(2, 2), shift=False)),
    ("attn_swin2d_s8_cross_shifted", (PLANES, "2B", "B"), (60, 104), dict(k=(2, 2), shift=True)),
    ("attn_swin2d_s4_self_shifted", (PLANES, "2B", "0"), (120, 208), dict(k=(8, 8), shift=True)),
    ("attn_swin2d_s4_cross", (PLANES, "2B", "B"), (120, 208), dict(k=(8, 8), shift=False)),
    ("attn_swin2d_s4_self_cuda_cores", (ATTN, "2B", "0"), (64, 80), dict(k=(8, 8), shift=True)),     # 80-token windows
    ("attn_stereo_swin1d_s4_cross", (ATTN, "2B", "B"), (136, 240), dict(k=(136, 8), shift=True)),
    ("attn_stereo_swin1d_s8_cross", (ATTN, "2B", "B"), (68, 120), dict(k=(68, 2), shift=False)),
    # softmax expectation: (op, streams, n_streams, kv_shift, value mode)
    ("corr_flow", (EXP, "2B", "B", "B", VC), (60, 104), {}),
    ("corr_flow_bidir", (EXP, "2B", "2B", "B", VC), (60, 104), {}),
    ("corr_stereo_causal", (EXP, "2B", "B", "B", VX), (68, 120), {}),
    ("prop_fd2", (EXP, "B", "B", "0", VT), (60, 104), dict(fd=2)),
    ("prop_fd1", (EXP, "B", "B", "0", VT), (68, 120), dict(fd=1)),
    ("prop_fd2_bidir", (EXP, "2B", "2B", "0", VT), (60, 104), dict(fd=2)),
    ("prop_fd1_bidir", (EXP, "2B", "2B", "0", VT), (48, 64), dict(fd=1)),
    # matching path on the CUDA cores: (op, streams, variant)
    ("lcs_stencil", ("local_corr_softmax", "B", False), (120, 208), {}),
    ("lcs_stereo_gather", ("local_corr_softmax", "B", True), (136, 240), {}),
    ("corr_volume_fd2", ("local_corr_volume", "B", 2), (120, 208), {}),
    ("corr_volume_fd1", ("local_corr_volume", "B", 1), (136, 240), {}),
    ("corr_volume_fd2_bidir", ("local_corr_volume", "2B", 2), (48, 64), {}),
    ("flow_warp_fd2", ("flow_warp", "B", 2), (120, 208), {}),
    ("flow_warp_fd1", ("flow_warp", "B", 1), (136, 240), {}),
    ("flow_warp_fd2_bidir", ("flow_warp", "2B", 2), (120, 208), {}),
    ("propagate_local_fd2", ("propagate_local", "B", 2), (120, 208), {}),
    ("propagate_local_fd1", ("propagate_local", "B", 1), (136, 240), {}),
    ("propagate_local_fd2_bidir", ("propagate_local", "2B", 2), (120, 208), {}),
    ("convex_f4_fd2", ("convex_upsample", "B", 4, 2, False), (120, 208), {}),
    ("convex_f4_fd1", ("convex_upsample", "B", 4, 1, False), (136, 240), {}),
    ("convex_f8_fd2", ("convex_upsample", "B", 8, 2, False), (60, 104), {}),
    ("convex_f8_depth", ("convex_upsample", "B", 8, 2, True), (48, 64), {}),
    ("convex_f8_depth_bidir", ("convex_upsample", "2B", 8, 2, True), (48, 64), {}),
    ("convex_f4_fd2_bidir", ("convex_upsample", "2B", 4, 2, False), (120, 208), {}),
    ("upsample2x_fd2", ("upsample2x", "B", 2), (60, 104), {}),
    ("upsample2x_fd1", ("upsample2x", "B", 1), (68, 120), {}),
    ("upsample2x_fd2_bidir", ("upsample2x", "2B", 2), (60, 104), {}),
    ("add_position", ("add_position", "2B"), (120, 208), dict(table=(15, 26))),
    ("add_position_bidir", ("add_position", "4B"), (120, 208), dict(table=(15, 26))),
    # depth plane sweep: (op, streams, intrinsics, poses, argmax)
    ("depth_softmax", ("depth_corr_softmax", "B", "B", "B", False), (48, 64), {}),
    ("depth_argmax", ("depth_corr_softmax", "B", "B", "B", True), (48, 64), {}),
    ("depth_softmax_bidir", ("depth_corr_softmax", "2B", "2B", "2B", False), (48, 64), {}),
    ("depth_argmax_bidir", ("depth_corr_softmax", "2B", "2B", "2B", True), (48, 64), {}),
    # encoder: (op, images, variant)
    ("in_stats_c64", ("instance_norm_stats", "2B"), (192, 256), dict(c=64)),
    ("in_apply_relu", ("instance_norm_apply", "2B", False, False), (192, 256), dict(c=64)),
    ("in_apply_res_identity", ("instance_norm_apply", "2B", True, False), (96, 128), dict(c=96)),
    ("in_apply_res_downsample", ("instance_norm_apply", "2B", True, True), (48, 64), dict(c=128)),
    ("stem", ("conv7x7_small", "B", "B", True), (384, 512), {}),
    ("flow_encoder_fd2", ("conv7x7_small", "B", None, False), (120, 208), dict(fd=2)),
    ("flow_encoder_fd1", ("conv7x7_small", "B", None, False), (136, 240), dict(fd=1)),
    ("flow_encoder_fd2_bidir", ("conv7x7_small", "2B", None, False), (48, 64), dict(fd=2)),
    # tensor-core convolution: (op, images or token rows, window-plane streams)
    ("conv_linear_rows", ("conv2d_tc", "rows", None), (48, 64), dict(layer="linear")),
    ("conv_ln_rows", ("conv2d_tc", "rows", None), (48, 64), dict(layer="ln")),
    ("conv_window_planes", ("conv2d_tc", "rows", "2B"), (48, 64), dict(layer="win")),
    ("conv_stride2", ("conv2d_tc", "2B", None), (96, 128), dict(layer="stride2")),
    ("conv_gru_zr_pre", ("conv2d_tc", "B", None), (48, 64), dict(layer="zr")),
    ("conv_gru_q_pre", ("conv2d_tc", "B", None), (48, 64), dict(layer="q")),
    ("conv_gru_zr_pre_bidir", ("conv2d_tc", "2B", None), (48, 64), dict(layer="zr")),
    ("ffn_rows", ("ffn_tc", "rows"), (48, 64), {}),
]


def rel(v, B):
    """A stream count or offset written relative to the batch B."""
    return {0: "0", B: "B", 2 * B: "2B", 4 * B: "4B"}.get(int(v), str(int(v)))


class StreamCensus:
    """Stands in for torch.ops.unimatch_sm100 in unimatch_b200.unimatch: records the stream pattern of every launch (the
    BATCH_TABLE form, relative to the batch B of the forward) and delegates to the real op."""

    def __init__(self, real, B):
        self.real, self.B, self.patterns = real, B, set()

    def __getattr__(self, name):
        fn = getattr(self.real, name)
        rec = getattr(self, "_p_" + name, None)
        if rec is None:
            return fn

        def wrapped(*a, **kw):
            self.patterns.add(rec(*a, **kw))
            return fn(*a, **kw)
        return wrapped

    def r(self, v):
        return rel(v, self.B)

    def _p_window_attention(self, q, k, v, kvs, *geo):
        return (ATTN, self.r(q.shape[0]), self.r(kvs))

    def _p_window_attention_planes(self, qp, kp, vp, n, kvs, *rest):
        return (PLANES, self.r(n), self.r(kvs))

    def _p_softmax_expectation(self, q, k, values, ns, kvs, vdim, vm, *rest):
        return (EXP, self.r(q.shape[0]), self.r(ns), self.r(kvs), vm)

    def _p_local_corr_softmax(self, f0, f1, h, w, ry, rx, stereo):
        return ("local_corr_softmax", self.r(f0.shape[0]), bool(stereo))

    def _p_local_corr_volume(self, f0, f1, flow, h, w, radius):
        return ("local_corr_volume", self.r(f0.shape[0]), flow.shape[-1])

    def _p_flow_warp(self, f, flow, h, w):
        return ("flow_warp", self.r(f.shape[0]), flow.shape[-1])

    def _p_propagate_local(self, q, k, flow, h, w, radius):
        return ("propagate_local", self.r(q.shape[0]), flow.shape[-1])

    def _p_convex_upsample(self, flow, mask, factor, mult):
        return ("convex_upsample", self.r(flow.shape[0]), factor, flow.shape[-1], mult == 1)

    def _p_upsample2x(self, flow, mult):
        return ("upsample2x", self.r(flow.shape[0]), flow.shape[-1])

    def _p_add_position(self, x, table, h, w):
        return ("add_position", self.r(x.shape[0]))

    def _p_depth_corr_softmax(self, f0, f1, K, Kinv, pose, cand, h, w, from_argmax):
        return ("depth_corr_softmax", self.r(f0.shape[0]), self.r(K.shape[0]), self.r(pose.shape[0]), bool(from_argmax))

    def _p_instance_norm_stats(self, x):
        return ("instance_norm_stats", self.r(x.shape[0]))

    def _p_instance_norm_apply(self, a, stats_a, relu_a, res, stats_res, *rest):
        return ("instance_norm_apply", self.r(a.shape[0]), res is not None, stats_res is not None)

    def _p_conv7x7_small(self, in0, in1, nchw, *rest):
        return ("conv7x7_small", self.r(in0.shape[0]), None if in1 is None else self.r(in1.shape[0]), bool(nchw))

    def _p_conv2d_tc(self, *a, **kw):
        p = _conv_args(*a, **kw)
        return ("conv2d_tc", "rows" if p["rows"] else self.r(p["src0"].shape[1]),
                None if p["win_dst"] is None else self.r(p["win_streams"]))

    def _p_ffn_tc(self, *a):
        return ("ffn_tc", "rows")


def _conv_args(*a, **kw):
    import inspect
    b = inspect.signature(ops._conv2d_tc).bind(*a, **kw)
    b.apply_defaults()
    return b.arguments


CENSUS_SIZE = {"flow": (128, 192), "stereo": (128, 192), "depth": (128, 192)}


def census_inputs(task, B, h, w, dev):
    from unimatch_b200.synthetic import synthetic_batch
    d = synthetic_batch(task, B, h, w)
    if task == "depth":
        d["intrinsics"], d["pose"] = cases.distinct_cameras(B, h, w)
    return {k: v.to(dev) for k, v in d.items()}


def run_batch_census(monkeypatch, dev, defect=None, B=3, size=CENSUS_SIZE):
    """One forward of every workload at batch B and `size` per task; returns the recorded stream patterns that are not rows of
    BATCH_TABLE (must be empty)."""
    import unimatch_b200.unimatch as um
    from unimatch_b200.synthetic import synthetic_model
    census = StreamCensus(um._OPS, B)
    monkeypatch.setattr(um, "_OPS", census if defect is None else OpsDefect(census, defect))
    for wl, cfg in WORKLOADS.items():
        task = cfg["model"]["task"]
        m = synthetic_model(wl, dev)
        inp = census_inputs(task, B, *size[task], dev)
        m(inp["img0"], inp["img1"], intrinsics=inp.get("intrinsics"), pose=inp.get("pose"), **cfg["call"])
    for p in sorted(census.patterns, key=str):
        print("batch census:", p)
    return census.patterns - {row[1] for row in BATCH_TABLE}


# ---- defects, injected by wrapping the op table the module calls -----------------------------------------------------
class OpsDefect:
    """Delegates to `real` (the op table or a census around it) except for one defect:
      camera0   every pair's depth sweep uses pair 0's intrinsics, inverse and pose;
      kvshift   the cross-attention partner of stream n is n + B + 1 mod 2B instead of n + B;
      swap      the two halves of a bidirectional output (forward / backward streams) are exchanged;
      stereo2b  the stereo correlation is launched with n_streams = 2B (its first B outputs are kept)."""

    def __init__(self, real, defect):
        self.real, self.defect = real, defect

    def __getattr__(self, name):
        fn = getattr(self.real, name)
        hook = getattr(self, "_%s_%s" % (self.defect, name), None)
        return fn if hook is None else functools.partial(hook, fn)

    @staticmethod
    def _camera0_depth_corr_softmax(fn, f0, f1, K, Kinv, pose, *rest):
        first = lambda t: t[:1].expand_as(t).contiguous()
        return fn(f0, f1, first(K), first(Kinv), first(pose), *rest)

    @staticmethod
    def _kvshift_window_attention(fn, q, k, v, kvs, *rest):
        return fn(q, k, v, (kvs + 1) % q.shape[0] if kvs else kvs, *rest)

    @staticmethod
    def _kvshift_window_attention_planes(fn, qp, kp, vp, n, kvs, *rest):
        return fn(qp, kp, vp, n, (kvs + 1) % n if kvs else kvs, *rest)

    @staticmethod
    def _swap_softmax_expectation(fn, q, k, values, ns, kvs, *rest):
        out = fn(q, k, values, ns, kvs, *rest)
        if ns == q.shape[0] and kvs:                                # the bidirectional flow correlation
            out = torch.cat((out[ns // 2:], out[:ns // 2]))
        return out

    @staticmethod
    def _swap_depth_corr_softmax(fn, *a):
        out = fn(*a)
        n = out.shape[0]                                            # at batch 3 only the bidirectional sweep is even
        return torch.cat((out[n // 2:], out[:n // 2])) if n % 2 == 0 else out

    @staticmethod
    def _stereo2b_softmax_expectation(fn, q, k, values, ns, kvs, vdim, vm, post, h, w, kh, kw, mask):
        if mask == ops.MASK_CAUSAL:
            return fn(q, k, values, q.shape[0], kvs, vdim, vm, post, h, w, kh, kw, mask)[:ns]
        return fn(q, k, values, ns, kvs, vdim, vm, post, h, w, kh, kw, mask)


# ---- batch 3 against the reference -----------------------------------------------------------------------------------
def batch3_tolerance(name):
    return cases.E2E_NOISE_FACTOR * cases.BATCH3_NOISE[name] + 1e-4


def check_against_reference(name, got, ref, B=3):
    """Pair by pair: the layout (bidirectional modes: forward outputs of the B pairs, then their backward outputs) and the
    mean error of each output within the E2E rule."""
    assert tuple(got.shape) == tuple(ref.shape), (name, got.shape, ref.shape)
    tol = batch3_tolerance(name)
    worst = 0.0
    for i in range(got.shape[0]):
        mean, mx = cases.epe(got[i:i + 1].cpu(), ref[i:i + 1])
        worst = max(worst, mean)
        assert mean <= tol, "%s: output %d of %d: mean err %.3e > tol %.3e (max %.3e)" % (name, i, got.shape[0], mean, tol, mx)
    print("%-32s worst pair mean err %.3e (tol %.3e)" % (name, worst, tol))


def module_forward(cfg, sd, batch, call, dev):
    m = UniMatch(**cfg["model"]).eval()
    m.load_state_dict(sd, strict=True)
    m = m.to(dev)
    d = {k: v.to(dev) for k, v in batch.items()}
    return m(d["img0"], d["img1"], intrinsics=d.get("intrinsics"), pose=d.get("pose"), **call)["flow_preds"][-1]


TINY = {"flow": (64, 96), "stereo": (64, 96), "depth": (64, 96)}


def tiny_setup(name):
    task = cases.WORKLOADS[cases.BATCH3_CASES[name][0]]["model"]["task"]
    h, w = TINY[task]
    if cases.BATCH3_CASES[name][0] == "gmflow-scale2-regrefine6":
        w = 128
    return cases.batch3_setup(name, h, w)


@pytest.mark.parametrize("name", sorted(cases.BATCH3_CASES))
def test_batch3_host_logic_matches_reference(name):
    refops.register_cpu_kernels()
    cfg, sd, batch, call = tiny_setup(name)
    check_against_reference(name, module_forward(cfg, sd, batch, call, "cpu"), cases.oracle_forward(cfg, sd, batch, call))


@pytest.mark.parametrize("bidir", [False, True])
def test_depth_cameras_are_per_pair(bidir):
    """The cameras of a batch are the cameras of its pairs, stacked: intrinsics scaled to the feature map, inverse and pose
    of every pair (and, bidirectional, of the backward streams B + b), bit for bit."""
    K, pose = cases.distinct_cameras(5, 384, 512)
    m = types.SimpleNamespace(_cands={})
    cams = UniMatch.depth_cameras(m, K, pose, 8, 0.1, 2.0, 64, bidir)
    assert len({tuple(k.flatten().tolist()) for k in cams["K"][:5]}) == 5
    for b in range(5):
        one = UniMatch.depth_cameras(m, K[b:b + 1], pose[b:b + 1], 8, 0.1, 2.0, 64, bidir)
        idx = [b, 5 + b] if bidir else [b]
        for key in ("K", "K_inv", "pose"):
            assert torch.equal(cams[key][idx], one[key]), (key, b)
    if bidir:
        assert torch.allclose(cams["pose"][5:] @ cams["pose"][:5], torch.eye(4).expand(5, 4, 4), atol=1e-5)


def test_batch_census_on_cpu(monkeypatch):
    refops.register_cpu_kernels()
    missing = run_batch_census(monkeypatch, "cpu")
    assert not missing, "batched launches without a row in BATCH_TABLE: %s" % sorted(missing, key=str)


# ---- the defects fail the checks that target them --------------------------------------------------------------------
DEFECT_CASES = [("camera0", "b3_gmdepth_s1"), ("camera0", "b3_gmdepth_s1_rr1_bidir"), ("kvshift", "b3_gmstereo_s2"),
                ("kvshift", "b3_gmflow_s1_bidir"), ("swap", "b3_gmflow_s1_bidir"), ("swap", "b3_gmdepth_s1_bidir")]


@pytest.mark.parametrize("defect,name", DEFECT_CASES)
def test_batch3_check_rejects_defect(monkeypatch, defect, name):
    import unimatch_b200.unimatch as um
    refops.register_cpu_kernels()
    cfg, sd, batch, call = tiny_setup(name)
    ref = cases.oracle_forward(cfg, sd, batch, call)
    monkeypatch.setattr(um, "_OPS", OpsDefect(um._OPS, defect))
    with pytest.raises(AssertionError) as e:
        check_against_reference(name, module_forward(cfg, sd, batch, call, "cpu"), ref)
    print("%s / %s rejected: %s" % (defect, name, str(e.value).splitlines()[0]))


def test_batch_census_rejects_stereo_2b(monkeypatch):
    refops.register_cpu_kernels()
    missing = run_batch_census(monkeypatch, "cpu", "stereo2b")
    print("stereo2b: patterns outside the table:", sorted(missing, key=str))
    assert (EXP, "2B", "2B", "B", VX) in missing
