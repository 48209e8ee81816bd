"""Mixed-size flow streaming on the device: each ragged flow kernel against the per-image kernel on mixed sizes (KITTI's
four, a portrait frame, a frame at the output size, a 1-pixel-high frame), bit for bit, skipped items left untouched, a
captured graph following its table; and `MixedSizeFlowRunner` against the same steps recomputed from existing functions
only (tests/refops_flow_ragged.py: the uniform conversion per frame, one forward per step, `_flow_outputs` per size,
`flow_to_image`), and against `infer_flow` on each pair alone."""
import numpy as np
import pytest
import torch

import refops_flow_ragged
import refops_ragged
from unimatch_b200 import MixedSizeFlowRunner, infer_flow, ops
from unimatch_b200.inference import flow_to_image
from unimatch_b200.synthetic import synthetic_batch, synthetic_model, synthetic_video, workload_call

pytestmark = pytest.mark.gpu
_OPS = torch.ops.unimatch_sm100
T = ops.RAGGED_TRANSPOSE
KITTI = [(375, 1242), (370, 1226), (374, 1238), (376, 1241)]


def _offsets(sizes, per_pixel, gap=0):
    offsets, off = [], 0
    for h, w in sizes:
        offsets.append(off)
        off += per_pixel * h * w + gap
    return offsets, off


def _lib(name, *args):
    """the C entry itself, for outputs the test fills with canaries first"""
    rc = getattr(ops.LIB, name)(*[ops._p(a) if torch.is_tensor(a) else a for a in args], ops._stream())
    assert rc == 0, ops.LIB.um_last_error()


def test_frames_to_planar_ragged_equals_per_frame():
    ho, wo = 384, 1248
    sizes = KITTI + [(1242, 375), (ho, wo), (1, 50), (wo, ho)]
    flags = [0, 0, 0, 0, T, 0, 0, T]
    g = torch.Generator().manual_seed(3)
    frames = [torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8) for h, w in sizes]
    offsets, total = _offsets(sizes, 3)
    packed = torch.cat([f.reshape(-1) for f in frames]).cuda()
    recs = [(o, h, w, 1.0, f) for o, (h, w), f in zip(offsets, sizes, flags)]
    recs += [(0, 1300, 10, 1.0, 0), (0, 0, 0, 1.0, 0), (total - 5, 2, 2, 1.0, 0)]     # too tall, empty, beyond the buffer
    items = refops_ragged.table(recs, "cuda")
    out = _OPS.frames_to_planar_ragged(packed, items, 1248, 1248, ho, wo)
    for i, (f, fl) in enumerate(zip(frames, flags)):
        one = _OPS.frames_to_planar(f[None].cuda().contiguous(), ho, wo, bool(fl))
        assert torch.equal(out[i], one[0]), i
    assert torch.equal(out[5].cpu(), frames[5].permute(2, 0, 1).float())                      # exact conversion
    assert torch.equal(out[7].cpu(), frames[7].permute(2, 1, 0).float())                      # and exact transpose
    assert torch.equal(out[:8], refops_flow_ragged.frames_to_planar_ragged(packed, items, 1248, 1248, ho, wo)[:8])
    canary = torch.full((len(recs), 3, ho, wo), -7.0, device="cuda")
    _lib("um_frames_to_planar_ragged", packed, packed.numel(), items, canary, len(recs), 1248, 1248, ho, wo)
    assert torch.equal(canary[:8], out[:8]) and (canary[8:] == -7).all()


def _flow_items(sizes, size, gap=0):
    """two plane items per flow, as the runner lays them out, `gap` floats apart"""
    recs, offs, off = [], [], 0
    for h, w in sizes:
        t = h > w
        ori = (w, h) if t else (h, w)
        su, sv = (np.float32(ori[1] / size[1]), np.float32(ori[0] / size[0])) if ori != size else (1.0, 1.0)
        recs += [(off, h, w, su, T if t else 0), (off + h * w, h, w, sv, T if t else 0)]
        offs.append(off)
        off += 2 * h * w + gap
    return recs, offs, off


def _resize_back(flow, h, w, size):
    """what `_flow_outputs` does with one flow [1, 2, H, W] of a pair stored as (h, w)"""
    t = h > w
    ori = (w, h) if t else (h, w)
    y = flow if ori == size else _OPS.resize_bilinear(flow, ori[0], ori[1], [ori[1] / size[1], ori[0] / size[0]], False)
    return (y.transpose(-2, -1) if t else y)[0].contiguous()


def test_resize_bilinear_ragged_transposed_flow_equals_per_image():
    size = (96, 312)
    sizes = [(94, 311), (93, 307), (312, 94), (96, 312), (312, 96), (1, 40), (40, 1), (150, 400)]
    g = torch.Generator().manual_seed(7)
    flow = (torch.randn((len(sizes), 2) + size, generator=g) * 30)
    flow[3, 0, 5, 6] = float("inf")
    flow[4, 1, 7, 8] = float("nan")
    flow = flow.cuda()
    recs, offs, total = _flow_items(sizes, size, gap=3)
    recs += [(0, 500, 10, 1.0, 0), (0, 0, 0, 1.0, 0)]                       # out of range and empty: skipped
    x = torch.cat((flow.view(-1, 1, *size), flow[:1].view(2, 1, *size)))
    out = torch.full((total,), -7.0, device="cuda")
    _lib("um_resize_bilinear_ragged", x, out, total, refops_ragged.table(recs, "cuda"), len(recs), size[0], size[1], 400,
         400)
    for i, (h, w) in enumerate(sizes):
        got, ref = out[offs[i]:offs[i] + 2 * h * w].view(2, h, w), _resize_back(flow[i:i + 1], h, w, size)
        assert torch.equal(got.isnan(), ref.isnan()) and torch.equal(got.nan_to_num(), ref.nan_to_num()), i
        assert (out[offs[i] + 2 * h * w:offs[i] + 2 * h * w + 3] == -7).all(), i        # the gaps between items are intact
    assert torch.equal(out[offs[3]:offs[3] + 2 * 96 * 312].view(2, 96, 312)[0], flow[3, 0])          # copied, inf included
    ref = refops_flow_ragged.resize_bilinear_ragged(x, refops_ragged.table(recs, "cuda"), 400, 400, total)
    keep = out != -7
    assert torch.equal(out[keep].nan_to_num(), ref[keep].nan_to_num())


def test_captured_resize_follows_the_table():
    size = (64, 96)
    g = torch.Generator().manual_seed(9)
    flow = (torch.randn((2, 2) + size, generator=g) * 10).cuda()
    x = flow.view(4, 1, *size)
    first, _, _ = _flow_items([(50, 90), (96, 64)], size)
    second, offs, _ = _flow_items([(90, 50), (33, 77)], size)
    items = refops_ragged.table(first, "cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        _OPS.resize_bilinear_ragged(x, items, 128, 128, 4 * 128 * 128)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = _OPS.resize_bilinear_ragged(x, items, 128, 128, 4 * 128 * 128)
    graph.replay()
    assert torch.equal(out[:2 * 50 * 90].view(2, 50, 90), _resize_back(flow[:1], 50, 90, size))
    items.copy_(refops_ragged.table(second, "cuda"))
    graph.replay()
    for i, (h, w) in enumerate([(90, 50), (33, 77)]):
        assert torch.equal(out[offs[i]:offs[i] + 2 * h * w].view(2, h, w), _resize_back(flow[i:i + 1], h, w, size)), i


def test_flow_to_image_ragged_equals_per_image():
    """mixed sizes with NaN, inf, unknown (> 1e7) and all-zero flows; the per-image scratch is reset inside every call"""
    sizes = KITTI + [(311, 94), (1, 50), (17, 19), (23, 45), (9, 9)]
    g = torch.Generator().manual_seed(11)
    flows = [torch.randn((2, h, w), generator=g) * 20 for h, w in sizes]
    flows[1][0, 10, 11] = float("nan")
    flows[2][1, 3, 3] = float("inf")
    flows[6][:] = 0
    flows[7][0, 0, 0] = 2e7
    flows[8][:] = float("nan")
    foffs, ftotal = _offsets(sizes, 2, gap=2)
    poffs, ptotal = _offsets(sizes, 3, gap=5)
    packed = torch.zeros((ftotal,))
    for o, f in zip(foffs, flows):
        packed[o:o + f.numel()] = f.reshape(-1)
    packed = packed.cuda()
    frecs = [(o, h, w, 1.0, 0) for o, (h, w) in zip(foffs, sizes)] + [(0, 2000, 4, 1.0, 0), (0, 0, 0, 1.0, 0), (0, 9, 9, 1.0, 0)]
    precs = [(o, h, w, 1.0, 0) for o, (h, w) in zip(poffs, sizes)] + [(0, 2000, 4, 1.0, 0), (0, 0, 0, 1.0, 0), (0, 9, 8, 1.0, 0)]
    pics = torch.full((ptotal,), 99, dtype=torch.uint8, device="cuda")
    for _ in range(2):
        _OPS.flow_to_image_ragged(packed, refops_ragged.table(frecs, "cuda"), pics, refops_ragged.table(precs, "cuda"), 400,
                                  1300)
    for i, ((h, w), f) in enumerate(zip(sizes, flows)):
        if i > 0:                                  # item 0's slot is where the mismatched item points: still picture 0
            assert (pics[poffs[i] - 5:poffs[i]] == 99).all(), i
        pic = pics[poffs[i]:poffs[i] + 3 * h * w].view(h, w, 3)
        assert torch.equal(pic, flow_to_image(f[None].cuda())[0]), i
    assert (pics[poffs[6]:poffs[6] + 3 * 17 * 19] == 255).all() and (pics[poffs[8]:poffs[8] + 243] == 0).all()
    ref = torch.full_like(pics, 99)
    refops_flow_ragged.flow_to_image_ragged(packed, refops_ragged.table(frecs, "cuda"), ref,
                                            refops_ragged.table(precs, "cuda"), 400, 1300)
    assert torch.equal(pics, ref)


def test_fb_consistency_ragged_equals_per_pair():
    sizes = [(94, 311), (93, 307), (311, 94), (2, 2), (1, 40)]              # the last one is below 2 x 2: skipped
    g = torch.Generator().manual_seed(13)
    fwd = [torch.randn((2, h, w), generator=g) * 3 for h, w in sizes]
    bwd = [-f + torch.randn((2, h, w), generator=g) * 0.4 for f, (h, w) in zip(fwd, sizes)]
    foffs, ftotal = _offsets(sizes + sizes, 2)
    ooffs, ototal = _offsets(sizes + sizes, 1, gap=4)
    packed = torch.cat([f.reshape(-1) for f in fwd + bwd]).cuda()
    fitems = refops_ragged.table([(o, h, w, 1.0, 0) for o, (h, w) in zip(foffs, sizes + sizes)], "cuda")
    oitems = refops_ragged.table([(o, h, w, 1.0, 0) for o, (h, w) in zip(ooffs, sizes + sizes)], "cuda")
    occ = torch.full((ototal,), -7.0, device="cuda")
    _OPS.fb_consistency_ragged(packed, fitems, occ, oitems, 400, 400, 0.01, 0.5)
    n = len(sizes)
    for i, (h, w) in enumerate(sizes[:4]):
        ref = _OPS.fb_consistency(fwd[i][None].cuda(), bwd[i][None].cuda(), 0.01, 0.5)
        for k in range(2):
            o = ooffs[k * n + i]
            assert torch.equal(occ[o:o + h * w].view(h, w), ref[k][0]), (i, k)
            assert (occ[o + h * w:o + h * w + 4] == -7).all(), (i, k)
    assert 0 < occ[:94 * 311].mean() < 1
    assert (occ[ooffs[4]:ooffs[4] + 44] == -7).all() and (occ[ooffs[9]:] == -7).all()
    ref = torch.full_like(occ, -7.0)
    refops_flow_ragged.fb_consistency_ragged(packed, fitems, ref, oitems, 400, 400, 0.01, 0.5)
    assert torch.equal(occ, ref)


# ---------------------------------------------------------------------------------------------------------------- the runner
# An interleaved mix; with padding 32 it falls into the (128, 256), (128, 224) and (64, 128) buckets: two portrait pairs
# share the first with landscape ones, and one pair is at (128, 256) itself, so its flow is not resized back
MIX = [(120, 250), (100, 220), (250, 120), (128, 256), (60, 100), (118, 245), (100, 220), (256, 128), (121, 249), (100, 60)]
CAP = (256, 256)


def _pairs(sizes, seed):
    out = []
    for i, (h, w) in enumerate(sizes):
        frames = synthetic_video(2, h, w, seed=seed + i).numpy()
        out.append((frames[0], frames[1]))
    return out


BIDIR = dict(pred_bidir_flow=True, fwd_bwd_consistency_check=True)
CASES = {                    # sizes, batch, max_buckets, runner arguments
    "buckets": (MIX, 2, 4, dict()),
    "inference_size": (MIX, 2, 4, dict(inference_size=(96, 192))),
    "bidir_check": (MIX, 2, 4, dict(BIDIR)),
    "bwd": (MIX, 2, 4, dict(pred_bwd_flow=True)),
    "eager": (MIX, 2, 4, dict(BIDIR, use_graph=False)),
    "short_tail": (MIX[:7], 3, 4, dict()),
    "max_buckets": (MIX + [(90, 150), (120, 250), (91, 151)], 2, 1, dict()),
    "pictures_only": (MIX, 2, 4, dict(pred_bidir_flow=True, return_flow=False)),
}


@pytest.mark.parametrize("workload", ["gmflow-scale1", "gmflow-scale2-regrefine6"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_mixed_flow_runner_equals_composed_reference(workload, case):
    sizes, batch, max_buckets, kw = CASES[case]
    kw = dict(kw)
    m, call = synthetic_model(workload), workload_call(workload, drop=("task",))
    pairs = _pairs(sizes, seed=40)
    return_flow = kw.get("return_flow", True)
    runner = MixedSizeFlowRunner(m, CAP, batch, "cuda", padding_factor=32, visualize=True, max_buckets=max_buckets, **kw,
                                 **call)
    got = [(i, {k: v.clone() for k, v in r.items()}) for i, r in runner.run(pairs)]
    assert sorted(i for i, _ in got) == list(range(len(pairs)))                  # every index exactly once
    kw.pop("use_graph", None), kw.pop("return_flow", None)
    ref = refops_flow_ragged.composed_flow_reference(m, call, pairs, batch, max_buckets, padding_factor=32, **kw)
    keys = {"flow", "vis"} | ({"flow_bwd", "vis_bwd"} if kw.get("pred_bidir_flow") else set())
    keys |= {"fwd_occ", "bwd_occ"} if kw.get("fwd_bwd_consistency_check") else set()
    if not return_flow:
        keys = {k for k in keys if k.startswith("vis")}
    for i, r in got:
        assert set(r) == keys, (case, i)
        h, w = sizes[i]
        for k in keys:
            shape = (2, h, w) if k.startswith("flow") else (h, w, 3) if k.startswith("vis") else (h, w)
            assert tuple(r[k].shape) == shape, (case, i, k)
            assert torch.equal(r[k], ref[i][k]), (case, i, k)
    assert runner.stats["pairs"] == len(pairs)
    if case == "max_buckets":
        assert runner.stats["captures"] > 3 and len(runner.buckets) == 1
    if case == "inference_size":
        assert runner.stats["captures"] == 1 and runner.stats["steps"] == 5
    if case == "buckets":
        assert runner.stats["captures"] == 3 and len(runner.buckets) == 3


@pytest.mark.parametrize("workload", ["gmflow-scale1", "gmflow-scale2-regrefine6"])
def test_mixed_flow_runner_close_to_infer_flow_on_each_pair(workload):
    """the step's batch changes `um_conv2d_tc`'s summation order (README, video flow: 3e-6 of the largest flow at the bench
    sizes), and six refinement iterations on these small frames carry it a little further, so the pair alone agrees to 1e-5
    of its largest flow"""
    m, call = synthetic_model(workload), workload_call(workload, drop=("task",))
    pairs = _pairs(MIX, seed=55)
    runner = MixedSizeFlowRunner(m, CAP, 2, "cuda", padding_factor=32, **BIDIR, **call)
    worst = 0.0
    for i, r in runner.run(pairs):
        a, b = (torch.from_numpy(f).permute(2, 0, 1)[None].float().cuda() for f in pairs[i])
        alone = infer_flow(m, a, b, padding_factor=32, **BIDIR, **call)
        for k in ("flow", "flow_bwd"):
            ref = alone[k][0].cpu()
            assert r[k].shape == ref.shape, (i, k)
            worst = max(worst, ((r[k] - ref).abs().max() / ref.abs().max()).item())
        for k in ("fwd_occ", "bwd_occ"):
            assert (r[k] != alone[k][0].cpu()).float().mean() < 1e-3, (i, k)
    print("largest difference to infer_flow on the pair alone, relative to its largest flow: %.2e" % worst)
    assert worst <= 1e-5


def test_mixed_flow_runner_survives_other_shapes():
    """capture three buckets, evict the module's cached planes with forwards at other batch sizes and shapes, check that
    the runner still holds every buffer its graphs write, then replay bit for bit"""
    m, call = synthetic_model("gmflow-scale2-regrefine6"), workload_call("gmflow-scale2-regrefine6", drop=("task",))
    pairs = _pairs(MIX, seed=70)
    runner = MixedSizeFlowRunner(m, CAP, 2, "cuda", padding_factor=32, visualize=True, **call)
    r1 = {i: {k: v.clone() for k, v in r.items()} for i, r in runner.run(pairs)}
    assert len(runner.buckets) == 3
    captured = {t.data_ptr() for t in m.cached_buffers()}
    captured_keys = set(m._attn_ws) | set(m._pad_ws)
    assert captured
    for n, h, w in [(1, 384, 512), (3, 384, 512), (2, 320, 448), (1, 256, 384), (4, 256, 384)]:
        d = {k: v.cuda() for k, v in synthetic_batch("flow", n, h, w).items()}
        m(d["img0"], d["img1"], **workload_call("gmflow-scale2-regrefine6"))
    assert captured_keys - (set(m._attn_ws) | set(m._pad_ws)), "the runner's planes were not evicted: the scenario was not reached"
    held = {t.data_ptr() for _, _, bufs in runner.buckets.values() for t in bufs}
    assert captured <= held, "cached buffers the runner's graphs write are no longer referenced"
    r2 = {i: {k: v.clone() for k, v in r.items()} for i, r in runner.run(pairs)}
    assert runner.stats["captures"] == 3
    for i in r1:
        assert torch.equal(r1[i]["flow"], r2[i]["flow"]) and torch.equal(r1[i]["vis"], r2[i]["vis"]), i
