"""Depth colouring on the device, bit for bit against the oracle (oracle/depth_viz.py): a full-size batch, odd shapes,
order statistics placed to stress the radix select, non-finite and negative depths, strided pictures, graph replay, and
`DepthSequenceRunner(visualize=True)` against the oracle applied to the runner's own depths."""
import math

import numpy as np
import pytest
import torch

from oracle import depth_viz as V
from unimatch_b200.inference import DepthSequenceRunner, depth_to_image
from unimatch_b200.synthetic import synthetic_model, synthetic_posed_sequence, workload_call

pytestmark = pytest.mark.gpu


def _check(depth, what=""):
    """depth: CPU float32 [N,H,W] -> the device pictures, asserted equal to the oracle's"""
    got = depth_to_image(depth.cuda()).cpu().numpy()
    ref = V.viz_inverse_depth_batch(depth.numpy())
    bad = (got != ref).any(-1)
    assert not bad.any(), (what, int(bad.sum()), np.argwhere(bad)[:5].tolist())
    return ref


def _smooth(n, h, w, seed, lo=0.5, hi=10.0):
    g = torch.Generator().manual_seed(seed)
    coarse = torch.rand((n, 1, max(h // 24, 2), max(w // 24, 2)), generator=g)
    d = torch.nn.functional.interpolate(coarse, size=(h, w), mode="bilinear", align_corners=True)[:, 0]
    return (lo + (hi - lo) * d).float().contiguous()


def _keys(inv):
    u = np.asarray(inv, np.float32).view(np.uint32).astype(np.int64)
    return np.where(u & 0x80000000, ~u & 0xffffffff, u | 0x80000000)


def _ranked(h, w, inv_a, inv_b, seed):
    """a depth map [h,w] whose sorted inverse depths hold inv_a at rank k and inv_b at rank k+1 (k = floor(0.95 (N-1)));
    the depths are 1 / inv, with inv chosen so that 1 / (1 / inv) == inv"""
    n = h * w
    k = math.floor(0.95 * (n - 1))
    g = np.random.default_rng(seed)
    below = g.uniform(0.2, 0.9, k) * min(inv_a, 1.0) if inv_a > 0 else inv_a - g.uniform(0.5, 4.0, k)
    above = inv_b + g.uniform(0.1, 3.0, n - k - 2) * max(abs(inv_b), 1.0)
    inv = np.concatenate([below, [inv_a, inv_b], above]).astype(np.float32)
    d = np.float32(1) / inv
    inv = V.inverse(d)
    s = np.sort(inv)
    assert s[k] == np.float32(inv_a) and s[k + 1] == np.float32(inv_b)
    return torch.from_numpy(g.permutation(d).reshape(h, w))


def _round_trip(x):
    """the first float32 at or above x whose inverse's inverse is itself"""
    x = np.float32(x)
    while np.float32(1) / (np.float32(1) / x) != x:
        x = np.nextafter(x, np.float32(np.inf))
    return x


def test_depth_to_image_full_size_batch():
    """16 x 480 x 640 (a pred_bidir_depth runner step of 8 ScanNet pairs), smooth depths in [0.5, 10], against the oracle"""
    depth = _smooth(16, 480, 640, seed=41)
    _check(depth, "full size")
    dd = depth.cuda()
    out = depth_to_image(dd)
    for _ in range(3):
        depth_to_image(dd, out)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(50):
        depth_to_image(dd, out)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 50
    nbytes = dd.numel() * (4 * 4 + 4 + 3)          # depth read by four select passes and the colouring, picture written once
    print("depth_to_image 16x480x640 on %s: %.4f ms, %.1f MB moved, %.0f GB/s" % (torch.cuda.get_device_name(), ms,
                                                                                 nbytes / 1e6, nbytes / ms / 1e6))


@pytest.mark.parametrize("shape", [(3, 37, 53), (1, 1, 1), (2, 1, 7)])
def test_depth_to_image_odd_shapes(shape):
    g = torch.Generator().manual_seed(sum(shape))
    _check((0.5 + 9.5 * torch.rand(shape, generator=g)).float(), shape)


def test_depth_to_image_adversarial_ranks():
    a = _round_trip(1.25)
    b = a
    for _ in range(200):                           # the next value above a that round-trips: they differ in the low bits
        b = _round_trip(np.nextafter(b, np.float32(np.inf)))
        if b != a:
            break
    assert (_keys(a) ^ _keys(b)) < 256 and a != b
    ka, kb = _keys(_round_trip(0.75)), _keys(_round_trip(3.0))
    assert (ka >> 24) != (kb >> 24)
    maps = {
        "low_bits": _ranked(480, 640, a, b, seed=1),
        "low_bits_small": _ranked(10, 10, a, b, seed=2),
        "top_digit": _ranked(480, 640, _round_trip(0.75), _round_trip(3.0), seed=3),
        "top_digit_odd": _ranked(37, 53, _round_trip(0.75), _round_trip(3.0), seed=4),
        "negative_ranks": _ranked(61, 67, _round_trip(-2.0), _round_trip(-0.5), seed=5),
        "sign_change": _ranked(61, 67, _round_trip(-0.5), _round_trip(0.5), seed=6),
    }
    ties = _smooth(1, 480, 640, seed=7)[0]         # a run of equal depths straddling rank k
    order = torch.argsort(1.0 / ties.ravel())
    k = math.floor(0.95 * (ties.numel() - 1))
    ties.view(-1)[order[k - 40:k + 41]] = ties.view(-1)[order[k]].item()
    maps["ties"] = ties
    for name, d in maps.items():
        _check(d[None].contiguous(), name)


def test_depth_to_image_non_finite_and_negative():
    base = _smooth(8, 96, 128, seed=9)
    base[0] = 2.5                                  # all pixels equal: the first colour
    base[1, 10, 20] = float("nan")                 # black
    base[2, 50, 60] = 0.0                          # inv = +inf above vmax: the last colour
    base[3].view(-1)[::10] = 0.0                   # 10% zeros: vmax = +inf, finite pixels t = 0, zeros NaN (black)
    base[4] = -base[4]                             # negative depths throughout
    base[5, :48] = -base[5, :48]                   # both signs
    base[6, 5, 5] = -0.0                           # inv = -inf as the minimum: every t is NaN (black)
    base[7] = float("inf")                         # inv = 0 everywhere: constant
    ref = _check(base, "non-finite")
    assert (ref[0] == V.PLASMA_U8[0]).all() and not ref[1].any() and not ref[6].any() and (ref[7] == V.PLASMA_U8[0]).all()
    assert (ref[2, 50, 60] == V.PLASMA_U8[255]).all()
    small = torch.rand((2, 3, 7), generator=torch.Generator().manual_seed(3)) + 0.5     # N = 21: g = 0
    small[0, 1, 1] = 0.0                           # b = +inf times g = 0: NaN vmax, black
    small[1, 0, 0] = 0.0
    small[1, 2, 6] = 0.0
    ref = _check(small.float(), "g = 0 with zeros")
    assert not ref.any()


def test_depth_to_image_strided_output():
    depth = _smooth(2, 37, 53, seed=11)
    ref = V.viz_inverse_depth_batch(depth.numpy())
    dd = depth.cuda()
    big = torch.zeros((2, 37, 2 * 53, 3), dtype=torch.uint8, device="cuda")
    depth_to_image(dd, big[:, :, 53:])
    assert np.array_equal(big[:, :, 53:].cpu().numpy(), ref) and not big[:, :, :53].any()
    tall = torch.zeros((3, 40, 53, 3), dtype=torch.uint8, device="cuda")       # 2 images into 3 slots of 3 extra rows
    depth_to_image(dd, tall[:2, :37])
    assert np.array_equal(tall[:2, :37].cpu().numpy(), ref) and not tall[:, 37:].any() and not tall[2].any()
    one = torch.zeros((37, 60, 3), dtype=torch.uint8, device="cuda")           # [H,W] into a [H,W,3] view
    depth_to_image(dd[1], one[:, 7:])
    assert np.array_equal(one[:, 7:].cpu().numpy(), ref[1]) and not one[:, :7].any()


def test_depth_to_image_graph_replay():
    first, second = _smooth(4, 120, 160, seed=12), _smooth(4, 120, 160, seed=13, lo=-3.0, hi=8.0)
    static = first.cuda()
    out = torch.empty((4, 120, 160, 3), dtype=torch.uint8, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        depth_to_image(static, out)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        depth_to_image(static, out)
    for d in (second, first, second):
        static.copy_(d)
        graph.replay()
        torch.cuda.synchronize()
        eager = depth_to_image(d.cuda()).cpu()
        assert torch.equal(out.cpu(), eager)
        assert np.array_equal(eager.numpy(), V.viz_inverse_depth_batch(d.numpy()))


def test_depth_sequence_runner_pictures():
    """11 frames of 90x150, batch 4 (steps of 4 / 4 / 2 + 2 repeats), pred_bidir_depth: the pictures are the oracle's on the
    runner's own depths, graph replay equals eager bit for bit, and return_depth=False sends back the same pictures alone"""
    m = synthetic_model("gmdepth-scale1-regrefine1")
    kw = workload_call("gmdepth-scale1-regrefine1", drop=("task", "min_depth", "max_depth", "num_depth_candidates"))
    frames, K, poses = synthetic_posed_sequence(11, 90, 150, seed=21)
    items = list(zip(frames.numpy(), poses.numpy()))
    runs = {}
    for use_graph, return_depth in ((False, True), (True, True), (True, False)):
        runner = DepthSequenceRunner(m, (90, 150), 4, "cuda", K, use_graph=use_graph, pred_bidir_depth=True, visualize=True,
                                     return_depth=return_depth, **kw)
        runs[use_graph, return_depth] = [{k: v.clone() for k, v in r.items()} for r in runner.run(items)]
    for res in runs.values():
        assert len(res) == 10
    for (use_graph, return_depth), res in runs.items():
        for t, r in enumerate(res):
            assert set(r) == ({"depth", "depth_bwd", "vis", "vis_bwd"} if return_depth else {"vis", "vis_bwd"})
            assert r["vis"].shape == (90, 150, 3) and r["vis"].dtype == torch.uint8
            if return_depth:
                assert np.array_equal(r["vis"].numpy(), V.viz_inverse_depth(r["depth"].numpy())), (use_graph, t)
                assert np.array_equal(r["vis_bwd"].numpy(), V.viz_inverse_depth(r["depth_bwd"].numpy())), (use_graph, t)
    for a, b, c in zip(runs[False, True], runs[True, True], runs[True, False]):
        for k in ("depth", "depth_bwd", "vis", "vis_bwd"):
            assert torch.equal(a[k], b[k]), k
        assert torch.equal(b["vis"], c["vis"]) and torch.equal(b["vis_bwd"], c["vis_bwd"])
