"""Mixed-size flow streaming without a device: the descriptor tables of a flow step (`_flow_step_layout`: offsets, used
prefixes, the two fp32 component scales, transpose flags, fillers, the bidirectional and occlusion layouts), the
`pred_bwd_flow` packing order, bucketing of portrait and landscape pairs, the ragged flow ops' statements against the uniform
ones, every argument error of `MixedSizeFlowRunner`, and the C-ABI argument checks of the new entries."""
import ctypes

import numpy as np
import pytest
import torch

import refops
import refops_flow_ragged
import refops_ragged
from oracle import flow_viz as OV
from unimatch_b200 import MixedSizeDepthRunner, MixedSizeFlowRunner, MixedSizeStereoRunner, UniMatch, ops
from unimatch_b200.inference import RAGGED_ITEM, _MixedSizeRunner, _flow_step_layout

ONE = ctypes.c_void_p(1024)          # any non-null address: validation never dereferences it
T = ops.RAGGED_TRANSPOSE
_OPS = torch.ops.unimatch_sm100


def test_flow_step_layout_offsets_scales_and_fillers():
    sizes = [(5, 7), (8, 4), (4, 8)]                       # landscape, portrait (the model sees 4x8), at the inference size
    frames, planes, flows, pictures, masks, nbytes, used, results = _flow_step_layout(sizes, 4, (4, 8), False, False)
    assert frames.dtype == RAGGED_ITEM
    assert list(frames["offset"]) == [0, 105, 201, 201, 297, 402, 498, 498]     # first frames, filler, second frames, filler
    assert list(frames["h"]) == [5, 8, 4, 4] * 2 and list(frames["w"]) == [7, 4, 8, 8] * 2
    assert list(frames["flags"]) == [0, T, 0, 0] * 2
    assert nbytes == 2 * 3 * (35 + 32 + 32)
    # u plane, v plane of each pair back to back; the filler pair's planes are empty items
    assert list(planes["offset"]) == [0, 35, 70, 102, 134, 166, 0, 0]
    assert list(planes["h"]) == [5, 5, 8, 8, 4, 4, 0, 0] and list(planes["w"]) == [7, 7, 4, 4, 8, 8, 0, 0]
    assert list(planes["flags"]) == [0, 0, T, T, 0, 0, 0, 0]
    assert planes["scale"][0] == np.float32(7 / 8) and planes["scale"][1] == np.float32(5 / 4)
    assert planes["scale"][2] == 1.0 and planes["scale"][3] == 1.0            # portrait 8x4 is the inference size transposed
    assert planes["scale"][4] == 1.0 and planes["scale"][5] == 1.0
    assert list(flows["offset"]) == [0, 70, 134, 0] and list(flows["h"]) == [5, 8, 4, 0] and not flows["flags"].any()
    assert list(pictures["offset"]) == [0, 105, 201, 0] and list(pictures["w"]) == [7, 4, 8, 0]
    assert len(masks) == 0
    assert used == {"flow": 198, "vis": 297, "occ": 0}
    assert results[1] == [("flow", "flow", 70, (2, 8, 4)), ("vis", "vis", 105, (8, 4, 3))]


def test_flow_step_layout_scales_are_the_drivers_fp32_values():
    """`_flow_outputs` passes [ori_w / size_w, ori_h / size_h] as Python floats, which the binding rounds to fp32"""
    _, planes, _, _, _, _, _, _ = _flow_step_layout([(375, 1242), (1242, 375)], 2, (384, 1248), False, False)
    su, sv = ctypes.c_float(1242 / 1248).value, ctypes.c_float(375 / 384).value
    assert [float(s) for s in planes["scale"]] == [su, sv, su, sv]           # the portrait pair is scaled as its transpose
    assert list(planes["flags"]) == [0, 0, T, T]


def test_flow_step_layout_bidirectional_and_masks():
    sizes = [(5, 7), (8, 4)]
    _, planes, flows, pictures, masks, _, used, results = _flow_step_layout(sizes, 3, (8, 8), True, True)
    assert len(planes) == 12 and len(flows) == 6 and len(pictures) == 6 and len(masks) == 6
    # forward flows of the step, then its backward flows, as the model returns them; fillers empty
    assert list(flows["offset"]) == [0, 70, 0, 134, 204, 0] and list(flows["h"]) == [5, 8, 0, 5, 8, 0]
    assert list(planes["offset"][6:10]) == [134, 169, 204, 236]
    assert list(pictures["offset"]) == [0, 105, 0, 201, 306, 0]
    assert list(masks["offset"]) == [0, 35, 0, 67, 102, 0] and list(masks["w"]) == [7, 4, 0, 7, 4, 0]
    assert used == {"flow": 268, "vis": 402, "occ": 134}
    assert [v[0] for v in results[0]] == ["flow", "vis", "flow_bwd", "vis_bwd", "fwd_occ", "bwd_occ"]
    assert results[1][2] == ("flow_bwd", "flow", 204, (2, 8, 4)) and results[1][5] == ("bwd_occ", "occ", 102, (8, 4))


def _bare(**kw):
    r = MixedSizeFlowRunner.__new__(MixedSizeFlowRunner)
    r.hmax, r.wmax, r.padding_factor, r.inference_size, r.batch, r.max_buckets = 96, 96, 32, None, 2, 2
    r.bidir = r.bwd = r.check = False
    r.buffers = ("flow",)
    for k, v in kw.items():
        setattr(r, k, v)
    return r


def test_pred_bwd_flow_swaps_the_packing_order():
    a, b, c, d = (np.full((4, 6, 3), v, np.uint8) for v in range(4))
    pairs = [_bare()._pair(p) for p in ((a, b), (c, d))]
    assert [int(f[0, 0, 0]) for f in _bare()._frame_order(pairs)] == [0, 2, 1, 3]
    assert [int(f[0, 0, 0]) for f in _bare(bwd=True)._frame_order(pairs)] == [1, 3, 0, 2]


def test_layout_keeps_only_the_returned_buffers():
    table, used, views = _bare(buffers=("vis",))._layout([(5, 7)], (32, 32))
    assert table.dtype == RAGGED_ITEM and len(table) == 2 * 2 + 4 * 2
    assert views == [[("vis", "vis", 0, (5, 7, 3))]]
    _, _, views = _bare(bidir=True, check=True, buffers=("flow", "occ"))._layout([(5, 7)], (32, 32))
    assert [v[0] for v in views[0]] == ["flow", "flow_bwd", "fwd_occ", "bwd_occ"]


def test_portrait_and_landscape_share_a_bucket_and_max_buckets_flushes():
    r = _bare()

    def z(h, w):
        return (np.zeros((h, w, 3), np.uint8),) * 2

    assert r._bucket(r._pair(z(40, 90))) == r._bucket(r._pair(z(90, 40))) == (64, 96)
    assert _bare(inference_size=(32, 64))._bucket(r._pair(z(90, 40))) == (32, 64)
    steps = list(r._chunks(enumerate([z(40, 90), z(10, 10), z(90, 40), z(60, 20), z(10, 12)])))
    # (64, 96) is filled by the landscape and the portrait pair, (32, 32) by pairs 1 and 4; (32, 64) is sent at the end
    assert [[i for i, _ in s] for s in steps] == [[0, 2], [1, 4], [3]]
    steps = list(_bare(max_buckets=1)._chunks(enumerate([z(40, 90), z(10, 10), z(90, 40)])))
    assert [[i for i, _ in s] for s in steps] == [[0], [1], [2]]           # opening a second bucket sends the open step early


def test_both_mixed_runners_share_one_implementation():
    for name in ("_capture_bucket", "_device_step", "_prepare_graphs", "_chunks", "_stage_host", "_download", "_results",
                 "_reset_inputs", "run", "_capture_graphs", "_frame", "_sizes", "_table"):
        assert getattr(MixedSizeFlowRunner, name) is getattr(MixedSizeStereoRunner, name) is getattr(_MixedSizeRunner, name)
    for name in ("_capture_bucket", "_device_step", "_chunks", "_download", "_results", "run", "_frame", "_bucket",
                 "_frame_order", "_layout", "_resize_back", "_returned"):
        assert getattr(MixedSizeDepthRunner, name) is getattr(MixedSizeStereoRunner, name) is getattr(_MixedSizeRunner, name)


def test_runner_argument_errors():
    """rejected before any device work"""
    m = UniMatch(num_scales=1, upsample_factor=8).eval()
    for kw in (dict(fwd_bwd_consistency_check=True), dict(return_flow=False), dict(task="stereo"), dict(batch=0),
               dict(max_buckets=0), dict(size=(0, 96)), dict(size=(64, -1)), dict(size=(1 << 16, 1 << 16)),
               dict(return_flow=False, visualize=True, pred_bidir_flow=True, fwd_bwd_consistency_check=True),
               dict(size=(1, 64), pred_bidir_flow=True, fwd_bwd_consistency_check=True)):
        args = dict(dict(batch=2, size=(64, 96)), **kw)
        with pytest.raises(ValueError):
            MixedSizeFlowRunner(m, args.pop("size"), args.pop("batch"), "cuda", **args)


def test_runner_frame_errors():
    """every frame is checked as it is read, before it is staged; the checks need no device"""
    r = _bare(hmax=64)
    ok = np.zeros((40, 90, 3), np.uint8)
    r._pair((ok, ok))
    for first, second in ((np.zeros((65, 90, 3), np.uint8),) * 2,          # taller than the capacity
                          (np.zeros((40, 97, 3), np.uint8),) * 2,          # wider
                          (ok, np.zeros((40, 91, 3), np.uint8)),           # two sizes in one pair
                          (ok.astype(np.float32), ok.astype(np.float32)),  # not uint8
                          (np.zeros((40, 90), np.uint8),) * 2,             # not [h, w, 3]
                          (np.zeros((40, 90, 4), np.uint8),) * 2):
        with pytest.raises(ValueError):
            r._pair((first, second))
    thin = np.zeros((1, 90, 3), np.uint8)
    r._pair((thin, thin))
    with pytest.raises(ValueError):                                         # the occlusion check samples a grid of >= 2 x 2
        _bare(check=True)._pair((thin, thin))
    with pytest.raises(ValueError):                                         # raised while steps are formed
        list(r._chunks(enumerate([(ok, ok), (ok, np.zeros((2, 2, 3), np.uint8))])))


def test_ragged_flow_statements_equal_the_uniform_ops_cpu():
    """the CPU statements place every item where its descriptors say, as the uniform op computes it"""
    refops.register_cpu_kernels()
    g = torch.Generator().manual_seed(5)
    frames = torch.randint(0, 256, (3 * (4 * 5 + 9 * 6),), generator=g, dtype=torch.uint8)
    fitems = refops_ragged.table([(0, 4, 5, 1.0, 0), (60, 9, 6, 1.0, T)])
    planes = _OPS.frames_to_planar_ragged(frames, fitems, 10, 10, 6, 9)
    assert torch.equal(planes[0], _OPS.frames_to_planar(frames[:60].view(1, 4, 5, 3), 6, 9, False)[0])
    assert torch.equal(planes[1], frames[60:].view(9, 6, 3).permute(2, 1, 0).float())        # exactly its transpose
    x = torch.randn((4, 1, 6, 9), generator=g)
    items = refops_ragged.table([(0, 4, 5, 1.25, 0), (20, 4, 5, 0.5, 0), (40, 9, 6, 1.0, T), (94, 9, 6, 1.0, T)])
    flow = refops_flow_ragged.resize_bilinear_ragged(x, items, 10, 10, 148)
    assert torch.equal(flow[:40].view(2, 4, 5), _OPS.resize_bilinear(x[:2].view(1, 2, 6, 9), 4, 5, [1.25, 0.5], False)[0])
    assert torch.equal(flow[40:].view(2, 9, 6), x[2:, 0].transpose(-2, -1))
    fl = refops_ragged.table([(0, 4, 5, 1.0, 0), (40, 9, 6, 1.0, 0)])
    pic = refops_ragged.table([(0, 4, 5, 1.0, 0), (60, 9, 6, 1.0, 0)])
    pics = torch.zeros((222,), dtype=torch.uint8)
    _OPS.flow_to_image_ragged(flow, fl, pics, pic, 10, 10)
    assert np.array_equal(pics[60:].view(9, 6, 3).numpy(), OV.flow_to_image_batch(flow[40:].view(1, 2, 9, 6).numpy())[0])
    both = torch.cat((flow[40:], -flow[40:]))
    occ = torch.full((2 * 54 + 3,), 7.0)
    _OPS.fb_consistency_ragged(both, refops_ragged.table([(0, 9, 6, 1.0, 0), (108, 9, 6, 1.0, 0)]), occ,
                               refops_ragged.table([(0, 9, 6, 1.0, 0), (57, 9, 6, 1.0, 0)]), 10, 10, 0.01, 0.5)
    ref = _OPS.fb_consistency(both[:108].view(1, 2, 9, 6), both[108:].view(1, 2, 9, 6), 0.01, 0.5)
    assert torch.equal(occ[:54].view(9, 6), ref[0][0]) and torch.equal(occ[57:111].view(9, 6), ref[1][0])
    assert (occ[54:57] == 7).all()


def test_new_entries_are_exported_and_validate_without_a_gpu():
    for name in ("um_frames_to_planar_ragged", "um_flow_to_image_ragged", "um_fb_consistency_ragged"):
        assert name in ops.SYMBOLS and hasattr(ops.LIB, name)
    assert ops.LIB.um_abi_version() == 4 and T == 2
    good = dict(n=2, h_max=8, w_max=8, h=4, w=4, numel=1024)
    for change in (dict(n=0), dict(n=65536), dict(h_max=0), dict(w_max=-1), dict(h=0), dict(w=0), dict(numel=0)):
        a = dict(good, **change)
        rc = ops.LIB.um_frames_to_planar_ragged(ONE, a["numel"], ONE, ONE, a["n"], a["h_max"], a["w_max"], a["h"], a["w"], None)
        assert rc == -22, change
        assert b"um_frames_to_planar_ragged" in ops.LIB.um_last_error()
        if "h" in change or "w" in change:
            continue
        rc = ops.LIB.um_flow_to_image_ragged(ONE, a["numel"], ONE, ONE, 1024, ONE, ONE, a["n"], a["h_max"], a["w_max"], None)
        assert rc == -22, change
        assert b"um_flow_to_image_ragged" in ops.LIB.um_last_error()
        rc = ops.LIB.um_fb_consistency_ragged(ONE, a["numel"], ONE, 0.01, 0.5, ONE, 1024, ONE, a["n"], a["h_max"], a["w_max"], None)
        assert rc == -22, change
        assert b"um_fb_consistency_ragged" in ops.LIB.um_last_error()
    assert ops.LIB.um_frames_to_planar_ragged(ONE, 64, None, ONE, 1, 4, 4, 4, 4, None) == -22
    assert ops.LIB.um_frames_to_planar_ragged(None, 64, ONE, ONE, 1, 4, 4, 4, 4, None) == -22
    assert ops.LIB.um_flow_to_image_ragged(ONE, 64, ONE, ONE, 0, ONE, ONE, 1, 4, 4, None) == -22            # no picture bytes
    assert ops.LIB.um_flow_to_image_ragged(ONE, 64, ONE, ONE, 64, None, ONE, 1, 4, 4, None) == -22          # no picture table
    assert ops.LIB.um_flow_to_image_ragged(ONE, 64, ONE, ONE, 64, ONE, None, 1, 4, 4, None) == -22          # no scratch
    assert ops.LIB.um_fb_consistency_ragged(ONE, 64, ONE, 0.01, 0.5, None, 64, ONE, 1, 4, 4, None) == -22
    assert ops.LIB.um_fb_consistency_ragged(ONE, 64, ONE, 0.01, 0.5, ONE, 64, ONE, 1, 1, 4, None) == -22    # capacity below 2 x 2
    assert ops.LIB.um_fb_consistency_ragged(ONE, 64, ONE, 0.01, 0.5, ONE, 64, ONE, 1, 1 << 16, 1 << 16, None) == -22
