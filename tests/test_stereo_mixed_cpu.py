"""Mixed-size stereo streaming without a device: step formation (`_batches` with and without its open-batch limit), the
descriptor tables of a step (`_ragged_step_layout`: offsets, used bytes, fp32 scales, flips, fillers), the ragged ops'
statements against the uniform ones, every argument error of `MixedSizeStereoRunner`, and the C-ABI argument checks of the
three ragged entries."""
import ctypes

import numpy as np
import pytest
import torch

import refops
import refops_ragged
from oracle import disp_viz as OD
from unimatch_b200 import MixedSizeStereoRunner, UniMatch, ops, submission
from unimatch_b200.inference import RAGGED_ITEM, _batches, _ragged_step_layout

ONE = ctypes.c_void_p(1024)          # any non-null address: validation never dereferences it


def _keys(batches):
    return [[i for i, _ in b] for b in batches]


def test_batches_without_limit_is_the_submission_rule():
    items = [(0, "a"), (1, "b"), (2, "a"), (3, "c"), (4, "b"), (5, "a"), (6, "c"), (7, "a")]
    got = _keys(_batches(items, 2, lambda s: s[1]))
    assert got == [[0, 2], [1, 4], [3, 6], [5, 7]]
    assert submission._batches is _batches
    assert _keys(_batches(items, 3, lambda s: s[1])) == [[0, 2, 5], [1, 4], [3, 6], [7]]   # "a" reopened last by 7
    assert _keys(_batches(items, 2, lambda s: s[1], None)) == got
    with pytest.raises(ValueError):
        list(_batches(items, 0, lambda s: s[1]))
    with pytest.raises(ValueError):
        list(_batches(items, 2, lambda s: s[1], 0))


def test_batches_limit_flushes_the_oldest_open_batch():
    items = [(0, "a"), (1, "b"), (2, "c"), (3, "a"), (4, "b"), (5, "b"), (6, "a")]
    # at most 2 open: opening "c" sends "a" ([0]) early, reopening "a" sends "b" ([1]), reopening "b" sends "c" ([2])
    got = _keys(_batches(items, 2, lambda s: s[1], 2))
    assert got == [[0], [1], [2], [4, 5], [3, 6]]
    assert _keys(_batches(items, 3, lambda s: s[1], 1)) == [[0], [1], [2], [3], [4, 5], [6]]
    assert _keys(_batches(items, 3, lambda s: s[1], 3)) == _keys(_batches(items, 3, lambda s: s[1]))
    flat = sorted(i for b in got for i in b)
    assert flat == list(range(len(items)))                        # every item exactly once


def test_step_layout_offsets_scales_and_fillers():
    sizes = [(5, 7), (4, 6), (8, 8)]
    frames, outputs, nbytes, used, results = _ragged_step_layout(sizes, 4, (8, 8), False, False)
    assert frames.dtype == RAGGED_ITEM and RAGGED_ITEM.itemsize == ops.RAGGED_ITEM_BYTES == ctypes.sizeof(ops.RaggedItem)
    assert list(frames["offset"]) == [0, 105, 177, 177, 369, 474, 546, 546]            # lefts, filler, rights, filler
    assert list(frames["h"]) == [5, 4, 8, 8, 5, 4, 8, 8] and list(frames["w"]) == [7, 6, 8, 8, 7, 6, 8, 8]
    assert nbytes == 2 * 3 * (35 + 24 + 64)
    assert list(outputs["offset"][:3]) == [0, 35, 59] and used == 123
    assert outputs["h"][3] == 0 and outputs["w"][3] == 0                                 # the filler is skipped
    assert outputs["scale"][0] == np.float32(7 / 8.0) and outputs["scale"][1] == np.float32(6 / 8.0)
    assert outputs["scale"][2] == 1.0 and not outputs["flags"].any()
    assert results == [[("disp", 0, 5, 7)], [("disp", 35, 4, 6)], [("disp", 59, 8, 8)]]
    # the scale is the driver's ratio rounded to fp32, as the ctypes binding rounds it for um_resize_bilinear
    _, o, _, _, _ = _ragged_step_layout([(370, 1226)], 1, (384, 1232), False, False)
    assert o["scale"][0] == ctypes.c_float(1226 / float(1232)).value


def test_step_layout_right_views():
    sizes = [(5, 7), (8, 8)]
    _, outputs, _, used, results = _ragged_step_layout(sizes, 2, (8, 8), True, False)
    assert list(outputs["offset"]) == [0, 35, 99, 134] and used == 198
    assert list(outputs["flags"]) == [0, 0, ops.RAGGED_FLIP_X, ops.RAGGED_FLIP_X]
    assert results[1] == [("disp", 35, 8, 8), ("disp_right", 134, 8, 8)]
    _, outputs, _, _, _ = _ragged_step_layout(sizes, 2, (8, 8), False, True)
    assert list(outputs["flags"]) == [ops.RAGGED_FLIP_X] * 2


def test_ragged_statements_equal_the_uniform_ops_cpu():
    """the CPU statements place every item where its descriptor says, as the uniform op computes it"""
    refops.register_cpu_kernels()
    g = torch.Generator().manual_seed(5)
    x = torch.randn((3, 1, 6, 9), generator=g)
    items = refops_ragged.table([(0, 4, 5, 1.25, 0), (20, 6, 9, 1.0, 0), (74, 6, 9, 1.0, ops.RAGGED_FLIP_X)])
    out = torch.ops.unimatch_sm100.resize_bilinear_ragged(x, items, 8, 10, 128)
    assert torch.equal(out[:20].view(4, 5), torch.ops.unimatch_sm100.resize_bilinear(x[:1], 4, 5, [1.25], False)[0, 0])
    assert torch.equal(out[20:74].view(6, 9), x[1, 0])
    assert torch.equal(out[74:128].view(6, 9), x[2, 0].flip(-1))
    pics = torch.zeros((3 * 128,), dtype=torch.uint8)
    torch.ops.unimatch_sm100.disparity_to_image_ragged(out, items, pics, 8, 10)
    assert torch.equal(pics[60:222].view(6, 9, 3), torch.from_numpy(OD.vis_disparity(x[1, 0].numpy())))
    assert torch.equal(pics[222:].view(6, 9, 3), torch.from_numpy(OD.vis_disparity(x[2, 0].flip(-1).numpy())))
    frames = torch.randint(0, 256, (3 * (4 * 5 + 6 * 9),), generator=g, dtype=torch.uint8)
    fitems = refops_ragged.table([(0, 4, 5, 1.0, 0), (60, 6, 9, 1.0, 0)])
    planes = torch.ops.unimatch_sm100.frames_to_planar_normalized_ragged(frames, fitems, 8, 10, 6, 9, [0.5] * 3, [0.25] * 3)
    assert torch.equal(planes[1], torch.ops.unimatch_sm100.frames_to_planar_normalized(frames[60:].view(1, 6, 9, 3), 6, 9,
                                                                                       [0.5] * 3, [0.25] * 3)[0])


def test_runner_argument_errors():
    """rejected before any device work"""
    m = UniMatch(num_scales=2, upsample_factor=4).eval()
    for kw in (dict(pred_bidir_disp=True, pred_right_disp=True), dict(return_disp=False), dict(task="flow"), dict(batch=0),
               dict(max_buckets=0), dict(size=(0, 96)), dict(size=(64, -1)), dict(size=(1 << 16, 1 << 16))):
        args = dict(dict(batch=2, size=(64, 96)), **kw)
        with pytest.raises(ValueError):
            MixedSizeStereoRunner(m, args.pop("size"), args.pop("batch"), "cuda", **args)


def test_runner_frame_errors():
    """every frame is checked as it is read, before it is staged; the checks need no device"""
    r = MixedSizeStereoRunner.__new__(MixedSizeStereoRunner)
    r.hmax, r.wmax, r.padding_factor, r.inference_size = 64, 96, 32, None
    ok = np.zeros((40, 90, 3), np.uint8)
    assert r._bucket(r._pair((ok, ok))) == (64, 96)
    for left, right in ((np.zeros((65, 90, 3), np.uint8),) * 2,            # taller than the capacity
                        (np.zeros((40, 97, 3), np.uint8),) * 2,            # wider
                        (ok, np.zeros((40, 91, 3), np.uint8)),             # left and right of different sizes
                        (ok.astype(np.float32), ok.astype(np.float32)),    # not uint8
                        (np.zeros((40, 90), np.uint8),) * 2,               # not [h, w, 3]
                        (np.zeros((40, 90, 4), np.uint8),) * 2):
        with pytest.raises(ValueError):
            r._pair((left, right))
    r.batch, r.max_buckets = 2, 2
    with pytest.raises(ValueError):                                       # raised while steps are formed
        list(r._chunks(enumerate([(ok, ok), (ok, np.zeros((2, 2, 3), np.uint8))])))
    steps = list(r._chunks(enumerate([(ok, ok), (np.zeros((10, 10, 3), np.uint8),) * 2, (ok, ok)])))
    assert [[i for i, _ in s] for s in steps] == [[0, 2], [1]]             # (64, 96) and (32, 32) buckets


def test_ragged_entries_validate_without_a_gpu():
    mean = (ctypes.c_float * 3)(0.5, 0.5, 0.5)
    good = dict(n=2, h_max=8, w_max=8, h=4, w=4, numel=1024)
    for change in (dict(n=0), dict(n=65536), dict(h_max=0), dict(w_max=-1), dict(h=0), dict(w=0), dict(numel=0)):
        a = dict(good, **change)
        rc = ops.LIB.um_frames_to_planar_normalized_ragged(ONE, a["numel"], ONE, ONE, a["n"], a["h_max"], a["w_max"], a["h"],
                                                           a["w"], mean, mean, None)
        assert rc == -22, change
        assert b"um_frames_to_planar_normalized_ragged" in ops.LIB.um_last_error()
        rc = ops.LIB.um_resize_bilinear_ragged(ONE, ONE, a["numel"], ONE, a["n"], a["h"], a["w"], a["h_max"], a["w_max"], None)
        assert rc == -22, change
        assert b"um_resize_bilinear_ragged" in ops.LIB.um_last_error()
        if "h" not in change and "w" not in change:
            rc = ops.LIB.um_disparity_to_image_ragged(ONE, a["numel"], ONE, ONE, ONE, a["n"], a["h_max"], a["w_max"], None)
            assert rc == -22, change
            assert b"um_disparity_to_image_ragged" in ops.LIB.um_last_error()
    assert ops.LIB.um_frames_to_planar_normalized_ragged(ONE, 64, None, ONE, 1, 4, 4, 4, 4, mean, mean, None) == -22
    assert ops.LIB.um_frames_to_planar_normalized_ragged(ONE, 64, ONE, ONE, 1, 4, 4, 4, 4, None, mean, None) == -22
    assert ops.LIB.um_resize_bilinear_ragged(ONE, None, 64, ONE, 1, 4, 4, 4, 4, None) == -22
    assert ops.LIB.um_disparity_to_image_ragged(ONE, 64, ONE, ONE, None, 1, 4, 4, None) == -22          # no scratch
    assert ops.LIB.um_disparity_to_image_ragged(ONE, 64, ONE, ONE, ONE, 1, 1 << 16, 1 << 16, None) == -22  # > 2^31 - 1 px
