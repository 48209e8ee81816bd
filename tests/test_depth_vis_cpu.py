"""Depth colouring without a device: the oracle's plasma table against cv2's and against the table compiled into the
library, the oracle's arithmetic on cases that can be checked by hand, and the argument checks of `um_depth_to_image`,
`depth_to_image` and `DepthSequenceRunner`."""
import ctypes
import math
import os
import re

import numpy as np
import pytest
import torch

from oracle import depth_viz as V
from unimatch_b200 import UniMatch, ops
from unimatch_b200.inference import DepthSequenceRunner, depth_to_image

HERE = os.path.dirname(os.path.abspath(__file__))


def test_plasma_table_rounds_to_cv2_lut():
    cv2 = pytest.importorskip("cv2")
    lut = cv2.applyColorMap(np.arange(256, dtype=np.uint8)[:, None], cv2.COLORMAP_PLASMA)[:, 0, ::-1]     # BGR -> RGB
    assert np.array_equal(np.round(V.PLASMA * 255).astype(np.uint8), lut)
    assert tuple(V.PLASMA[0]) == (0.050383, 0.029803, 0.527975) and tuple(V.PLASMA[-1]) == (0.940015, 0.975158, 0.131326)


def test_library_table_equals_oracle_table():
    src = open(os.path.join(os.path.dirname(HERE), "unimatch_b200", "csrc", "um_misc.cu")).read()
    body = re.search(r"kPlasma\[768\]\s*=\s*\{(.*?)\};", src, flags=re.S).group(1)
    table = np.array([int(v) for v in body.replace(",", " ").split()], np.uint8).reshape(256, 3)
    assert np.array_equal(table, np.floor(V.PLASMA * 255).astype(np.uint8))
    assert np.array_equal(table, V.PLASMA_U8)


def test_constant_map_takes_the_first_colour():
    for value in (2.5, 0.7, -3.0):
        img = V.viz_inverse_depth(np.full((5, 7), value, np.float32))
        assert (img == V.PLASMA_U8[0]).all(), value


def test_one_nan_paints_the_picture_black():
    d = np.random.default_rng(1).uniform(0.5, 10, (6, 9)).astype(np.float32)
    d[2, 3] = np.nan
    assert math.isnan(V.percentile95(V.inverse(d)))
    assert not V.viz_inverse_depth(d).any()


def test_exact_index_takes_rank_k():
    """N = 21: 0.95 * 20 rounds to 19.0 exactly, so vmax is the sorted value at rank 19 and g = 0"""
    assert 0.95 * 20 == 19.0
    inv = np.random.default_rng(2).permutation(np.arange(1, 22, dtype=np.float32)).reshape(3, 7)
    assert V.percentile95(inv) == 20.0
    t = V.normalized(inv)
    assert t.dtype == np.float32
    assert np.array_equal(t, (inv - np.float32(1)) / np.float32(19))


def test_ties_across_ranks_k_and_k_plus_1():
    """N = 100: k = 94, g = 0.05 (rounded); a run of equal values over ranks 92..97, then a and b apart"""
    idx = 0.95 * 99
    k, g = math.floor(idx), idx - math.floor(idx)
    assert k == 94
    inv = np.concatenate([np.arange(92) / 128, np.full(6, 7.0), [20.0, 30.0]]).astype(np.float32)      # sorted
    got = V.percentile95(np.random.default_rng(3).permutation(inv))
    assert got == 7.0 * (1 - g) + 7.0 * g and abs(got - 7.0) <= 1e-15 * 7
    inv[95:98] = 9.0                                         # a = 7 (rank 94), b = 9 (rank 95)
    assert V.percentile95(np.random.default_rng(4).permutation(inv)) == 7.0 * (1 - g) + 9.0 * g


def test_values_above_vmax_take_the_last_colour():
    d = np.float32(1) / np.arange(1, 101, dtype=np.float32).reshape(10, 10)
    inv = V.inverse(d)
    vmax = V.percentile95(inv)
    img = V.viz_inverse_depth(d)
    above = inv > vmax
    assert above.sum() == 5
    assert (img[above] == V.PLASMA_U8[255]).all()
    assert (img[inv == 1] == V.PLASMA_U8[0]).all()
    i = V.colour_index(V.normalized(inv))
    assert i.min() == 0 and i.max() == 255 and (np.diff(i.ravel()) >= 0).all()


def test_zero_depth_follows_the_arithmetic():
    """inv = +inf: with g = 0 and b = +inf, vmax = a * 1 + inf * 0 is NaN and the picture black; with g > 0 vmax is +inf,
    the finite pixels take t = 0 and the infinite ones NaN (black)"""
    d = np.random.default_rng(5).uniform(0.5, 10, 21).astype(np.float32).reshape(3, 7)
    d[1, 1] = 0
    assert math.isnan(V.percentile95(V.inverse(d))) and not V.viz_inverse_depth(d).any()
    d = np.random.default_rng(6).uniform(0.5, 10, 100).astype(np.float32).reshape(10, 10)
    d.ravel()[:5] = 0
    assert V.percentile95(V.inverse(d)) == math.inf
    img = V.viz_inverse_depth(d)
    assert not img.reshape(-1, 3)[:5].any() and (img.reshape(-1, 3)[5:] == V.PLASMA_U8[0]).all()


def test_oracle_inverse_equals_torch_reciprocal():
    g = np.random.default_rng(7)
    d = np.concatenate([g.uniform(0.5, 10, 4096), g.uniform(-10, 10, 4096), 10.0 ** g.uniform(-40, 38, 4096),
                        [0.0, -0.0, np.inf, -np.inf, np.nan, 1e-45, 3e-39]]).astype(np.float32)
    ref = (1. / torch.from_numpy(d)).numpy()
    assert np.array_equal(V.inverse(d).view(np.uint32), ref.view(np.uint32))


def test_depth_to_image_bad_arguments_are_reported_without_a_gpu():
    one = ctypes.c_void_p(1024)
    good = dict(row=3 * 8, image=3 * 8 * 4, n=2, h=4, w=8)
    assert ops.LIB.um_depth_to_image(None, one, 24, 96, one, 2, 4, 8, None) == -22
    assert b"um_depth_to_image" in ops.LIB.um_last_error()
    assert ops.LIB.um_depth_to_image(one, None, 24, 96, one, 2, 4, 8, None) == -22
    assert ops.LIB.um_depth_to_image(one, one, 24, 96, None, 2, 4, 8, None) == -22          # no scratch
    for change in (dict(row=3 * 8 - 1), dict(image=3 * 8 * 4 - 1), dict(n=0), dict(h=0), dict(w=-1), dict(n=-3)):
        a = dict(good, **change)
        rc = ops.LIB.um_depth_to_image(one, one, a["row"], a["image"], one, a["n"], a["h"], a["w"], None)
        assert rc == -22, change
        assert b"um_depth_to_image" in ops.LIB.um_last_error(), change


def test_depth_to_image_shape_errors():
    for bad in (torch.zeros(5), torch.zeros((1, 1, 4, 5)), torch.zeros((2, 0, 5)), torch.zeros((4, 5), dtype=torch.int32)):
        with pytest.raises(ValueError):
            depth_to_image(bad)
    with pytest.raises(ValueError):
        depth_to_image(torch.ones((2, 4, 5)), torch.zeros((2, 4, 5, 3), dtype=torch.uint8)[:1])
    with pytest.raises(ValueError):
        depth_to_image(torch.ones((2, 4, 5)), torch.zeros((2, 4, 5, 3)))


def test_depth_runner_rejects_nothing_to_return():
    """rejected before any device work (the constructor would otherwise create a CUDA stream first)"""
    m = UniMatch(num_scales=1, upsample_factor=8).eval()
    with pytest.raises(ValueError):
        DepthSequenceRunner(m, (64, 96), 2, "cuda", np.eye(3, dtype=np.float32), return_depth=False)
