"""Stereo scene flow without a GPU: the numpy statement of the disparity warp and of the KITTI 2015 counts
(tests/refops_sceneflow.py) on analytic cases and hand-made maps, the results dict formed from a count table, the argument
checks that run before any device call (Python and C ABI), and the submission's file names."""
import ctypes

import numpy as np
import pytest
import torch

import refops_sceneflow as R
from unimatch_b200 import ops
from unimatch_b200.evaluation import _scene_flow_fields, scene_flow_results, validate_scene_flow
from unimatch_b200.inference import SceneFlowRunner, infer_scene_flow, warp_disparity
from unimatch_b200.submission import scene_flow_name
from unimatch_b200.synthetic import synthetic_stereo_video


# ---- the warp ----------------------------------------------------------------------------------------------------------
def _plane(h, w, a, b, c):
    """disparity of a plane, a x + b y + c, at every pixel"""
    ys, xs = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing="ij")
    return a * xs + b * ys + c


def test_translating_plane_warp_is_exact():
    """A fronto-parallel plane (constant disparity) moving in x and y, and a slanted plane read at a sub-pixel shift: inside
    the frame the bilinear sample of a plane is the plane, so disp_1 is known exactly."""
    h, w = 9, 13
    d = np.full((1, h, w), 17.25)
    flow = np.zeros((1, 2, h, w))
    flow[:, 0], flow[:, 1] = 2.0, -1.0
    for dt in (np.float64, np.float32):
        out, inside = R.warp_disparity(d, flow, dt)
        assert np.array_equal(out, d.astype(dt))
        assert inside[0, 1:, :w - 2].all() and not inside[0, 0].any() and not inside[0, :, w - 2:].any()
    slanted = _plane(h, w, 0.5, 0.25, 4.0)[None]
    flow[:, 0], flow[:, 1] = 1.5, 0.75
    out, inside = R.warp_disparity(slanted, flow)
    expect = _plane(h, w, 0.5, 0.25, 4.0 + 0.5 * 1.5 + 0.25 * 0.75)[None]
    assert np.allclose(out[inside], expect[inside], rtol=0, atol=1e-6)
    assert np.abs(R.warp_disparity(slanted, flow, np.float32)[0] - out).max() <= 1e-5


@pytest.mark.parametrize("side", ["left", "right", "top", "bottom"])
def test_points_leaving_each_border_take_the_nearest_in_frame_value(side):
    """A point past a border is out of frame and samples the border (padding_mode='border'), so disp_1 stays dense."""
    h, w = 6, 8
    d = _plane(h, w, 1.0, 10.0, 1.0)[None]
    flow = np.zeros((1, 2, h, w))
    axis, shift = {"left": (0, -20.0), "right": (0, 20.0), "top": (1, -20.0), "bottom": (1, 20.0)}[side]
    flow[:, axis] = shift
    out, inside = R.warp_disparity(d, flow)
    assert not inside.any()
    if axis == 0:
        col = 0 if shift < 0 else w - 1
        assert np.array_equal(out[0], np.repeat(d[0][:, col:col + 1], w, axis=1))
    else:
        row = 0 if shift < 0 else h - 1
        assert np.array_equal(out[0], np.repeat(d[0][row:row + 1], h, axis=0))
    exact = np.zeros((1, 2, h, w))                       # exactly on the last row / column: still inside
    exact[:, axis] = (w - 1 if axis == 0 else h - 1) - (np.arange(w)[None] if axis == 0 else np.arange(h)[:, None])
    assert R.warp_disparity(d, exact)[1].all()


def test_nan_flow_is_out_of_frame_and_clamps_to_zero():
    h, w = 4, 5
    d = _plane(h, w, 1.0, 7.0, 3.0)[None].astype(np.float32)
    flow = np.zeros((1, 2, h, w), np.float32)
    flow[0, 0, 1, 2] = np.nan                            # x NaN: x clamps to 0
    flow[0, 1, 2, 3] = np.nan                            # y NaN: y clamps to 0
    flow[0, :, 3, 4] = np.inf                            # +inf clamps to the last column / row
    for dt in (np.float64, np.float32):
        out, inside = R.warp_disparity(d, flow, dt)
        assert not inside[0, 1, 2] and not inside[0, 2, 3] and not inside[0, 3, 4]
        assert out[0, 1, 2] == d[0, 1, 0] and out[0, 2, 3] == d[0, 0, 3] and out[0, 3, 4] == d[0, h - 1, w - 1]
        assert inside.sum() == h * w - 3


# ---- the counts --------------------------------------------------------------------------------------------------------
def _gt(h, w, disp=10.0, flow=(1.0, 0.0)):
    f = np.zeros((1, 2, h, w), np.float32)
    f[:, 0], f[:, 1] = flow
    return {"disp0": np.full((1, h, w), disp, np.float32), "disp1": np.full((1, h, w), disp, np.float32), "flow": f,
            "flow_valid": np.ones((1, h, w), np.float32)}


def _pred(gt):
    return gt["disp0"].copy(), gt["disp1"].copy(), gt["flow"].copy()


def _c(t, s, r, m, k):
    return int(t[0, R.sf_col(s, r, m, k)])


def test_one_outlier_of_each_kind():
    h, w = 2, 3
    gt = _gt(h, w)
    d0, d1, fl = _pred(gt)
    d0[0, 0, 0] += 4.0                                   # D1 outlier (4 > 3, 0.4 > 0.05)
    d1[0, 0, 1] -= 4.0                                   # D2 outlier
    fl[0, 1, 1, 0] += 4.0                                # Fl outlier (epe 4 > 3, 4 / 1 > 0.05)
    t = R.scene_flow_counts(d0, d1, fl, gt)
    for m, outliers in ((0, 1), (1, 1), (2, 1), (3, 3)):
        assert _c(t, 0, 0, m, 0) == h * w and _c(t, 0, 0, m, 1) == outliers
    assert t[0, 8:].sum() == 0                           # fg and the noc set stay empty


def test_thresholds_at_three_pixels_and_five_percent():
    """Both conditions are strict: e = 3 exactly is not an outlier, nor is e / gt = 0.05 exactly (in fp32)."""
    gt = _gt(1, 4, disp=100.0, flow=(0.0, 0.0))
    gt["disp0"][0, 0] = [100.0, 100.0, 60.0, 60.0]
    d0, d1, fl = _pred(gt)
    d0[0, 0] = [103.0, 103.5, 63.0, 57.0]                # e = 3 (no), 3.5 but 3.5% (no), 3 at 5% (no), 3 at 5% (no)
    t = R.scene_flow_counts(d0, d1, fl, gt)
    assert _c(t, 0, 0, 0, 1) == 0
    d0[0, 0] = [103.0, 106.0, 63.01, 56.99]              # 6% and just over 5 %
    t = R.scene_flow_counts(d0, d1, fl, gt)
    assert _c(t, 0, 0, 0, 1) == 3
    at5 = _gt(1, 2, disp=80.0, flow=(0.0, 0.0))
    d0, d1, fl = _pred(at5)
    d0[0, 0] = [84.0, 84.5]                              # e = 4 > 3 at 4 / 80 = 0.05f exactly: no; 4.5 / 80: yes
    assert _c(R.scene_flow_counts(d0, d1, fl, at5), 0, 0, 0, 1) == 1
    gf = _gt(1, 2, flow=(60.0, 0.0))
    d0, d1, fl = _pred(gf)
    fl[0, 0, 0] = [63.0, 63.5]                           # flow epe 3 exactly at 5 %: no; 3.5 at 5.8 %: yes
    assert _c(R.scene_flow_counts(d0, d1, fl, gf), 0, 0, 2, 1) == 1


def test_invalid_ground_truth_in_one_map_only():
    h, w = 1, 4
    gt = _gt(h, w)
    gt["disp0"][0, 0, 0] = 0.0                           # no D1 gt here
    gt["disp1"][0, 0, 1] = 0.0                           # no D2 gt here
    gt["flow_valid"][0, 0, 2] = 0.25                     # no flow gt here
    d0, d1, fl = _pred(gt)
    d0[0, 0, :] += 5.0
    t = R.scene_flow_counts(d0, d1, fl, gt)
    assert [_c(t, 0, 0, m, 0) for m in range(4)] == [3, 3, 3, 1]
    assert _c(t, 0, 0, 0, 1) == 3 and _c(t, 0, 0, 3, 1) == 1     # SF only where all three are valid


def test_foreground_background_split_and_noc_set():
    h, w = 2, 2
    gt, noc = _gt(h, w), _gt(h, w)
    noc["flow_valid"][0, 0] = 0.0
    d0, d1, fl = _pred(gt)
    d0[0] += 5.0
    obj = np.array([[[0, 2], [0, 0]]], np.float32)
    t = R.scene_flow_counts(d0, d1, fl, gt, noc, obj)
    assert (_c(t, 0, 0, 0, 0), _c(t, 0, 1, 0, 0)) == (3, 1)
    assert (_c(t, 0, 0, 0, 1), _c(t, 0, 1, 0, 1)) == (3, 1)
    assert (_c(t, 1, 0, 2, 0), _c(t, 1, 1, 2, 0)) == (2, 0)      # noc flow valid on row 1 only, both background
    assert (_c(t, 1, 0, 3, 1), _c(t, 1, 1, 3, 1)) == (2, 0)


def test_results_dict_from_a_count_table():
    counts = np.zeros(ops.SF_COLS)
    counts[ops.sf_col(0, 0, 0, 0)], counts[ops.sf_col(0, 0, 0, 1)] = 200, 3
    counts[ops.sf_col(0, 1, 0, 0)], counts[ops.sf_col(0, 1, 0, 1)] = 50, 7
    res = scene_flow_results(counts, noc=False)
    assert len(res) == 4 * 3 and not any("noc" in k for k in res)
    assert res["kitti_sf_occ_d1_bg"] == 1.5 and res["kitti_sf_occ_d1_fg"] == 14.0 and res["kitti_sf_occ_d1_all"] == 4.0
    assert np.isnan(res["kitti_sf_occ_sf_all"]) and np.isnan(res["kitti_sf_occ_fl_fg"])
    res = scene_flow_results(counts, noc=True)
    assert len(res) == 2 * 4 * 3 and np.isnan(res["kitti_sf_noc_d2_bg"])
    assert list(ops.SF_SETS) == ["occ", "noc"] and ops.sf_col(1, 1, 3, 1) == 31 == R.sf_col(1, 1, 3, 1)


# ---- argument checks before any device call -----------------------------------------------------------------------------
def _frames(b=1, h=4, w=6):
    return torch.zeros((b, h, w, 3), dtype=torch.uint8)


def test_infer_scene_flow_refuses_mismatched_quadruples():
    f = _frames()
    with pytest.raises(ValueError, match="one shape"):
        infer_scene_flow(None, None, f, f, f, _frames(w=8))
    with pytest.raises(ValueError, match="uint8"):
        infer_scene_flow(None, None, f, f.float(), f, f)
    with pytest.raises(ValueError, match="not supported"):
        infer_scene_flow(None, None, f, f, f, f, flow_kwargs={"pred_bidir_flow": True})
    with pytest.raises(ValueError, match="stereo task only"):
        infer_scene_flow(None, None, f, f, f, f, stereo_kwargs={"task": "flow"})


def test_warp_disparity_refuses_bad_shapes():
    with pytest.raises(ValueError, match=r"\[B,H,W\]"):
        warp_disparity(torch.zeros(4, 5), torch.zeros(1, 2, 4, 5))
    with pytest.raises(ValueError, match="planar"):
        warp_disparity(torch.zeros(1, 4, 5), torch.zeros(1, 2, 5, 4))


def _sample(h=4, w=6, **drop):
    f = torch.zeros((h, w, 3), dtype=torch.uint8)
    s = {"left0": f, "right0": f, "left1": f, "right1": f, "disp0": torch.zeros(h, w), "disp1": torch.zeros(h, w),
         "flow": torch.zeros(2, h, w), "flow_valid": torch.ones(h, w)}
    for k in drop:
        s.pop(k)
    return s


def test_validate_scene_flow_checks_samples_before_the_device():
    with pytest.raises(ValueError, match="lacks"):
        validate_scene_flow(None, None, [_sample(disp1=True)])
    with pytest.raises(ValueError, match="batch"):
        validate_scene_flow(None, None, [_sample()], batch=0)
    bad = _sample()
    bad["right1"] = torch.zeros((4, 8, 3), dtype=torch.uint8)
    with pytest.raises(ValueError, match="one size"):
        validate_scene_flow(None, None, [bad])
    bad = _sample()
    bad["flow"] = torch.zeros(4, 6)
    with pytest.raises(ValueError, match="flow must be"):
        validate_scene_flow(None, None, [bad])
    partial = dict(_sample(), disp0_noc=torch.zeros(4, 6))
    with pytest.raises(ValueError, match="noc maps"):
        validate_scene_flow(None, None, [partial])
    with pytest.raises(ValueError, match="differs from the first"):
        validate_scene_flow(None, None, [_sample(), dict(_sample(), obj_map=torch.zeros(4, 6))], batch=4)


@pytest.mark.parametrize("noc,obj", [(False, False), (True, False), (False, True), (True, True)])
def test_sample_fields_keep_their_places(noc, obj):
    """views, gt, the four noc maps (or four Nones), obj_map (or None): the order the batches are run in, whichever of the
    optional maps the dataset has"""
    s = _sample()
    for i, k in enumerate(("disp0_noc", "disp1_noc", "flow_noc", "flow_noc_valid")):
        if noc:
            s[k] = torch.full((2, 4, 6) if k == "flow_noc" else (4, 6), float(10 + i))
    if obj:
        s["obj_map"] = torch.full((4, 6), 7.0)
    f = _scene_flow_fields(s, 0, noc, obj)
    assert len(f) == 13
    for i in range(4):
        assert f[i].dtype == torch.uint8 and f[i].shape == (4, 6, 3)
    assert f[6].shape == (2, 4, 6)
    for i in range(4):
        assert (f[8 + i] is None) == (not noc)
        if noc:
            assert (f[8 + i] == 10 + i).all()
    assert (f[12] is None) == (not obj)
    if obj:
        assert (f[12] == 7).all()


def test_runner_refuses_bad_options_before_the_device():
    with pytest.raises(ValueError, match="batch must be positive"):
        SceneFlowRunner(None, None, (4, 6), 0, "cuda")
    with pytest.raises(ValueError, match="not supported"):
        SceneFlowRunner(None, None, (4, 6), 2, "cuda", stereo_kwargs={"pred_bidir_disp": True})


def test_bad_c_abi_arguments_are_reported_without_a_gpu():
    one = ctypes.c_void_p(1024)
    lib = ops.LIB
    assert lib.um_warp_disparity(None, one, one, one, 1, 4, 4, None) == -22
    assert b"um_warp_disparity" in lib.um_last_error()
    assert lib.um_warp_disparity(one, one, one, one, 0, 4, 4, None) == -22
    assert lib.um_warp_disparity(one, one, ctypes.c_void_p(1026), one, 1, 4, 4, None) == -22        # misaligned
    assert lib.um_warp_disparity(one, one, one, ctypes.c_void_p(1030), 1, 4, 4, None) == -22        # overlap

    def ptrs(occ, noc):
        return (ctypes.c_void_p * 2)(occ, noc)
    full = [ptrs(4096, 8192) for _ in range(4)]
    ok = [one, one, one] + full + [None, 1, 4, 4, one, one, None]
    partial = [one, one, one] + full[:3] + [ptrs(4096, None)] + [None, 1, 4, 4, one, one, None]
    assert lib.um_scene_flow_stats(*partial) == -22
    assert b"noc set" in lib.um_last_error()
    no_occ = [one, one, one, ptrs(None, None)] + full[1:] + [None, 1, 4, 4, one, one, None]
    assert lib.um_scene_flow_stats(*no_occ) == -22
    zero_batch = list(ok)
    zero_batch[8] = 0
    assert lib.um_scene_flow_stats(*zero_batch) == -22
    assert b"um_scene_flow_stats" in lib.um_last_error()


# ---- submission names and the synthetic clip ---------------------------------------------------------------------------
def test_submission_names():
    assert scene_flow_name({"left0": None}, 7) == "000007_10"
    assert scene_flow_name({"name": "000123_10"}, 0) == "000123_10"
    assert scene_flow_name({"name": None}, 199) == "000199_10"


@pytest.mark.parametrize("seed", [3, 4, 5])
def test_synthetic_stereo_video_is_a_shifted_moving_crop(seed):
    """The right view is the left shifted right by one whole-pixel disparity d in [0, 32] for the whole clip:
    right[x + d] = left[x], as in `synthetic_pair` / `synthetic_stereo_frames`.  w = 48 > 32 keeps every overlap
    non-empty, so exactly one shift matches."""
    w = 48
    left, right = synthetic_stereo_video(5, 12, w, seed=seed)
    assert left.shape == right.shape == (5, 12, w, 3) and left.dtype == torch.uint8
    d = [s for s in range(33) if torch.equal(right[:, :, s:], left[:, :, :w - s])]
    assert len(d) == 1
    assert not torch.equal(left[0], left[1]) or not torch.equal(left[1], left[2])     # the crops move
    again = synthetic_stereo_video(5, 12, w, seed=seed)
    assert torch.equal(again[0], left) and torch.equal(again[1], right)
