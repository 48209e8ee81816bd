"""Mixed-size depth and the rest of the drop-in surface without a device: the step layout of `MixedSizeDepthRunner` (which
frame picks the bucket, the item tables, the staged poses), the driver's choice of runner, the mp4 writer round trip, the
`save_vis_depth` numbering of `validate_depth`, the C-ABI checks of `um_depth_to_image_ragged`, and the drivers'
remaining refusals."""
import ctypes
import os

import numpy as np
import pytest

from unimatch_b200 import MixedSizeDepthRunner, ops
from unimatch_b200 import inference_io as IO
from unimatch_b200.evaluation import _DepthVisNames
from unimatch_b200.inference import RAGGED_ITEM, _depth_step_layout, _relative_poses

ONE = ctypes.c_void_p(1024)          # any non-null address: validation never dereferences it


def test_step_layout_frames_outputs_and_fillers():
    sizes = [((5, 7), (6, 8)), ((4, 6), (4, 6))]
    frames, outputs, nbytes, used, results = _depth_step_layout(sizes, 3, False)
    assert frames.dtype == RAGGED_ITEM and len(frames) == 6 and len(outputs) == 3
    # frames t back to back (filler repeats the last), then frames t+1, each at its own size
    assert list(frames["offset"]) == [0, 105, 105, 177, 321, 321]
    assert list(frames["h"]) == [5, 4, 4, 6, 4, 4] and list(frames["w"]) == [7, 6, 6, 8, 6, 6]
    assert nbytes == 3 * (35 + 24 + 48 + 24) and not frames["flags"].any()
    # the depth comes back at frame t's size, scale 1 (depth is not rescaled), the filler is an empty item
    assert list(outputs["offset"][:2]) == [0, 35] and used == 59
    assert list(outputs["h"]) == [5, 4, 0] and list(outputs["w"]) == [7, 6, 0]
    assert (outputs["scale"][:2] == 1.0).all() and not outputs["flags"].any()
    assert results == [[("depth", 0, 5, 7)], [("depth", 35, 4, 6)]]


def test_step_layout_bidirectional():
    sizes = [((5, 7), (5, 7)), ((8, 8), (4, 4))]
    _, outputs, _, used, results = _depth_step_layout(sizes, 2, True)
    assert list(outputs["offset"]) == [0, 35, 99, 134] and used == 198
    assert list(outputs["h"]) == [5, 8, 5, 8]
    assert results[1] == [("depth", 35, 8, 8), ("depth_bwd", 134, 8, 8)]


def _bare_runner(**attrs):
    r = MixedSizeDepthRunner.__new__(MixedSizeDepthRunner)
    r.hmax, r.wmax, r.padding_factor, r.inference_size, r.batch, r.bidir, r.max_buckets = 64, 96, 16, None, 3, False, 4
    r.return_depth, r.visualize = True, True
    for k, v in attrs.items():
        setattr(r, k, v)
    return r


def test_bucket_is_frame_t_and_layout_views():
    r = _bare_runner()
    a, b = np.zeros((40, 90, 3), np.uint8), np.zeros((50, 60, 3), np.uint8)
    pair = r._pair((a, b, np.eye(4)))
    assert r._bucket(pair) == (48, 96)                                   # frame t's size rounded up to 16
    assert r._bucket(r._pair((b, a, np.eye(4)))) == (64, 64)
    assert r._sizes([pair]) == [((40, 90), (50, 60))]
    assert _bare_runner(inference_size=(32, 48))._bucket(pair) == (32, 48)
    table, used, views = r._layout(r._sizes([pair]), (48, 96))
    assert table.dtype == RAGGED_ITEM and len(table) == 3 * 3
    assert used == {"depth": 3600, "vis": 10800}
    assert views == [[("depth", "depth", 0, (40, 90)), ("vis", "vis", 0, (40, 90, 3))]]
    r.return_depth = False
    assert r._layout(r._sizes([pair]), (48, 96))[2] == [[("vis", "vis", 0, (40, 90, 3))]]
    steps = list(r._chunks(enumerate([(a, b, np.eye(4)), (b, a, np.eye(4)), (a, a, np.eye(4))])))
    assert [[i for i, _ in s] for s in steps] == [[0, 2], [1]]


def test_pair_errors():
    r = _bare_runner()
    ok = np.zeros((40, 90, 3), np.uint8)
    for item in ((np.zeros((65, 90, 3), np.uint8), ok, np.eye(4)),          # taller than the capacity
                 (ok, np.zeros((40, 97, 3), np.uint8), np.eye(4)),          # frame t+1 wider
                 (ok.astype(np.float32), ok, np.eye(4)),                    # not uint8
                 (ok, ok, np.eye(3)),                                       # not a [4, 4] pose
                 (ok, ok)):                                                 # no pose
        with pytest.raises(ValueError):
            r._pair(item)


def test_staged_poses_with_and_without_bidir():
    rng = np.random.default_rng(3)
    abs_poses = []
    for _ in range(3):
        p = np.eye(4, dtype=np.float32)
        p[:3, :3] = np.linalg.qr(rng.standard_normal((3, 3)))[0]
        p[:3, 3] = rng.standard_normal(3)
        abs_poses.append(p.astype(np.float32))
    want = _relative_poses(abs_poses, False)
    pairs = [(None, None, want[0]), (None, None, want[1])]
    got = _bare_runner()._poses(pairs)
    assert got.dtype == np.float32 and got.shape == (3, 4, 4)
    assert np.array_equal(got[:2], want) and np.array_equal(got[2], want[1])      # the filler repeats the last pair
    got = _bare_runner(bidir=True)._poses(pairs)
    assert got.shape == (6, 4, 4)
    assert np.array_equal(got[:2], _relative_poses(abs_poses, True)[:2])
    assert np.array_equal(got[3:5], _relative_poses(abs_poses, True)[2:])         # inverses as the sequence path forms them


# ------------------------------------------------------------------------------------------------------------ the driver
def _save(path, h, w, seed):
    from PIL import Image
    Image.fromarray(np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)).save(path)


def _scannet(root, sizes):
    for sub in ("color", "pose", "intrinsic"):
        os.makedirs(os.path.join(root, sub))
    for i, (h, w) in enumerate(sizes):
        _save(os.path.join(root, "color", "%d.png" % i), h, w, 50 + i)
        pose = np.eye(4)
        pose[0, 3] = 0.1 * i
        np.savetxt(os.path.join(root, "pose", "%d.txt" % i), pose, delimiter=" ")
    np.savetxt(os.path.join(root, "intrinsic", "intrinsic_color.txt"), np.diag([50.0, 50.0, 1.0, 1.0]))
    return root


class _Chosen(Exception):
    pass


class _Model:
    def eval(self):
        return self


@pytest.mark.parametrize("sizes,mixed", [([(48, 64)] * 3, False), ([(50, 64), (50, 64), (48, 64)], True)])
def test_inference_depth_chooses_the_runner(tmp_path, monkeypatch, sizes, mixed):
    seen = {}

    def fake(name):
        def make(model, size, batch, device, K, **kw):
            seen.update(name=name, size=tuple(size), kw=kw)
            raise _Chosen()
        return make

    monkeypatch.setattr(IO, "DepthSequenceRunner", fake("sequence"))
    monkeypatch.setattr(IO, "MixedSizeDepthRunner", fake("mixed"))
    root = _scannet(str(tmp_path / "scene"), sizes)
    with pytest.raises(_Chosen):
        IO.inference_depth(_Model(), inference_dir=root, output_path=str(tmp_path / "out"), max_buckets=3)
    if mixed:
        assert seen["name"] == "mixed" and seen["size"] == (50, 64) and seen["kw"]["max_buckets"] == 3
    else:
        assert seen["name"] == "sequence" and seen["size"] == (48, 64) and "max_buckets" not in seen["kw"]
    assert seen["kw"]["visualize"] and not seen["kw"]["return_depth"]


def test_save_video_and_mixed_depth_refusals(tmp_path):
    """refused before any device work: save_video without a video, or on a video cv2 cannot open; a depth pair of two
    sizes whose first frame needs no resize (the reference would give its model frames of two sizes), unless
    `inference_size` resizes it"""
    from test_inference_io_cpu import NoDevice
    out = str(tmp_path / "out")
    with pytest.raises(ValueError, match="save_video needs inference_video"):
        IO.inference_flow(NoDevice(), inference_dir=str(tmp_path), output_path=out, save_video=True)
    with pytest.raises(ValueError, match="cannot open the video"):
        IO.inference_flow(NoDevice(), inference_video=str(tmp_path / "v.mp4"), output_path=out, save_video=True)
    root = _scannet(str(tmp_path / "scene"), [(50, 64), (48, 64), (50, 64)])     # pair 1: 48x64 needs no resize at 16
    with pytest.raises(ValueError, match="1.png and .*2.png differ in size and the first needs no resize"):
        IO.inference_depth(NoDevice(), inference_dir=root, output_path=out)
    with pytest.raises(AssertionError, match="device work started"):          # resized to 32x64: accepted
        IO.inference_depth(NoDevice(), inference_dir=root, output_path=out, inference_size=(32, 64))


# ------------------------------------------------------------------------------------------------------------ the video
def test_video_names_and_frames():
    assert IO.video_name("/data/demo/kitti.mp4", False) == "kitti_flow.mp4"
    assert IO.video_name("kitti.avi", True) == "kitti_flow_img.mp4"
    rgb = np.arange(5 * 3 * 3, dtype=np.uint8).reshape(5, 3, 3)
    f = IO.video_frame(rgb)
    assert f.shape == (6, 4, 3) and f.flags["C_CONTIGUOUS"]
    assert np.array_equal(f[:5, :3], rgb[..., ::-1])                        # BGR
    assert np.array_equal(f[5, :3], rgb[4, :, ::-1]) and np.array_equal(f[:5, 3], rgb[:, 2, ::-1])
    even = np.zeros((4, 6, 3), np.uint8)
    assert IO.video_frame(even).shape == (4, 6, 3)


def test_video_writer_round_trip(tmp_path):
    cv2 = pytest.importorskip("cv2")
    h, w, n, fps = 75, 96, 6, 12.0
    yy, xx = np.mgrid[0:h, 0:w]
    frames = [np.stack([(xx * 2 + 10 * t) % 256, (yy * 3) % 256, np.full_like(xx, 40 * t % 256)], -1).astype(np.uint8)
              for t in range(n)]
    path = str(tmp_path / "clip_flow.mp4")
    vw = IO._VideoWriter(path, fps, ahead=2)
    for f in frames:
        vw.submit(f)
    vw.close()
    assert vw.frames == n
    cap = cv2.VideoCapture(path)
    assert cap.isOpened()
    assert cap.get(cv2.CAP_PROP_FPS) == pytest.approx(fps)
    got = []
    while True:
        ok, img = cap.read()
        if not ok:
            break
        got.append(cv2.cvtColor(img, cv2.COLOR_BGR2RGB))
    cap.release()
    assert len(got) == n
    assert got[0].shape == (h + 1, w, 3)                                    # the odd height padded by a repeated row
    mae = max(np.abs(g[:h].astype(np.float64) - f).mean() for g, f in zip(got, frames))
    assert mae < 6.0, mae


# ---------------------------------------------------------------------------------------------------- validate_depth
def test_validate_depth_vis_names():
    counts = [5, 0, 3, 7, 0, 0, 2]
    names = _DepthVisNames("scannet")
    # batches arrive grouped by size, out of dataset order; a name is given once every earlier count is known
    assert names.add([2, 3], [counts[2], counts[3]]) == []
    assert names.add([0, 5], [counts[0], counts[5]]) == [(0, "0001_depth_pred.png")]
    assert names.add([1, 4], [counts[1], counts[4]]) == [(2, "0002_depth_pred.png"), (3, "0003_depth_pred.png")]
    assert names.add([6], [counts[6]]) == [(6, "0004_depth_pred.png")]
    demon = _DepthVisNames("demon")
    assert demon.add(list(range(7)), counts) == [(0, "0001.png"), (2, "0002.png"), (3, "0003.png"), (6, "0004.png")]


def test_validate_depth_save_vis_needs_save_dir():
    from unimatch_b200.evaluation import validate_depth
    with pytest.raises(ValueError, match="save_dir"):
        validate_depth(None, [], protocol="scannet", save_vis_depth=True)


# ---------------------------------------------------------------------------------------------------------------- C ABI
def test_depth_to_image_ragged_validates_without_a_gpu():
    good = dict(n=2, h_max=8, w_max=8, numel=1024)
    for change in (dict(n=0), dict(n=65536), dict(h_max=0), dict(w_max=-1), dict(numel=0)):
        a = dict(good, **change)
        rc = ops.LIB.um_depth_to_image_ragged(ONE, a["numel"], ONE, ONE, ONE, a["n"], a["h_max"], a["w_max"], None)
        assert rc == -22, change
        assert b"um_depth_to_image_ragged" in ops.LIB.um_last_error()
    assert ops.LIB.um_depth_to_image_ragged(ONE, 64, ONE, ONE, None, 1, 4, 4, None) == -22             # no scratch
    assert ops.LIB.um_depth_to_image_ragged(ONE, 64, None, ONE, ONE, 1, 4, 4, None) == -22             # no items
    assert ops.LIB.um_depth_to_image_ragged(ONE, 64, ONE, ONE, ONE, 1, 1 << 16, 1 << 16, None) == -22  # > 2^31 - 1 px
