"""The drop-in inference commands without a GPU: file listing and naming against the reference's own `inference_flow` /
`inference_stereo` run on the CPU (in a subprocess, with its random-init model at a tiny size and its import-only
dependencies stubbed), the argument checks that must refuse before any device work, and the writer jobs read back."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from PIL import Image

from unimatch_b200 import inference_io as IO

REFERENCE = os.environ.get("UNIMATCH_REFERENCE", "/root/reference")
needs_reference = pytest.mark.skipif(not os.path.isdir(os.path.join(REFERENCE, "unimatch")),
                                     reason="the reference tree is not available (set UNIMATCH_REFERENCE)")

# runs the reference's inference function on the CPU with its own model; argv: reference root, task, JSON kwargs
_RUN_REFERENCE = r"""
import json, sys, types
sys.dont_write_bytecode = True
ref, task, kwargs = sys.argv[1], sys.argv[2], json.loads(sys.argv[3])
sys.path.insert(0, ref)
for name in ("imageio", "skimage", "skimage.io", "matplotlib", "matplotlib.cm", "matplotlib.colors"):
    mod = types.ModuleType(name)
    mod.get_cmap = lambda *a, **k: None
    sys.modules.setdefault(name, mod)
sys.modules["skimage"].io = sys.modules["skimage.io"]
sys.modules["matplotlib"].cm = sys.modules["matplotlib.cm"]
import torch
torch.manual_seed(0)
from unimatch.unimatch import UniMatch
model = UniMatch(num_scales=1, feature_channels=128, upsample_factor=8, num_head=1, ffn_dim_expansion=4,
                 num_transformer_layers=6, reg_refine=False, task=task)
if task == "flow":
    import evaluate_flow
    evaluate_flow.inference_flow(model, **kwargs)
else:
    import evaluate_stereo
    evaluate_stereo.inference_stereo(model, **kwargs)
"""
FLOW_MODEL = dict(attn_type="swin", attn_splits_list=[2], corr_radius_list=[-1], prop_radius_list=[-1])
STEREO_MODEL = dict(attn_type="self_swin2d_cross_swin1d", attn_splits_list=[2], corr_radius_list=[-1], prop_radius_list=[-1])


def _run_reference(task, **kwargs):
    r = subprocess.run([sys.executable, "-c", _RUN_REFERENCE, REFERENCE, task, json.dumps(kwargs)], capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]


def _save(path, h, w, seed, grey=False):
    a = np.random.default_rng(seed).integers(0, 256, (h, w) if grey else (h, w, 3), dtype=np.uint8)
    Image.fromarray(a).save(path, quality=95) if path.endswith(".jpg") else Image.fromarray(a).save(path)


# a flow directory: .png and .jpg mixed, an odd count, sizes that change between frames (every such pair's first frame is
# resized, as the reference needs) and a portrait pair; no grey image, which the reference takes only in a pair of two
# (it tiles both frames when the first is grey, evaluate_flow.py:700-705)
FLOW_DIR = [("f_000.png", 62, 94, False), ("f_001.jpg", 62, 94, False), ("f_002.png", 58, 90, False),
            ("f_003.png", 58, 90, False), ("f_004.jpg", 94, 62, False), ("f_005.png", 94, 62, False), ("f_006.png", 62, 94, False)]


def _flow_dir(root):
    d = os.path.join(root, "frames")
    os.makedirs(d)
    for k, (name, h, w, grey) in enumerate(FLOW_DIR):
        _save(os.path.join(d, name), h, w, k, grey)
    return d


def _names(flags, files, video=False):
    keys = IO.flow_keys(**flags)
    return {n for t in range(len(files) - 1) for n in IO.output_names(IO.FLOW_FILES, keys, IO.flow_prefix(files, t, video)).values()}


def test_flow_listing_and_pairs(tmp_path):
    d = _flow_dir(str(tmp_path))
    files = IO.flow_inputs(d)
    assert [os.path.basename(f) for f in files] == [n for n, *_ in FLOW_DIR]
    assert IO.flow_prefix(files, 1, False) == "f_001" and IO.flow_prefix(files, 1, True) == "0001"


@needs_reference
@pytest.mark.parametrize("flags", [dict(), dict(pred_bidir_flow=True, fwd_bwd_consistency_check=True, save_flo_flow=True),
                                   dict(save_flo_flow=True)])
def test_flow_names_equal_reference(tmp_path, flags):
    d = _flow_dir(str(tmp_path))
    out = str(tmp_path / "out")
    _run_reference("flow", inference_dir=d, output_path=out, padding_factor=16, **FLOW_MODEL, **flags)
    assert set(os.listdir(out)) == _names(flags, IO.flow_inputs(d))


def _stereo_dirs(root, n_left=3, n_right=3):
    one, left, right = (os.path.join(root, k) for k in ("one", "left", "right"))
    for d in (one, left, right):
        os.makedirs(d)
    sizes = [(62, 94), (58, 90), (62, 94)]
    for i in range(3):
        h, w = sizes[i]
        ext = ".jpg" if i == 1 else ".png"
        _save(os.path.join(one, "s_%02d_a%s" % (i, ext)), h, w, 10 + i)
        _save(os.path.join(one, "s_%02d_b%s" % (i, ext)), h, w, 20 + i)
    for i in range(n_left):
        _save(os.path.join(left, "im%d%s" % (i, ".jpg" if i == 1 else ".png")), *sizes[i % 3], 30 + i)
    for i in range(n_right):
        _save(os.path.join(right, "im%d.png" % i), *sizes[i % 3], 40 + i)
    return one, left, right


def test_stereo_listing(tmp_path):
    one, left, right = _stereo_dirs(str(tmp_path))
    l1, r1 = IO.stereo_inputs(inference_dir=one)
    assert [os.path.basename(f) for f in l1] == ["s_00_a.png", "s_01_a.jpg", "s_02_a.png"]
    assert [os.path.basename(f) for f in r1] == ["s_00_b.png", "s_01_b.jpg", "s_02_b.png"]
    l2, r2 = IO.stereo_inputs(inference_dir_left=left, inference_dir_right=right)
    assert [os.path.basename(f) for f in l2] == ["im0.png", "im1.jpg", "im2.png"]
    assert [os.path.basename(f) for f in r2] == ["im0.png", "im1.png", "im2.png"]


@needs_reference
@pytest.mark.parametrize("layout", ["one", "left_right"])
@pytest.mark.parametrize("flags", [dict(), dict(pred_bidir_disp=True, save_pfm_disp=True), dict(pred_right_disp=True)])
def test_stereo_names_equal_reference(tmp_path, layout, flags):
    one, left, right = _stereo_dirs(str(tmp_path))
    dirs = dict(inference_dir=one) if layout == "one" else dict(inference_dir_left=left, inference_dir_right=right)
    out = str(tmp_path / "out")
    _run_reference("stereo", output_path=out, padding_factor=16, **dirs, **STEREO_MODEL, **flags)
    lefts, _ = IO.stereo_inputs(**dirs)
    keys = IO.stereo_keys(flags.get("pred_bidir_disp", False), flags.get("save_pfm_disp", False))
    want = {n for f in lefts for n in IO.output_names(IO.STEREO_FILES, keys, os.path.basename(f)[:-4]).values()}
    assert set(os.listdir(out)) == want


def _scannet(root, sizes=((48, 64),) * 5):
    for sub in ("color", "pose", "intrinsic"):
        os.makedirs(os.path.join(root, sub))
    for i, (h, w) in enumerate(sizes):
        _save(os.path.join(root, "color", "%d%s" % (i, ".png" if i % 2 else ".jpg")), h, w, 50 + i)
        pose = np.eye(4)
        pose[0, 3] = 0.1 * i
        np.savetxt(os.path.join(root, "pose", "%d.txt" % i), pose, delimiter=" ")
    np.savetxt(os.path.join(root, "intrinsic", "intrinsic_color.txt"), np.diag([50.0, 50.0, 1.0, 1.0]))
    return root


def test_depth_listing_and_names(tmp_path):
    root = _scannet(str(tmp_path / "scene"))
    imgs, poses, intr = IO.depth_inputs(root)
    assert [os.path.basename(f) for f in imgs] == ["0.jpg", "1.png", "2.jpg", "3.png", "4.jpg"]
    assert [os.path.basename(f) for f in poses] == ["%d.txt" % i for i in range(5)]
    assert os.path.basename(intr) == "intrinsic_color.txt"
    names = [IO.output_names(IO.DEPTH_FILES, IO.depth_keys(True), os.path.basename(f)[:-4]) for f in imgs[:-1]]
    assert names[1] == {"vis": "1.png", "vis_bwd": "1_bwd.png"}


# ------------------------------------------------------------------------------------------------------- argument checks
class NoDevice:
    """a model that must not be touched"""

    def __getattr__(self, name):
        raise AssertionError("device work started before the arguments were checked")


def test_refusals_come_before_device_work(tmp_path):
    d = _flow_dir(str(tmp_path))
    out = str(tmp_path / "out")
    with pytest.raises(ValueError, match="imageio"):
        IO.inference_flow(NoDevice(), inference_video=str(tmp_path / "v.mp4"), output_path=out, save_video=True)
    with pytest.raises(ValueError, match="pred_bidir_flow"):
        IO.inference_flow(NoDevice(), inference_dir=d, output_path=out, fwd_bwd_consistency_check=True)
    with pytest.raises(ValueError, match="one of"):
        IO.inference_flow(NoDevice(), output_path=out)
    # a size change after a frame that needs no resize: the reference's model would get frames of two sizes
    bad = str(tmp_path / "bad")
    os.makedirs(bad)
    _save(os.path.join(bad, "a.png"), 64, 96, 1)
    _save(os.path.join(bad, "b.png"), 60, 90, 2)
    with pytest.raises(ValueError, match="differ in size"):
        IO.inference_flow(NoDevice(), inference_dir=bad, output_path=out, padding_factor=16)
    one, left, right = _stereo_dirs(str(tmp_path / "st"), n_left=3, n_right=2)
    with pytest.raises(ValueError, match="choose one"):
        IO.inference_stereo(NoDevice(), inference_dir=one, output_path=out, pred_bidir_disp=True, pred_right_disp=True)
    with pytest.raises(ValueError, match="3 left images but 2 right"):
        IO.inference_stereo(NoDevice(), inference_dir_left=left, inference_dir_right=right, output_path=out)
    _save(os.path.join(one, "z_odd.png"), 62, 94, 3)
    with pytest.raises(ValueError, match="4 left images but 3 right"):
        IO.inference_stereo(NoDevice(), inference_dir=one, output_path=out)
    with pytest.raises(ValueError, match="inference_dir"):
        IO.inference_stereo(NoDevice(), output_path=out)
    root = _scannet(str(tmp_path / "scene"), sizes=[(48, 64), (48, 64), (50, 64)])
    with pytest.raises(ValueError, match="differ in size"):
        IO.inference_depth(NoDevice(), inference_dir=root, output_path=out)
    os.remove(os.path.join(root, "pose", "2.txt"))
    with pytest.raises(ValueError, match="3 frames but 2 poses"):
        IO.inference_depth(NoDevice(), inference_dir=root, output_path=out)


# ----------------------------------------------------------------------------------------------------------- writer jobs
def test_writer_jobs_round_trip(tmp_path):
    g = torch.Generator().manual_seed(4)
    flow = torch.randn((2, 5, 7), generator=g) * 9
    disp = torch.rand((6, 4), generator=g) * 30
    rgb = torch.randint(0, 256, (5, 7, 3), generator=g, dtype=torch.uint8)
    occ = (torch.rand((5, 7), generator=g) > 0.5).float()
    results = [(0, {"flow": flow, "disp": disp, "vis": rgb, "bgr": rgb, "occ": occ})]
    p = {k: str(tmp_path / ("x_" + k + ext)) for k, ext in (("flow", ".flo"), ("disp", ".pfm"), ("vis", ".png"),
                                                           ("bgr", ".png"), ("occ", ".png"))}
    enc = {"flow": "flo", "disp": "pfm", "vis": "rgb", "bgr": "bgr", "occ": "mask"}
    IO._write_results(results, lambda i: {k: (p[k], enc[k]) for k in p}, writers=2, group=1)
    data = open(p["flow"], "rb").read()
    assert data[:4] == b"PIEH" and np.frombuffer(data[4:12], "<i4").tolist() == [7, 5]
    assert np.array_equal(np.frombuffer(data[12:], "<f4").reshape(5, 7, 2), flow.permute(1, 2, 0).numpy())
    data = open(p["disp"], "rb").read()
    head = b"Pf\n4 6\n-1.000000\n"
    assert data.startswith(head) and np.array_equal(np.frombuffer(data[len(head):], "<f4").reshape(6, 4), disp.numpy()[::-1])
    assert np.array_equal(np.array(Image.open(p["vis"])), rgb.numpy())
    assert np.array_equal(np.array(Image.open(p["bgr"])), rgb.numpy()[..., ::-1])
    grey = Image.open(p["occ"])
    assert grey.mode == "L" and np.array_equal(np.array(grey), (occ.numpy() * 255.).astype(np.uint8))


def test_writer_error_reaches_the_caller(tmp_path):
    blocker = tmp_path / "file"
    blocker.write_bytes(b"")
    results = [(0, {"vis": torch.zeros((2, 2, 3), dtype=torch.uint8)})]
    with pytest.raises(OSError):
        IO._write_results(results, lambda i: {"vis": (str(blocker / "sub" / "a.png"), "rgb")}, writers=1, group=1)
