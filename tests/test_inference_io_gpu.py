"""The drop-in inference commands on the device, from synthetic PNG directories (and a video, or its frame stream) to files:
every file decodes to exactly what the runner produced for that pair, every picture is the oracle's colouring of the
written data, the predictions agree with the per-pair drivers, and the file set is exactly the one the naming functions
give.  Nothing here reads the reference tree."""
import os

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import depth_viz as ODE
from oracle import disp_viz as ODI
from oracle import flow_viz as OF
from unimatch_b200 import (DepthSequenceRunner, MixedSizeFlowRunner, MixedSizeStereoRunner, infer_depth_sequence, infer_flow,
                           infer_flow_video)
from unimatch_b200 import inference_io as IO
from unimatch_b200.inference import _stereo_from_frames, flow_to_image
from unimatch_b200.submission import flo_header, pfm_header
from unimatch_b200.synthetic import synthetic_model, synthetic_posed_sequence, synthetic_video, workload_call

pytestmark = pytest.mark.gpu


def _png(path):
    return np.array(Image.open(path))


def _vis_close(got, ref, what):
    """the device colouring against the numpy statement: every byte within 1, at most 0.1 % different (float64 atan2 on
    the device against numpy's, as in test_video_gpu.py)"""
    d = got.astype(np.int16) - ref.astype(np.int16)
    assert np.abs(d).max() <= 1 and (d != 0).mean() <= 1e-3, what


def _read_flo(path):
    data = open(path, "rb").read()
    w, h = np.frombuffer(data[4:12], "<i4")
    return data, np.frombuffer(data[12:], "<f4").reshape(h, w, 2)


def _read_pfm(path):
    data = open(path, "rb").read()
    head = data.split(b"\n", 3)
    w, h = (int(v) for v in head[1].split())
    return data, np.frombuffer(head[3], "<f4").reshape(h, w)[::-1]


def _check_file_set(out, want):
    assert set(os.listdir(out)) == set(want), sorted(set(os.listdir(out)) ^ set(want))


# --------------------------------------------------------------------------------------------------------------------- flow
# KITTI-like sizes, scaled down: sizes change between pairs (those pairs run alone), a portrait pair and a grey pair
FLOW_FRAMES = [((94, 311), 0), ((94, 311), 0), ((93, 307), 1), ((93, 307), 1), ((311, 94), 2), ((311, 94), 2),
               ((94, 311), "grey"), ((94, 311), "grey")]


def _flow_dir(root):
    d = os.path.join(root, "frames")
    os.makedirs(d)
    for k, ((h, w), clip) in enumerate(FLOW_FRAMES):
        grey = clip == "grey"
        f = synthetic_video(2, h, w, seed=60 + (3 if grey else clip))[k % 2].numpy()
        img = Image.fromarray(f[..., 0] if grey else f)
        img.save(os.path.join(d, "k%03d.png" % k))
    return d


FLOW_FLAGS = {"plain": dict(), "bidir_check_flo": dict(pred_bidir_flow=True, fwd_bwd_consistency_check=True, save_flo_flow=True),
              "bwd_flo": dict(pred_bwd_flow=True, save_flo_flow=True), "size_flo": dict(inference_size=(96, 320), save_flo_flow=True)}


@pytest.mark.parametrize("case", sorted(FLOW_FLAGS))
def test_inference_flow_directory(tmp_path, case):
    flags = FLOW_FLAGS[case]
    m = synthetic_model("gmflow-scale1")
    call = workload_call("gmflow-scale1", drop=("task", "min_depth", "max_depth", "num_depth_candidates"))
    d = _flow_dir(str(tmp_path))
    out = str(tmp_path / "out")
    stats = IO.inference_flow(m, inference_dir=d, output_path=out, padding_factor=16, batch=2, **flags, **call)
    files = IO.flow_inputs(d)
    keys = IO.flow_keys(flags.get("pred_bidir_flow", False), flags.get("fwd_bwd_consistency_check", False),
                        flags.get("save_flo_flow", False))
    names = [IO.output_names(IO.FLOW_FILES, keys, IO.flow_prefix(files, t, False)) for t in range(len(files) - 1)]
    _check_file_set(out, [n for ns in names for n in ns.values()])
    assert stats["pairs"] == len(files) - 1

    # the runner alone on the pairs of one size, as the driver streams them
    frames = [IO._flow_frame(f) for f in files]
    assert frames[6].shape == (94, 311, 3) and (frames[6][..., 0] == frames[6][..., 2]).all()       # grey, tiled
    streamed = [t for t in range(len(files) - 1) if frames[t].shape == frames[t + 1].shape]
    assert streamed == [0, 2, 4, 6]
    runner_kw = {k: v for k, v in flags.items() if k != "save_flo_flow"}
    runner = MixedSizeFlowRunner(m, (311, 311), 2, "cuda", padding_factor=16, visualize=True, **runner_kw, **call)
    ref = {streamed[i]: {k: v.clone() for k, v in r.items()}
           for i, r in runner.run((frames[t], frames[t + 1]) for t in streamed)}

    worst = 0.0
    for t in range(len(files) - 1):
        p = {k: os.path.join(out, n) for k, n in names[t].items()}
        h, w = frames[t].shape[:2]
        for key in ("vis", "vis_bwd"):
            if key in p:
                pic = _png(p[key])
                assert pic.shape == (h, w, 3), (t, key)
                if t in ref:
                    assert np.array_equal(pic, ref[t][key].numpy()), (t, key)                # lossless
        for key in ("fwd_occ", "bwd_occ"):
            if key in p:
                mask = _png(p[key])
                assert Image.open(p[key]).mode == "L" and set(np.unique(mask)) <= {0, 255}
                if t in ref:
                    assert np.array_equal(mask, (ref[t][key].numpy() * 255.).astype(np.uint8)), (t, key)
        for key, vis in (("flow", "vis"), ("flow_bwd", "vis_bwd")):
            if key not in p:
                continue
            data, flo = _read_flo(p[key])
            assert flo.shape == (h, w, 2), (t, key)
            if t in ref:
                want = ref[t][key].permute(1, 2, 0).contiguous().numpy()
                assert data == flo_header(h, w) + want.tobytes(), (t, key)                  # lossless
            if vis in p:
                pic = _png(p[vis])
                assert np.array_equal(pic, flow_to_image(torch.from_numpy(flo.copy()).permute(2, 0, 1)[None].cuda())[0].cpu().numpy())
                _vis_close(pic, OF.flow_to_image(flo), (t, vis))                        # the picture of the written flow
            # the prediction against `infer_flow` on the pair alone (a pair whose frames differ in size has no such
            # counterpart: `infer_flow` takes one size)
            if t in ref and key == "flow" and not flags.get("pred_bwd_flow"):
                a, b = (torch.from_numpy(frames[i]).permute(2, 0, 1)[None].float().cuda() for i in (t, t + 1))
                alone = infer_flow(m, a, b, padding_factor=16, inference_size=flags.get("inference_size"),
                                   pred_bidir_flow=flags.get("pred_bidir_flow", False), **call)
                r = alone["flow"][0].permute(1, 2, 0).cpu().numpy()
                worst = max(worst, float(np.abs(flo - r).max() / np.abs(r).max()))
    print("%s: largest difference to infer_flow on the pair alone, relative to its largest flow: %.2e" % (case, worst))
    assert worst <= 1e-5


def _video_frames(tmp_path, frames):
    """a short MJPG video and the frames cv2 decodes from it, or None when cv2 here cannot read back what it writes"""
    import cv2
    path = str(tmp_path / "clip.avi")
    writer = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"MJPG"), 10, (frames.shape[2], frames.shape[1]))
    if not writer.isOpened():
        return None, None
    for f in frames:
        writer.write(cv2.cvtColor(f, cv2.COLOR_RGB2BGR))
    writer.release()
    cap = cv2.VideoCapture(path)
    decoded = []
    while cap.isOpened():
        ok, img = cap.read()
        if not ok:
            break
        decoded.append(cv2.cvtColor(img, cv2.COLOR_BGR2RGB))
    cap.release()
    return (path, np.stack(decoded)) if len(decoded) == len(frames) else (None, None)


def test_inference_flow_video_bwd(tmp_path):
    """`pred_bwd_flow` on a video: each pair in swapped order, as `infer_flow_video(..., pred_bwd_flow=True)`"""
    m = synthetic_model("gmflow-scale1")
    call = workload_call("gmflow-scale1", drop=("task", "min_depth", "max_depth", "num_depth_candidates"))
    frames = synthetic_video(8, 96, 160, seed=23).numpy()
    path, decoded = _video_frames(tmp_path, frames)
    out = str(tmp_path / "out")
    flags = dict(pred_bidir_flow=True, fwd_bwd_consistency_check=True, pred_bwd_flow=True, save_flo_flow=True)
    if path is not None:
        print("video: written and decoded by cv2, driven through inference_flow(inference_video=...)")
        IO.inference_flow(m, inference_video=path, output_path=out, padding_factor=16, batch=3, **flags, **call)
    else:
        print("video: cv2 cannot read back a video here; the in-memory frame stream goes through the same path from the "
              "reader onward")
        decoded = frames
        os.makedirs(out)
        kw = dict(padding_factor=16, inference_size=None, pred_bidir_flow=True, fwd_bwd_consistency_check=True, **call)
        rd = IO._Readers(1, 8)
        IO._video_flow(m, rd.map(lambda f: f, iter(decoded)), out, IO.flow_keys(True, True, True), True, True, 3, "cuda", 2,
                       kw, rd)
    n = len(decoded) - 1
    names = [IO.output_names(IO.FLOW_FILES, IO.flow_keys(True, True, True), IO.flow_prefix(None, t, True)) for t in range(n)]
    _check_file_set(out, [v for ns in names for v in ns.values()])
    ref = infer_flow_video(m, torch.from_numpy(decoded).cuda(), padding_factor=16, pred_bidir_flow=True, pred_bwd_flow=True,
                           fwd_bwd_consistency_check=True, **call)
    for t in range(n):
        for key, vis in (("flow", "vis"), ("flow_bwd", "vis_bwd")):
            _, flo = _read_flo(os.path.join(out, names[t][key]))
            r = ref[key][t].permute(1, 2, 0).cpu().numpy()
            assert np.abs(flo - r).max() <= 1e-4 * max(1.0, np.abs(r).max()), (t, key)
            pic = _png(os.path.join(out, names[t][vis]))
            assert np.array_equal(pic, flow_to_image(torch.from_numpy(flo.copy()).permute(2, 0, 1)[None].cuda())[0].cpu().numpy())
        for key in ("fwd_occ", "bwd_occ"):
            mask = _png(os.path.join(out, names[t][key]))
            assert ((mask == 255) != (ref[key][t].cpu().numpy() == 1)).mean() < 0.01, (t, key)


# ------------------------------------------------------------------------------------------------------------------- stereo
STEREO_SIZES = [(94, 311), (93, 307), (94, 311), (96, 320), (91, 300)]
STEREO_FLAGS = {"plain": dict(), "bidir_pfm": dict(pred_bidir_disp=True, save_pfm_disp=True),
                "right_pfm": dict(pred_right_disp=True, save_pfm_disp=True),
                "size_pfm": dict(inference_size=(96, 320), save_pfm_disp=True)}


@pytest.mark.parametrize("case", sorted(STEREO_FLAGS))
def test_inference_stereo_directories(tmp_path, case):
    flags = STEREO_FLAGS[case]
    m = synthetic_model("gmstereo-scale2")
    call = workload_call("gmstereo-scale2", drop=("task", "min_depth", "max_depth", "num_depth_candidates"))
    left_dir, right_dir = str(tmp_path / "left"), str(tmp_path / "right")
    os.makedirs(left_dir), os.makedirs(right_dir)
    for i, (h, w) in enumerate(STEREO_SIZES):
        pair = synthetic_video(2, h, w, seed=80 + i).numpy()
        Image.fromarray(pair[0]).save(os.path.join(left_dir, "%06d_10.png" % i))
        Image.fromarray(pair[1]).save(os.path.join(right_dir, "%06d_10.png" % i))
    out = str(tmp_path / "out")
    IO.inference_stereo(m, inference_dir_left=left_dir, inference_dir_right=right_dir, output_path=out, padding_factor=32,
                        batch=2, **flags, **call)
    lefts, rights = IO.stereo_inputs(inference_dir_left=left_dir, inference_dir_right=right_dir)
    keys = IO.stereo_keys(flags.get("pred_bidir_disp", False), flags.get("save_pfm_disp", False))
    names = [IO.output_names(IO.STEREO_FILES, keys, os.path.basename(f)[:-4]) for f in lefts]
    _check_file_set(out, [n for ns in names for n in ns.values()])

    pairs = [(IO._rgb_frame(a), IO._rgb_frame(b)) for a, b in zip(lefts, rights)]
    runner_kw = {k: v for k, v in flags.items() if k != "save_pfm_disp"}
    runner = MixedSizeStereoRunner(m, (96, 320), 2, "cuda", padding_factor=32, visualize=True, **runner_kw, **call)
    ref = {i: {k: v.clone() for k, v in r.items()} for i, r in runner.run(pairs)}
    worst = 0.0
    for i, (h, w) in enumerate(STEREO_SIZES):
        p = {k: os.path.join(out, n) for k, n in names[i].items()}
        for disp_key, vis_key in (("disp", "vis"), ("disp_right", "vis_right")):
            if vis_key not in p:
                continue
            pic = _png(p[vis_key])
            assert np.array_equal(pic, ref[i][vis_key].numpy()[..., ::-1]), (i, vis_key)     # cv2.imwrite's RGB, lossless
            if disp_key not in p:
                continue
            data, disp = _read_pfm(p[disp_key])
            assert data == pfm_header(h, w) + np.ascontiguousarray(ref[i][disp_key].numpy()[::-1]).tobytes(), (i, disp_key)
            assert np.array_equal(pic, ODI.vis_disparity(disp)[..., ::-1]), (i, vis_key)    # the picture of the written data
            frames = torch.from_numpy(np.stack(pairs[i])).cuda()
            alone = _stereo_from_frames(m, frames, padding_factor=32, inference_size=flags.get("inference_size"),
                                        pred_bidir_disp=flags.get("pred_bidir_disp", False),
                                        pred_right_disp=flags.get("pred_right_disp", False), **call)[disp_key][0].cpu().numpy()
            worst = max(worst, float(np.abs(disp - alone).max() / np.abs(alone).max()))
    print("%s: largest difference to the pair alone, relative to its largest disparity: %.2e" % (case, worst))
    assert worst <= 1e-4


# -------------------------------------------------------------------------------------------------------------------- depth
@pytest.mark.parametrize("bidir", [False, True])
def test_inference_depth_scannet(tmp_path, bidir):
    m = synthetic_model("gmdepth-scale1-regrefine1")
    call = workload_call("gmdepth-scale1-regrefine1", drop=("task", "min_depth", "max_depth", "num_depth_candidates"))
    frames, K, poses = synthetic_posed_sequence(7, 90, 150, seed=31)
    root = str(tmp_path / "scene")
    for sub in ("color", "pose", "intrinsic"):
        os.makedirs(os.path.join(root, sub))
    for i, (f, p) in enumerate(zip(frames.numpy(), poses.numpy())):
        Image.fromarray(f).save(os.path.join(root, "color", "%d.png" % (10 * i)))
        np.savetxt(os.path.join(root, "pose", "%d.txt" % (10 * i)), p, delimiter=" ")
    K4 = np.eye(4, dtype=np.float32)
    K4[:3, :3] = K.numpy()
    np.savetxt(os.path.join(root, "intrinsic", "intrinsic_color.txt"), K4)
    out = str(tmp_path / "out")
    IO.inference_depth(m, inference_dir=root, output_path=out, batch=4, pred_bidir_depth=bidir, **call)
    imgs, pose_files, intr = IO.depth_inputs(root)
    names = [IO.output_names(IO.DEPTH_FILES, IO.depth_keys(bidir), os.path.basename(f)[:-4]) for f in imgs[:-1]]
    _check_file_set(out, [n for ns in names for n in ns.values()])

    Kf = np.loadtxt(intr).astype(np.float32).reshape(4, 4)[:3, :3]
    items = [(IO._rgb_frame(f), IO._pose(p)) for f, p in zip(imgs, pose_files)]
    runner = DepthSequenceRunner(m, (90, 150), 4, "cuda", Kf, visualize=True, pred_bidir_depth=bidir, **call)
    ref = [{k: v.clone() for k, v in r.items()} for r in runner.run(items)]
    seq = infer_depth_sequence(m, torch.from_numpy(np.stack([f for f, _ in items])).cuda(), Kf, [p for _, p in items],
                               pred_bidir_depth=bidir, **call)
    for t in range(len(imgs) - 1):
        for key, dkey in (("vis", "depth"), ("vis_bwd", "depth_bwd")):
            if key not in names[t]:
                continue
            pic = _png(os.path.join(out, names[t][key]))
            assert np.array_equal(pic, ref[t][key].numpy()), (t, key)                         # lossless
            assert np.array_equal(pic, ODE.viz_inverse_depth(ref[t][dkey].numpy())), (t, key)  # the oracle's picture
            r = seq[dkey][t].cpu()
            assert (ref[t][dkey] - r).abs().max() <= 1e-4 * r.abs().max(), (t, dkey)
