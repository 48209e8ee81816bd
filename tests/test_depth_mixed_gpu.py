"""Mixed-size depth and the rest of the drop-in surface on the device: `um_depth_to_image_ragged` per item against
`um_depth_to_image` (bit for bit) and the oracle, skipped items, a graph following its table; `MixedSizeDepthRunner`
against `infer_depth` on each pair alone and its pictures against `depth_to_image` of its own depths; `inference_depth` on
a directory of mixed sizes; `inference_flow(save_video=True)`; `validate_depth(save_vis_depth=True)`.

Depths are compared within 1e-5 of the largest depth, not bit for bit: the runner encodes a step's frames t and t+1 in one
batch whose size differs from the pair alone, and um_conv2d_tc's summation order follows the launch's tile count (see
UniMatch.encode_frames)."""
import os

import numpy as np
import pytest
import torch
from PIL import Image

import refops_depth
import refops_ragged
from oracle import depth_viz as V
from unimatch_b200 import MixedSizeDepthRunner, VideoFlowRunner
from unimatch_b200 import inference_io as IO
from unimatch_b200.evaluation import validate_depth
from unimatch_b200.inference import _relative_poses, _resize, depth_to_image, infer_depth
from unimatch_b200.synthetic import (IMAGENET_MEAN, IMAGENET_STD, synthetic_model, synthetic_posed_sequence, synthetic_video,
                                     workload_call)

pytestmark = pytest.mark.gpu
_OPS = torch.ops.unimatch_sm100


def _smooth(h, w, seed, lo=0.5, hi=10.0):
    g = torch.Generator().manual_seed(seed)
    coarse = torch.rand((1, 1, max(h // 24, 2), max(w // 24, 2)), generator=g)
    d = torch.nn.functional.interpolate(coarse, size=(h, w), mode="bilinear", align_corners=True)[0, 0]
    return (lo + (hi - lo) * d).float()


def _items():
    """depths from 1x1 to 480x640 with the NaN, constant, inf and negative cases"""
    ds = [_smooth(1, 1, 1), _smooth(480, 640, 2), _smooth(37, 53, 3), _smooth(2, 3, 4), _smooth(100, 1, 5), _smooth(1, 100, 6)]
    nan = _smooth(5, 5, 7)
    nan[2, 3] = float("nan")
    inf = _smooth(16, 16, 8)
    inf[4, 4] = float("inf")                                  # inverse 0: the minimum
    zero = _smooth(9, 11, 9)
    zero[0, 0] = 0.0                                          # inverse +inf at the top rank
    neg = _smooth(13, 7, 10) - 3.0
    ds += [nan, torch.full((7, 9), 2.5), inf, zero, neg, _smooth(480, 1, 11)]
    return ds


def _pack(depths, gap=5):
    recs, off = [], 0
    for d in depths:
        recs.append((off, d.shape[0], d.shape[1], 1.0, 0))
        off += d.numel() + gap
    flat = torch.full((off,), 7.0)
    for (o, h, w, _, _), d in zip(recs, depths):
        flat[o:o + h * w] = d.reshape(-1)
    return flat.cuda(), recs


def test_depth_to_image_ragged_equals_uniform_and_oracle():
    depths = _items()
    flat, recs = _pack(depths)
    skipped = [(0, 481, 4, 1.0, 0), (0, 0, 4, 1.0, 0), (flat.numel() - 3, 2, 2, 1.0, 0)]   # too tall, empty, past the end
    out = torch.full((3 * flat.numel(),), 0xAB, dtype=torch.uint8, device="cuda")
    before = out.clone()
    _OPS.depth_to_image_ragged(flat, refops_ragged.table(recs + skipped, "cuda"), out, 480, 640)
    written = torch.zeros_like(out, dtype=torch.bool)
    for (o, h, w, _, _), d in zip(recs, depths):
        got = out[3 * o:3 * (o + h * w)].view(h, w, 3)
        ref = depth_to_image(d.cuda())
        assert torch.equal(got, ref), (h, w)
        assert np.array_equal(got.cpu().numpy(), V.viz_inverse_depth(d.numpy())), (h, w)
        written[3 * o:3 * (o + h * w)] = True
    assert torch.equal(out[~written], before[~written])                    # gaps and skipped items untouched


def test_depth_to_image_ragged_graph_follows_its_table():
    depths = _items()
    flat, recs = _pack(depths)
    table = refops_ragged.table(recs, "cuda")
    out = torch.zeros((3 * flat.numel(),), dtype=torch.uint8, device="cuda")
    _OPS.depth_to_image_ragged(flat, table, out, 480, 640)                  # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        _OPS.depth_to_image_ragged(flat, table, out, 480, 640)
    # a different table: the items reversed in place, other sizes over the same packed floats
    recs2 = [(o, w, h, 1.0, 0) if h * w > 1 else (o, h, w, 1.0, 0) for (o, h, w, _, _) in reversed(recs)]
    table.copy_(refops_ragged.table(recs2, "cuda"))
    out.zero_()
    g.replay()
    ref = torch.zeros_like(out)
    _OPS.depth_to_image_ragged(flat, refops_ragged.table(recs2, "cuda"), ref, 480, 640)
    torch.cuda.synchronize()
    assert torch.equal(out, ref)


# ------------------------------------------------------------------------------------------------------------ the runner
# consecutive frames change size; in FRAMES the 64x96 frame t of pair 5 needs no resize at padding 16 (the runner still
# converts its 77x120 frame t+1, which the reference's loop cannot run and the driver refuses), DIR_FRAMES avoids that
FRAMES = [(90, 150), (90, 150), (77, 120), (77, 120), (90, 150), (64, 96), (77, 120), (64, 96)]
DIR_FRAMES = [(90, 150), (90, 150), (77, 120), (77, 120), (90, 150), (66, 100), (77, 120), (64, 96)]


def _frames_and_poses(sizes=FRAMES):
    seq, K, poses = synthetic_posed_sequence(len(sizes), 96, 160, seed=31)
    frames = [np.array(Image.fromarray(f).resize((w, h), Image.BILINEAR)) for f, (h, w) in zip(seq.numpy(), sizes)]
    return frames, K, [p.numpy() for p in poses]


def _alone(m, call, f0, f1, K, rel, bidir, inference_size):
    """`infer_depth` on one pair: frames normalised on the CPU, frame t+1 resized to frame t's inference size"""
    n0, n1 = (refops_depth.normalize_frames(torch.from_numpy(f)[None], IMAGENET_MEAN, IMAGENET_STD).cuda() for f in (f0, f1))
    size = inference_size or tuple(-(-s // 16) * 16 for s in f0.shape[:2])
    if tuple(n1.shape[-2:]) != tuple(size):
        n1 = _resize(n1, size)
    pose = np.stack([rel, np.linalg.inv(rel)]) if bidir else rel[None]
    return infer_depth(m, n0, n1, K.cuda()[None], torch.from_numpy(pose.astype(np.float32)).cuda(), padding_factor=16,
                       inference_size=inference_size, pred_bidir_depth=bidir, **call)


CASES = {"plain": dict(), "bidir": dict(pred_bidir_depth=True), "size": dict(inference_size=(64, 96)),
         "buckets": dict(max_buckets=1)}


@pytest.mark.parametrize("case", sorted(CASES))
def test_mixed_size_depth_runner(case):
    flags = CASES[case]
    bidir = flags.get("pred_bidir_depth", False)
    m = synthetic_model("gmdepth-scale1-regrefine1")
    call = workload_call("gmdepth-scale1-regrefine1", drop=("task", "min_depth", "max_depth", "num_depth_candidates"))
    frames, K, poses = _frames_and_poses()
    pairs = [(frames[t], frames[t + 1], _relative_poses(poses[t:t + 2], False)[0]) for t in range(len(frames) - 1)]
    runner = MixedSizeDepthRunner(m, (90, 150), 2, "cuda", K, visualize=True, **flags, **call)
    got = {i: {k: v.clone() for k, v in r.items()} for i, r in runner.run(pairs)}
    assert sorted(got) == list(range(len(pairs)))
    assert runner.stats["pairs"] == len(pairs)
    if case == "buckets":
        assert runner.stats["captures"] > 1 and len(runner.buckets) == 1
    worst = 0.0
    for i, (f0, f1, rel) in enumerate(pairs):
        ref = _alone(m, call, f0, f1, K, rel, bidir, flags.get("inference_size"))
        for dkey, vkey in (("depth", "vis"), ("depth_bwd", "vis_bwd")) if bidir else (("depth", "vis"),):
            d = got[i][dkey]
            assert d.shape == f0.shape[:2]
            r = ref[dkey][0].cpu()
            worst = max(worst, float((d - r).abs().max() / r.abs().max()))
            assert torch.equal(got[i][vkey], depth_to_image(d.cuda()).cpu()), (i, vkey)
    print("%s: largest difference to the pair alone, relative to its largest depth: %.2e" % (case, worst))
    assert worst <= 1e-5


def _scannet_dir(root, frames, poses, K):
    for sub in ("color", "pose", "intrinsic"):
        os.makedirs(os.path.join(root, sub))
    for i, (f, p) in enumerate(zip(frames, poses)):
        Image.fromarray(f).save(os.path.join(root, "color", "%03d.png" % i))
        np.savetxt(os.path.join(root, "pose", "%03d.txt" % i), p, delimiter=" ")
    K4 = np.eye(4, dtype=np.float32)
    K4[:3, :3] = K.numpy()
    np.savetxt(os.path.join(root, "intrinsic", "intrinsic_color.txt"), K4)


@pytest.mark.parametrize("bidir", [False, True])
def test_inference_depth_mixed_directory(tmp_path, bidir):
    m = synthetic_model("gmdepth-scale1-regrefine1")
    call = workload_call("gmdepth-scale1-regrefine1", drop=("task", "min_depth", "max_depth", "num_depth_candidates"))
    frames, K, poses = _frames_and_poses(DIR_FRAMES)
    root = str(tmp_path / "scene")
    _scannet_dir(root, frames, poses, K)
    out = str(tmp_path / "out")
    stats = IO.inference_depth(m, inference_dir=root, output_path=out, batch=2, pred_bidir_depth=bidir, **call)
    imgs, pose_files, intr = IO.depth_inputs(root)
    names = [IO.output_names(IO.DEPTH_FILES, IO.depth_keys(bidir), os.path.basename(f)[:-4]) for f in imgs[:-1]]
    assert set(os.listdir(out)) == {n for ns in names for n in ns.values()}
    assert stats["pairs"] == len(imgs) - 1
    # the reference's loop restated around the same module: each pair alone, its picture painted from that depth
    Kf = torch.from_numpy(np.loadtxt(intr).astype(np.float32).reshape(4, 4)[:3, :3])
    items = [(IO._rgb_frame(f), IO._pose(p)) for f, p in zip(imgs, pose_files)]
    worst = 0.0
    for t in range(len(items) - 1):
        rel = np.linalg.inv(items[t + 1][1]) @ items[t][1]
        ref = _alone(m, call, items[t][0], items[t + 1][0], Kf, rel, bidir, None)
        for key, dkey in (("vis", "depth"), ("vis_bwd", "depth_bwd")):
            if key not in names[t]:
                continue
            pic = np.array(Image.open(os.path.join(out, names[t][key])))
            want = depth_to_image(ref[dkey][0]).cpu().numpy()
            assert pic.shape == want.shape
            frac = float((pic != want).any(-1).mean())
            worst = max(worst, frac)
            assert frac <= 0.01 and np.abs(pic.astype(np.int16) - want).max() <= 16, (t, key, frac)
    print("pixels whose colour differs from the pair alone: at most %.2e of a picture" % worst)


# ------------------------------------------------------------------------------------------------------------ the video
def _mp4(tmp_path, frames, fps):
    import cv2
    path = str(tmp_path / "clip.mp4")
    w = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"mp4v"), fps, (frames.shape[2], frames.shape[1]))
    assert w.isOpened()
    for f in frames:
        w.write(cv2.cvtColor(f, cv2.COLOR_RGB2BGR))
    w.release()
    cap = cv2.VideoCapture(path)
    decoded = []
    while True:
        ok, img = cap.read()
        if not ok:
            break
        decoded.append(cv2.cvtColor(img, cv2.COLOR_BGR2RGB))
    cap.release()
    return path, np.stack(decoded)


def _read_video(path):
    import cv2
    cap = cv2.VideoCapture(path)
    fps = cap.get(cv2.CAP_PROP_FPS)
    frames = []
    while True:
        ok, img = cap.read()
        if not ok:
            break
        frames.append(cv2.cvtColor(img, cv2.COLOR_BGR2RGB))
    cap.release()
    return fps, frames


@pytest.mark.parametrize("concat", [False, True])
def test_inference_flow_save_video(tmp_path, concat):
    m = synthetic_model("gmflow-scale1")
    call = workload_call("gmflow-scale1", drop=("task", "min_depth", "max_depth", "num_depth_candidates"))
    path, decoded = _mp4(tmp_path, synthetic_video(7, 96, 160, seed=23).numpy(), 10.0)
    flags = dict(pred_bidir_flow=True, save_flo_flow=True, padding_factor=16, batch=3)
    out, plain = str(tmp_path / "out"), str(tmp_path / "plain")
    IO.inference_flow(m, inference_video=path, output_path=out, save_video=True, concat_flow_img=concat, **flags, **call)
    IO.inference_flow(m, inference_video=path, output_path=plain, **flags, **call)
    n = len(decoded) - 1
    video = IO.video_name(path, concat)
    assert video == ("clip_flow_img.mp4" if concat else "clip_flow.mp4")
    assert set(os.listdir(out)) == {f for f in os.listdir(plain) if not f.endswith("_flow.png")} | {video}
    for f in os.listdir(out):                                  # the other files are what a run without save_video writes
        if f != video:
            assert open(os.path.join(out, f), "rb").read() == open(os.path.join(plain, f), "rb").read(), f
    fps, got = _read_video(os.path.join(out, video))
    assert fps == pytest.approx(10.0) and len(got) == n
    runner = VideoFlowRunner(m, decoded.shape[1:3], 3, "cuda", padding_factor=16, visualize=True, concat_frame=concat,
                             pred_bidir_flow=True, **call)
    want = [r["vis"].numpy().copy() for r in runner.run(decoded)]
    assert len(want) == n
    mae = max(float(np.abs(g.astype(np.float64) - w).mean()) for g, w in zip(got, want))
    assert got[0].shape == want[0].shape
    print("video (%s): largest mean absolute error of a decoded frame against its picture: %.2f" % (video, mae))
    assert mae <= 10.0


# ------------------------------------------------------------------------------------------------------- validate_depth
def _depth_samples():
    """five posed samples of two interleaved sizes; sample 3's mask is empty"""
    out = []
    for i, (h, w) in enumerate([(64, 96), (48, 80), (64, 96), (48, 80), (64, 96)]):
        frames, K, poses = synthetic_posed_sequence(2, h, w, seed=60 + i)
        img = refops_depth.normalize_frames(frames, IMAGENET_MEAN, IMAGENET_STD)
        p = poses.numpy()
        rel = torch.from_numpy((np.linalg.inv(p[1]) @ p[0]).astype(np.float32))
        gt = torch.full((h, w), 2.0) + 0.1 * torch.rand((h, w), generator=torch.Generator().manual_seed(i))
        valid = torch.zeros((h, w)) if i == 3 else torch.ones((h, w))
        out.append({"img_ref": img[0], "img_tgt": img[1], "intrinsics": K, "pose": rel, "depth": gt, "valid": valid})
    return out


@pytest.mark.parametrize("protocol,size", [("scannet", None), ("demon", (64, 96))])
def test_validate_depth_save_vis(tmp_path, monkeypatch, protocol, size):
    import unimatch_b200.evaluation as E
    m = synthetic_model("gmdepth-scale1-regrefine1")
    call = workload_call("gmdepth-scale1-regrefine1", drop=("task", "min_depth", "max_depth", "num_depth_candidates"))
    samples = _depth_samples()
    plain = validate_depth(m, samples, protocol=protocol, batch=2, inference_size=size, **call)
    painted = []

    def recording(pred, out=None):
        pics = depth_to_image(pred, out)
        painted.append((pred.clone(), pics.clone()))
        return pics

    monkeypatch.setattr(E, "depth_to_image", recording)
    save_dir = str(tmp_path / "vis")
    res = validate_depth(m, samples, protocol=protocol, batch=2, inference_size=size, save_vis_depth=True, save_dir=save_dir,
                         **call)
    assert res == plain
    # batches: samples 0 and 2 (64x96, full), 1 and 3 (48x80, full), then 4; sample 3 has an empty mask
    order = [0, 2, 1, 3, 4]
    preds = {}
    for pred, pics in painted:
        for j in range(pred.shape[0]):
            preds[order[len(preds)]] = (pred[j], pics[j])
    pattern = "%04d_depth_pred.png" if protocol == "scannet" else "%04d.png"
    valid = [0, 1, 2, 4]
    assert sorted(os.listdir(save_dir)) == [pattern % (k + 1) for k in range(len(valid))]
    for k, i in enumerate(valid):
        pic = np.array(Image.open(os.path.join(save_dir, pattern % (k + 1))))
        pred, pics = preds[i]
        assert np.array_equal(pic, pics.cpu().numpy()), i
        assert np.array_equal(pic, depth_to_image(pred).cpu().numpy()), i
        assert np.array_equal(pic, V.viz_inverse_depth(pred.cpu().numpy())), i
