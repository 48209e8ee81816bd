#!/usr/bin/env python
"""The drop-in inference commands against the reference's loop, end to end from image files on disk to result files on disk.

    python tools/inference_dir_bench.py [--frames N] [--batch B] [--readers R] [--writers W] [--reps K]

Synthetic inputs (seeded, written as PNG to a temporary directory that is removed at the end):
  * davis: a flow directory of `--frames` 480x854 frames (DAVIS), gmflow-scale2-regrefine6, padding 32;
  * kitti_flow: KITTI's layout, `<scene>_10.png` and `<scene>_11.png` per scene, at KITTI's four sizes in turn, so that the
    pairs across scenes have frames of two sizes (they run alone, as the reference takes them); same model;
  * kitti_stereo: left / right directories at KITTI's four sizes, gmstereo-scale2-regrefine3, padding 32;
  * eth3d_stereo: one directory of alternating left / right files of ETH3D-like sizes, `inference_size` 512x768;
  * davis_video / davis_video_save: the DAVIS frames as an mp4 (cv2, mp4v), through `inference_video`, without and with
    `save_video` (the flow pictures go to one mp4 instead of PNG files);
  * scannet_depth: a ScanNet-layout directory of `--frames` 480x640 frames, gmdepth-scale1-regrefine1 (one frame size:
    the sequence runner, every frame encoded once);
  * scannet_mixed_depth / scannet_mixed_depth_size: the same layout with three interleaved frame sizes (468x624,
    470x630, 375x500), without and with `inference_size` 384x512 (the mixed-size depth runner).
Two arms per input, alternated `--reps` times in one process:
  1. driver: `inference_flow` / `inference_stereo` / `inference_depth` (readers, runner with CUDA graphs, device pictures,
     writer threads); its first pass (graph captures included) is reported separately as `first_pass_s`;
  2. loop: the reference's loop restated around the same module: one pair per call, decoded on the main thread,
     uploaded as float32, `infer_flow` / `infer_stereo` / `infer_depth` at batch 1, the results downloaded, coloured on the
     CPU by the oracle's `flow_to_image` / `vis_disparity` / `viz_inverse_depth`, and saved with PIL (the reference saves
     flow and depth pictures with PIL and disparity pictures with cv2; both deflate at zlib's default level), or for
     `save_video` appended to one mp4 by cv2.
Also `depth_to_image_us`: `um_depth_to_image_ragged` against `um_depth_to_image` on one full step of 16 480x640 depths
(a `pred_bidir_depth` step of 8 pairs), CUDA events over 50 calls of each, alternated three times.
Pairs/s is pairs over a host clock around the whole call, ending in a device synchronise.  Reader and writer occupancy is
the threads' busy time over (threads x wall time).  Prints ONE JSON line with the GPU name, power limit and max SM clock,
read in the same run.  Fails without a CUDA device.  Writes nothing to the tree.
"""
import argparse
import json
import os
import shutil
import sys
import tempfile

import numpy as np
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.common import card, timed  # noqa: E402

KITTI_SIZES = [(375, 1242), (370, 1226), (374, 1238), (376, 1241)]
ETH3D_SIZES = [(489, 754), (455, 742), (501, 720), (480, 752)]
SCANNET_MIXED = [(468, 624), (470, 630), (375, 500)]     # none already at its inference size (see inference_depth)


def _write_inputs(root, n_frames):
    from unimatch_b200.synthetic import synthetic_video
    dirs = {k: os.path.join(root, k) for k in ("davis", "kitti_flow", "kitti_left", "kitti_right", "eth3d")}
    for d in dirs.values():
        os.makedirs(d)
    for t, f in enumerate(synthetic_video(n_frames, 480, 854, seed=5).numpy()):
        Image.fromarray(f).save(os.path.join(dirs["davis"], "%05d.png" % t), compress_level=1)
    for s in range(n_frames // 2):
        h, w = KITTI_SIZES[s % 4]
        a, b = synthetic_video(2, h, w, seed=100 + s).numpy()
        Image.fromarray(a).save(os.path.join(dirs["kitti_flow"], "%06d_10.png" % s), compress_level=1)
        Image.fromarray(b).save(os.path.join(dirs["kitti_flow"], "%06d_11.png" % s), compress_level=1)
        Image.fromarray(a).save(os.path.join(dirs["kitti_left"], "%06d_10.png" % s), compress_level=1)
        Image.fromarray(b).save(os.path.join(dirs["kitti_right"], "%06d_10.png" % s), compress_level=1)
        h, w = ETH3D_SIZES[s % 4]
        a, b = synthetic_video(2, h, w, seed=200 + s).numpy()
        Image.fromarray(a).save(os.path.join(dirs["eth3d"], "scene%03d_0.png" % s), compress_level=1)
        Image.fromarray(b).save(os.path.join(dirs["eth3d"], "scene%03d_1.png" % s), compress_level=1)
    import cv2
    dirs["video"] = os.path.join(root, "davis.mp4")
    writer = cv2.VideoWriter(dirs["video"], cv2.VideoWriter_fourcc(*"mp4v"), 24.0, (854, 480))
    for t in range(n_frames):
        writer.write(cv2.cvtColor(np.array(Image.open(os.path.join(dirs["davis"], "%05d.png" % t))), cv2.COLOR_RGB2BGR))
    writer.release()
    for name, sizes in (("scannet", [(480, 640)]), ("scannet_mixed", SCANNET_MIXED)):
        dirs[name] = _write_scannet(os.path.join(root, name), n_frames, sizes)
    return dirs


def _write_scannet(root, n_frames, sizes):
    from unimatch_b200.synthetic import synthetic_posed_sequence
    for sub in ("color", "pose", "intrinsic"):
        os.makedirs(os.path.join(root, sub))
    frames, K, poses = synthetic_posed_sequence(n_frames, 480, 640, seed=7)
    for t, (f, p) in enumerate(zip(frames.numpy(), poses.numpy())):
        h, w = sizes[t % len(sizes)]
        img = Image.fromarray(f)
        img = img if (h, w) == (480, 640) else img.resize((w, h), Image.BILINEAR)
        img.save(os.path.join(root, "color", "%06d.png" % t), compress_level=1)
        np.savetxt(os.path.join(root, "pose", "%06d.txt" % t), p, delimiter=" ")
    K4 = np.eye(4, dtype=np.float32)
    K4[:3, :3] = K.numpy()
    np.savetxt(os.path.join(root, "intrinsic", "intrinsic_color.txt"), K4)
    return root


def _flow_loop(model, inference_dir, output_path, padding_factor, call):
    from oracle import flow_viz as OV
    from unimatch_b200 import infer_flow
    from unimatch_b200.inference import _resize
    from unimatch_b200.inference_io import flow_inputs
    files = flow_inputs(inference_dir)
    for t in range(len(files) - 1):
        a, b = (np.array(Image.open(f)).astype(np.uint8)[..., :3] for f in files[t:t + 2])
        a, b = (torch.from_numpy(x).permute(2, 0, 1).float()[None].cuda() for x in (a, b))
        if a.shape != b.shape:     # a timing arm: the second frame is brought to the first one's size on the device
            b = _resize(b, a.shape[-2:])
        flow = infer_flow(model, a, b, padding_factor=padding_factor, **call)["flow"][0].permute(1, 2, 0).cpu().numpy()
        Image.fromarray(OV.flow_to_image(flow)).save(os.path.join(output_path, os.path.basename(files[t])[:-4] + "_flow.png"))


def _video_loop(model, video, output_path, padding_factor, save_video, call):
    """the reference's video branch: every frame decoded first, then one pair per call; with `save_video` the pictures go
    to one mp4 (cv2, mp4v) at the end, as the reference writes its video after the loop"""
    import cv2
    from oracle import flow_viz as OV
    from unimatch_b200 import infer_flow
    from unimatch_b200.inference_io import _VideoWriter, video_name
    cap = cv2.VideoCapture(video)
    fps, frames = cap.get(cv2.CAP_PROP_FPS), []
    while True:
        ok, img = cap.read()
        if not ok:
            break
        frames.append(cv2.cvtColor(img, cv2.COLOR_BGR2RGB))
    cap.release()
    pictures = []
    for t in range(len(frames) - 1):
        a, b = (torch.from_numpy(x).permute(2, 0, 1).float()[None].cuda() for x in frames[t:t + 2])
        flow = infer_flow(model, a, b, padding_factor=padding_factor, **call)["flow"][0].permute(1, 2, 0).cpu().numpy()
        pic = OV.flow_to_image(flow)
        if save_video:
            pictures.append(pic)
        else:
            Image.fromarray(pic).save(os.path.join(output_path, "%04d_flow.png" % t))
    if save_video:
        writer = _VideoWriter(os.path.join(output_path, video_name(video, False)), fps)
        for pic in pictures:
            writer.submit(pic)
        writer.close()


def _depth_loop(model, inference_dir, output_path, inference_size, call):
    """the reference's depth loop (evaluate_depth.py:338-417) around the same module; both frames of a pair are resized to
    the first one's inference size (every first frame of these inputs needs a resize, as the driver requires)"""
    from oracle import depth_viz as ODV
    from unimatch_b200 import infer_depth
    from unimatch_b200.inference import _inference_size, _resize
    from unimatch_b200.inference_io import depth_inputs
    from unimatch_b200.synthetic import IMAGENET_MEAN, IMAGENET_STD
    mean, std = torch.tensor(IMAGENET_MEAN).view(3, 1, 1), torch.tensor(IMAGENET_STD).view(3, 1, 1)
    imgs, poses, intr = depth_inputs(inference_dir)
    K = torch.from_numpy(np.loadtxt(intr).astype(np.float32).reshape((4, 4))[:3, :3]).cuda()[None]
    for t in range(len(imgs) - 1):
        a, b = ((torch.from_numpy(np.array(Image.open(f).convert("RGB")).astype(np.float32)).permute(2, 0, 1) / 255. - mean)
                / std for f in imgs[t:t + 2])
        p0, p1 = (np.loadtxt(f, delimiter=" ").astype(np.float32).reshape((4, 4)) for f in poses[t:t + 2])
        pose = torch.from_numpy(np.linalg.inv(p1) @ p0).cuda()[None]
        a, b = a[None].cuda(), b[None].cuda()
        size = _inference_size(tuple(a.shape[-2:]), 16, inference_size)
        if b.shape != a.shape:
            b = _resize(b, size)
        depth = infer_depth(model, a, b, K, pose, padding_factor=16, inference_size=inference_size, **call)["depth"][0]
        Image.fromarray(ODV.viz_inverse_depth(depth.cpu().numpy())).save(
            os.path.join(output_path, os.path.basename(imgs[t])[:-4] + ".png"))


def _depth_to_image_us():
    """mean microseconds per call of the uniform and the ragged depth colouring on one full bidirectional step"""
    from unimatch_b200.inference import RAGGED_ITEM
    ops_ = torch.ops.unimatch_sm100
    n, h, w = 16, 480, 640
    g = torch.Generator().manual_seed(3)
    coarse = torch.rand((n, 1, 20, 26), generator=g)
    depth = (0.5 + 9.5 * torch.nn.functional.interpolate(coarse, size=(h, w), mode="bilinear",
                                                         align_corners=True)[:, 0]).contiguous().cuda()
    pics, flat = torch.empty((n, h, w, 3), dtype=torch.uint8, device="cuda"), depth.view(-1)
    table = np.array([(i * h * w, h, w, 1.0, 0) for i in range(n)], RAGGED_ITEM)
    items = torch.from_numpy(table.view(np.uint8).reshape(n, -1).copy()).cuda()
    ragged = torch.empty((3 * flat.numel(),), dtype=torch.uint8, device="cuda")
    arms = {"uniform": lambda: ops_.depth_to_image(depth, pics),
            "ragged": lambda: ops_.depth_to_image_ragged(flat, items, ragged, h, w)}
    times = {k: [] for k in arms}
    for fn in arms.values():
        for _ in range(5):
            fn()
    for _ in range(3):
        for k, fn in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(50):
                fn()
            e1.record()
            e1.synchronize()
            times[k].append(round(e0.elapsed_time(e1) * 1000.0 / 50, 1))
    torch.cuda.synchronize()
    return dict(times, equal=bool(torch.equal(pics.view(-1), ragged)))


def _stereo_loop(model, dirs, output_path, padding_factor, inference_size, call):
    from oracle import disp_viz as OD
    from unimatch_b200 import infer_stereo
    from unimatch_b200.inference_io import stereo_inputs
    from unimatch_b200.synthetic import IMAGENET_MEAN, IMAGENET_STD
    mean, std = torch.tensor(IMAGENET_MEAN).view(3, 1, 1), torch.tensor(IMAGENET_STD).view(3, 1, 1)
    left, right = stereo_inputs(**dirs)
    for name_l, name_r in zip(left, right):
        a, b = ((torch.from_numpy(np.array(Image.open(f).convert("RGB")).astype(np.float32)).permute(2, 0, 1) / 255. - mean)
                / std for f in (name_l, name_r))
        disp = infer_stereo(model, a[None].cuda(), b[None].cuda(), padding_factor=padding_factor, inference_size=inference_size,
                            **call)["disp"][0].cpu().numpy()
        Image.fromarray(OD.vis_disparity(disp)[..., ::-1]).save(os.path.join(output_path,
                                                                             os.path.basename(name_l)[:-4] + "_disp.png"))


@torch.no_grad()
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=24)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--readers", type=int, default=4)
    ap.add_argument("--writers", type=int, default=8)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--only", default="", help="comma-separated input names to run (default: all)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("inference_dir_bench needs a CUDA device: nothing is measured without one")
    from unimatch_b200 import inference_depth, inference_flow, inference_stereo
    from unimatch_b200.synthetic import synthetic_model, workload_call

    def model(name):
        return synthetic_model(name), workload_call(name, drop=("task",))

    root = tempfile.mkdtemp(prefix="inference_dir_bench_")
    res = {"metric": "pairs/s from image files on disk to result files on disk: drop-in driver vs the reference's loop "
                     "restated around the same module", "gpu": "%(name)s, %(power_limit)s, %(max_sm_clock)s" % card(),
           "device": torch.cuda.get_device_name(0),
           "batch": args.batch, "readers": args.readers, "writers": args.writers, "runs": {}}
    try:
        dirs = _write_inputs(root, args.frames)
        flow_m, flow_call = model("gmflow-scale2-regrefine6")
        stereo_m, stereo_call = model("gmstereo-scale2-regrefine3")
        depth_m, depth_call = model("gmdepth-scale1-regrefine1")
        # the workload's min / max are the model's inverse depths; the drivers take the metric defaults (0.5 m, 10 m)
        depth_call = {k: v for k, v in depth_call.items() if k not in ("min_depth", "max_depth")}
        loop_depth_call = depth_call
        opts = dict(batch=args.batch, readers=args.readers, writers=args.writers)
        cases = {
            "davis_flow": (lambda out: inference_flow(flow_m, inference_dir=dirs["davis"], output_path=out, padding_factor=32,
                                                      **opts, **flow_call),
                           lambda out: _flow_loop(flow_m, dirs["davis"], out, 32, flow_call)),
            "kitti_flow": (lambda out: inference_flow(flow_m, inference_dir=dirs["kitti_flow"], output_path=out,
                                                      padding_factor=32, **opts, **flow_call),
                           lambda out: _flow_loop(flow_m, dirs["kitti_flow"], out, 32, flow_call)),
            "kitti_stereo": (lambda out: inference_stereo(stereo_m, inference_dir_left=dirs["kitti_left"],
                                                          inference_dir_right=dirs["kitti_right"], output_path=out,
                                                          padding_factor=32, **opts, **stereo_call),
                             lambda out: _stereo_loop(stereo_m, dict(inference_dir_left=dirs["kitti_left"],
                                                                     inference_dir_right=dirs["kitti_right"]), out, 32, None,
                                                      stereo_call)),
            "eth3d_stereo": (lambda out: inference_stereo(stereo_m, inference_dir=dirs["eth3d"], output_path=out,
                                                          inference_size=(512, 768), **opts, **stereo_call),
                             lambda out: _stereo_loop(stereo_m, dict(inference_dir=dirs["eth3d"]), out, 32, (512, 768),
                                                      stereo_call)),
            "davis_video": (lambda out: inference_flow(flow_m, inference_video=dirs["video"], output_path=out,
                                                       padding_factor=32, **opts, **flow_call),
                            lambda out: _video_loop(flow_m, dirs["video"], out, 32, False, flow_call)),
            "davis_video_save": (lambda out: inference_flow(flow_m, inference_video=dirs["video"], output_path=out,
                                                            padding_factor=32, save_video=True, **opts, **flow_call),
                                 lambda out: _video_loop(flow_m, dirs["video"], out, 32, True, flow_call)),
            "scannet_depth": (lambda out: inference_depth(depth_m, inference_dir=dirs["scannet"], output_path=out, **opts,
                                                          **depth_call),
                              lambda out: _depth_loop(depth_m, dirs["scannet"], out, None, loop_depth_call)),
            "scannet_mixed_depth": (lambda out: inference_depth(depth_m, inference_dir=dirs["scannet_mixed"], output_path=out,
                                                                **opts, **depth_call),
                                    lambda out: _depth_loop(depth_m, dirs["scannet_mixed"], out, None, loop_depth_call)),
            "scannet_mixed_depth_size": (lambda out: inference_depth(depth_m, inference_dir=dirs["scannet_mixed"],
                                                                     output_path=out, inference_size=(384, 512), **opts,
                                                                     **depth_call),
                                         lambda out: _depth_loop(depth_m, dirs["scannet_mixed"], out, (384, 512),
                                                                 loop_depth_call)),
        }
        if args.only:
            cases = {k: v for k, v in cases.items() if k in args.only.split(",")}
        for name, (driver, loop) in cases.items():
            run = {"driver": {"wall_s": []}, "loop": {"wall_s": []}}
            for rep in range(args.reps + 1):                      # the first driver pass includes the graph captures
                for arm, fn in (("driver", driver), ("loop", loop)):
                    out = os.path.join(root, "out", name, arm, str(rep))
                    os.makedirs(out)
                    wall, stats = timed(lambda: fn(out))
                    if rep == 0:
                        run[arm]["first_pass_s"] = round(wall, 4)
                        continue
                    run[arm]["wall_s"].append(round(wall, 4))
                    if arm == "driver":
                        run["driver"].update(
                            pairs=stats["pairs"], steps=stats["steps"], h2d_bytes=stats["h2d_bytes"],
                            d2h_bytes=stats["d2h_bytes"], files=len(os.listdir(out)),
                            reader_occupancy=round(stats["reader_seconds"] / (args.readers * wall), 3),
                            writer_occupancy=round(stats["writer_seconds"] / (args.writers * wall), 3))
                    shutil.rmtree(out)
            pairs = run["driver"]["pairs"]
            for arm in ("driver", "loop"):
                run[arm]["pairs_per_s"] = [round(pairs / w, 2) for w in run[arm]["wall_s"]]
            run["loop"]["h2d_bytes_note"] = "float32 frames: 24 bytes per pixel of each pair; flows or disparities back as float32"
            res["runs"][name] = run
            torch.cuda.empty_cache()
        res["depth_to_image_us"] = _depth_to_image_us()
    finally:
        shutil.rmtree(root, ignore_errors=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
