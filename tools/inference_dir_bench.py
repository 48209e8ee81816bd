#!/usr/bin/env python
"""The drop-in inference commands against the reference's loop, end to end from image files on disk to result files on disk.

    python tools/inference_dir_bench.py [--frames N] [--batch B] [--readers R] [--writers W] [--reps K]

Synthetic inputs (seeded, written as PNG to a temporary directory that is removed at the end):
  * davis: a flow directory of `--frames` 480x854 frames (DAVIS), gmflow-scale2-regrefine6, padding 32;
  * kitti_flow: KITTI's layout, `<scene>_10.png` and `<scene>_11.png` per scene, at KITTI's four sizes in turn, so that the
    pairs across scenes have frames of two sizes (they run alone, as the reference takes them); same model;
  * kitti_stereo: left / right directories at KITTI's four sizes, gmstereo-scale2-regrefine3, padding 32;
  * eth3d_stereo: one directory of alternating left / right files of ETH3D-like sizes, `inference_size` 512x768.
Two arms per input, alternated `--reps` times in one process:
  1. driver: `inference_flow` / `inference_stereo` (readers, runner with CUDA graphs, device pictures, writer threads);
     its first pass (graph captures included) is reported separately as `first_pass_s`;
  2. loop: the reference's loop restated around the same module: one pair per call, decoded on the main thread,
     uploaded as float32, `infer_flow` / `infer_stereo` at batch 1, the results downloaded, coloured on the CPU by the
     oracle's `flow_to_image` / `vis_disparity`, and saved with PIL (the reference saves flow pictures with PIL and
     disparity pictures with cv2; both deflate at zlib's default level).
Pairs/s is pairs over a host clock around the whole call, ending in a device synchronise.  Reader and writer occupancy is
the threads' busy time over (threads x wall time).  Prints ONE JSON line with the GPU name, power limit and max SM clock,
read in the same run.  Fails without a CUDA device.  Writes nothing to the tree.
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KITTI_SIZES = [(375, 1242), (370, 1226), (374, 1238), (376, 1241)]
ETH3D_SIZES = [(489, 754), (455, 742), (501, 720), (480, 752)]


def _gpu():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


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
    return dirs


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


def _timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


@torch.no_grad()
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=24)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--readers", type=int, default=4)
    ap.add_argument("--writers", type=int, default=8)
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("inference_dir_bench needs a CUDA device: nothing is measured without one")
    from unimatch_b200 import UniMatch, inference_flow, inference_stereo
    from unimatch_b200.spec import WORKLOADS
    from unimatch_b200.synthetic import BENCH_WEIGHTS, synthetic_state_dict

    def model(name):
        cfg = WORKLOADS[name]
        m = UniMatch(**cfg["model"]).eval()
        m.load_state_dict(synthetic_state_dict(seed=326, **BENCH_WEIGHTS, **cfg["model"]), strict=True)
        return m.cuda(), {k: v for k, v in cfg["call"].items() if k != "task"}

    root = tempfile.mkdtemp(prefix="inference_dir_bench_")
    res = {"metric": "pairs/s from image files on disk to result files on disk: drop-in driver vs the reference's loop "
                     "restated around the same module", "gpu": _gpu(), "device": torch.cuda.get_device_name(0),
           "batch": args.batch, "readers": args.readers, "writers": args.writers, "runs": {}}
    try:
        dirs = _write_inputs(root, args.frames)
        flow_m, flow_call = model("gmflow-scale2-regrefine6")
        stereo_m, stereo_call = model("gmstereo-scale2-regrefine3")
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
        }
        for name, (driver, loop) in cases.items():
            run = {"driver": {"wall_s": []}, "loop": {"wall_s": []}}
            for rep in range(args.reps + 1):                      # the first driver pass includes the graph captures
                for arm, fn in (("driver", driver), ("loop", loop)):
                    out = os.path.join(root, "out", name, arm, str(rep))
                    os.makedirs(out)
                    wall, stats = _timed(lambda: fn(out))
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
    finally:
        shutil.rmtree(root, ignore_errors=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
