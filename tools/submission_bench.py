#!/usr/bin/env python
"""Submission throughput: the reference's one-pair-at-a-time `--submission` loop against the batched drivers, on one GPU.

    python tools/submission_bench.py --protocol sintel|kitti|kitti15 [--samples N] [--batch B] [--writers T]

Workload: a seeded synthetic dataset at the protocol's real size (Sintel 436x1024 `.flo`; KITTI flow and KITTI 2015
disparity 16-bit PNGs at 375x1242) run by gmflow-scale2-regrefine6 or gmstereo-scale2 with
`synthetic_state_dict(**BENCH_WEIGHTS)`.  Timed, after one untimed pass of each, into fresh temporary directories:
  * reference loop, restated around this module: one pair per `model(...)` call, the prediction unpadded and copied to the
    host as float32, the file written on the main thread -- writeFlow's numpy interleave for `.flo`, and for the PNGs the
    reference's numpy expression then cv2.imwrite when cv2 is installed (else the same numpy and this project's PNG writer);
  * batched: `create_flow_submission` / `create_stereo_submission` at batch B with T writer threads.
Also: device-to-host bytes per sample of both, the `um_encode_submission` time on one batch (CUDA events over 50 launches),
and the writer pool's occupancy (summed job time / (T x wall time)).  Prints the card, its power limit and SM clocks
(query-only nvidia-smi) and ONE JSON line.  Checks that both paths wrote the same number of files.  Writes nothing to the
tree.
"""
import argparse
import json
import os
import shutil
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True

from tools.common import card, timed  # noqa: E402
from unimatch_b200 import ops, submission  # noqa: E402
from unimatch_b200.inference import InputPadder  # noqa: E402
from unimatch_b200.spec import WORKLOADS  # noqa: E402
from unimatch_b200.synthetic import IMAGENET_MEAN, IMAGENET_STD, synthetic_model, workload_call  # noqa: E402

PROTOCOLS = {  # protocol -> (task, workload, size, padding factor, InputPadder mode, format)
    "sintel": ("flow", "gmflow-scale2-regrefine6", (436, 1024), 32, "sintel", ops.SUBMIT_FLO),
    "kitti": ("flow", "gmflow-scale2-regrefine6", (375, 1242), 32, "kitti", ops.SUBMIT_KITTI_FLOW_PNG),
    "kitti15": ("stereo", "gmstereo-scale2", (375, 1242), 32, "sintel", ops.SUBMIT_KITTI_DISP_PNG),
}


def dataset(task, protocol, size, n, seed=0):
    g = torch.Generator().manual_seed(seed)
    mean, std = torch.tensor(IMAGENET_MEAN).view(3, 1, 1), torch.tensor(IMAGENET_STD).view(3, 1, 1)
    out = []
    for i in range(n):
        a, b = (torch.rand((3,) + size, generator=g) * 255 for _ in range(2))
        if task == "stereo":
            out.append({"left": (a / 255 - mean) / std, "right": (b / 255 - mean) / std, "left_name": "%06d_10.png" % i})
        elif protocol == "sintel":
            out.append((a, b, ("scene_%d" % (i // 8), i % 8)))
        else:
            out.append((a, b, ("%06d_10.png" % i,)))
    return out


def _cv2():
    try:
        import cv2
        return cv2
    except ImportError:
        return None


def _write_png16(path, px, cv2):
    """The reference's PNG write of a uint16 image (RGB [H, W, 3] or grey [H, W])."""
    if cv2 is not None:
        cv2.imwrite(path, px[..., ::-1] if px.ndim == 3 else px)
        return
    rows = np.concatenate([np.zeros((px.shape[0], 1), np.uint8), px.astype(">u2").view(np.uint8).reshape(px.shape[0], -1)], 1)
    submission._write_png(path, rows.tobytes(), px.shape[0], px.shape[1], 16, 2 if px.ndim == 3 else 0)


@torch.no_grad()
def reference_loop(model, data, out, task, protocol, pad, mode, kw, cv2):
    """create_sintel_submission / create_kitti_submission (evaluate_flow.py:19-156) and evaluate_stereo.py's
    create_kitti_submission (:28-91) with the dataset and `.cuda()` taken out; returns device-to-host bytes."""
    d2h = 0
    os.makedirs(out, exist_ok=True)
    for s in data:
        a, b = (s["left"], s["right"]) if task == "stereo" else (s[0], s[1])
        a, b = a[None].cuda(), b[None].cuda()
        padder = InputPadder(a.shape, mode=mode, padding_factor=pad)
        a, b = padder.pad(a, b)
        pred = model(a, b, task=task, **kw)["flow_preds"][-1]
        if task == "stereo":
            disp = padder.unpad(pred)[0].cpu().numpy()
            d2h += disp.nbytes
            _write_png16(os.path.join(out, s["left_name"]), (disp * 256.).astype(np.uint16), cv2)
            continue
        flow = padder.unpad(pred[0]).permute(1, 2, 0).cpu().numpy()
        d2h += flow.nbytes
        if protocol == "sintel":
            d = os.path.join(out, "clean", s[2][0])
            os.makedirs(d, exist_ok=True)
            h, w = flow.shape[:2]
            tmp = np.zeros((h, w * 2))
            tmp[:, np.arange(w) * 2] = flow[:, :, 0]
            tmp[:, np.arange(w) * 2 + 1] = flow[:, :, 1]
            with open(os.path.join(d, "frame%04d.flo" % (s[2][1] + 1)), "wb") as f:
                f.write(submission.flo_header(h, w))
                tmp.astype(np.float32).tofile(f)
        else:
            uv = 64.0 * flow + 2 ** 15
            uv = np.concatenate([uv, np.ones(uv.shape[:2] + (1,))], axis=-1).astype(np.uint16)
            _write_png16(os.path.join(out, s[2][0]), uv, cv2)
    return d2h


def _count(root):
    return sum(len(fs) for _, _, fs in os.walk(root))


def encode_ms(batch, size, pad, fmt, iters=50):
    """um_encode_submission on one batch of padded model outputs, unpad crop: CUDA events around `iters` launches."""
    c = ops.SUBMIT_CHANNELS[fmt]
    ph, pw = (-size[0]) % pad, (-size[1]) % pad
    pred = torch.randn((batch, c, size[0] + ph, size[1] + pw), device="cuda") * 20
    enc = torch.ops.unimatch_sm100.encode_submission
    for _ in range(3):
        enc(pred, fmt, size[0], size[1], False, ph // 2, pw // 2)
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        enc(pred, fmt, size[0], size[1], False, ph // 2, pw // 2)
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--protocol", required=True, choices=sorted(PROTOCOLS))
    ap.add_argument("--samples", type=int, default=32)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--writers", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("submission_bench needs a CUDA device")
    task, workload, size, pad, mode, fmt = PROTOCOLS[args.protocol]
    model = synthetic_model(workload)
    kw = workload_call(workload, drop=("task",))
    data = dataset(task, args.protocol, size, args.samples)
    cv2 = _cv2()
    driver = submission.create_stereo_submission if task == "stereo" else submission.create_flow_submission
    proto = "kitti" if task == "stereo" else args.protocol

    def loop(d, out):
        return {"d2h_bytes": reference_loop(model, d, out, task, args.protocol, pad, mode, kw, cv2), "samples": len(d)}

    def batched(d, out):
        return driver(model, d, protocol=proto, output_path=out, batch=args.batch, padding_factor=pad, writers=args.writers, **kw)

    gpu = ", ".join(card().values())
    print("card:", gpu, flush=True)
    root = tempfile.mkdtemp(prefix="submission_bench.")
    res = dict(protocol=args.protocol, workload=workload, size=list(size), samples=args.samples, batch=args.batch,
               writers=args.writers, reference_png_writer="cv2" if cv2 is not None else "numpy + stdlib zlib")
    try:
        files = {}
        for name, fn in (("reference_loop", loop), ("batched", batched)):
            fn(data[:args.batch], os.path.join(root, name + "_warm"))
            out = os.path.join(root, name)
            wall, stats = timed(lambda: fn(data, out))
            files[name] = _count(out)
            res[name + "_samples_per_s"] = args.samples / wall
            res[name + "_d2h_bytes_per_sample"] = stats["d2h_bytes"] / args.samples
            if name == "batched":
                res["writer_occupancy"] = stats["writer_seconds"] / (args.writers * wall)
        res["speedup"] = res["batched_samples_per_s"] / res["reference_loop_samples_per_s"]
        res["encode_ms_per_batch"] = encode_ms(args.batch, size, pad, fmt)
        res["files"] = files
    finally:
        shutil.rmtree(root, ignore_errors=True)
    res["card"] = gpu
    print(json.dumps(res))
    if files["reference_loop"] != files["batched"] or files["batched"] != args.samples:
        sys.exit("the two paths wrote different numbers of files")


if __name__ == "__main__":
    main()
