"""Generate tests/golden/golden_submission.pt by running the REFERENCE's submission writers (build container only).

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_submission.py

`writeFlow` / `writeFlowKITTI` (utils/frame_utils.py:70-121) and `write_pfm` (utils/file_io.py:98-127) are imported from
`/root/reference` read-only and run on seeded float32 maps; the KITTI disparity PNG is the expression of
evaluate_stereo.py:91, and the resize back is the F.interpolate + two-step rescale of evaluate_flow.py:66-70 /
evaluate_stereo.py:86-87.  Only data is stored: the inputs, the file bytes (`.flo`, `.pfm`), the KITTI flow PNGs decoded
with `cv2.imread(IMREAD_ANYDEPTH | IMREAD_COLOR)` (BGR, as cv2 returns them), the uint16 disparities, and the resized maps.

Inputs hold the boundary cases of numpy's float -> uint16 cast: values whose float32 sum with 32768 rounds across an
integer, negative values, values past the 16-bit wrap and past int32, NaN and +-inf -- in short maps and in maps of more
than 4096 elements, so that numpy's SIMD cast path is pinned too.  The resize maps are dyadic (multiples of 1/16 on grids
whose align-corners weights are multiples of 1/8): ATen's CPU kernel sums the four taps in another order than its CUDA kernel,
and only there do both orders give the same bits.  The rescale after it rounds twice, which these maps do exercise.
"""
import os
import sys
import tempfile

import cv2
import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, "/root/reference")

from utils.file_io import write_pfm  # noqa: E402
from utils.frame_utils import writeFlow, writeFlowKITTI  # noqa: E402

SPECIALS = [np.nan, np.inf, -np.inf, -np.nan, 0.0, -0.0, 512.0, -512.0, 511.99, -512.01, 1e6, -1e6, 3.0e38, -3.0e38, 1e10,
            33554432.0, 2147483520.0 / 64, -2147483648.0 / 64, -1.5 / 64, -0.5 / 64, 70000.7 / 64, -70000.2 / 64]


def _flow_values(rng, n):
    """n float32 flow components: near-integer 64 u (the float32 sum with 32768 rounds across the integer), small and
    large negatives, the specials, and a smooth bulk."""
    k = rng.integers(-600, 600, n).astype(np.float64)
    r = rng.choice([1e-3, 2e-3, 3e-3, 0.5 / 256, 1.5 / 256, 0.4999, 0.5, 0.5001], n) * rng.choice([-1, 1], n)
    near = ((k + 1 + r) / 64).astype(np.float32)
    bulk = (rng.standard_normal(n) * 300).astype(np.float32)
    vals = np.where(rng.random(n) < 0.5, near, bulk)
    idx = rng.choice(n, size=min(n, 3 * len(SPECIALS)), replace=False)
    vals[idx] = np.resize(np.array(SPECIALS, dtype=np.float32), len(idx))
    return vals.astype(np.float32)


def _disp_values(rng, n):
    k = rng.integers(-300, 70000, n)
    d = np.where(rng.random(n) < 0.5, (k / 256.0) + rng.choice([-1e-6, 0.0, 1e-6, 0.5 / 256, -0.5 / 256], n),
                 rng.random(n) * 400 - 20).astype(np.float32)
    idx = rng.choice(n, size=min(n, 3 * len(SPECIALS)), replace=False)
    d[idx] = np.resize(np.array([s * 64 / 256 for s in SPECIALS], dtype=np.float32), len(idx))
    return d


def _read(path):
    with open(path, "rb") as f:
        return f.read()


def main():
    rng = np.random.default_rng(2024)
    tmp = tempfile.mkdtemp()
    flows, discs = [], []
    for h, w in ((3, 7), (1, 1), (67, 71), (45, 101)):            # 67 x 71 and 45 x 101: > 4096 elements per channel
        flows.append(_flow_values(rng, 2 * h * w).reshape(2, h, w))
        discs.append(_disp_values(rng, h * w).reshape(h, w))
    out = {"flow": [], "flo_bytes": [], "kitti_flow_bgr": [], "disp": [], "kitti_disp_u16": [], "pfm_bytes": []}
    for f in flows:
        uv = np.moveaxis(f, 0, -1)                                 # the drivers' flow_pr[0].permute(1, 2, 0).numpy()
        writeFlow(os.path.join(tmp, "a.flo"), uv)
        writeFlowKITTI(os.path.join(tmp, "a.png"), uv)
        out["flow"].append(torch.from_numpy(f.copy()))
        out["flo_bytes"].append(torch.frombuffer(bytearray(_read(os.path.join(tmp, "a.flo"))), dtype=torch.uint8))
        bgr = cv2.imread(os.path.join(tmp, "a.png"), cv2.IMREAD_ANYDEPTH | cv2.IMREAD_COLOR)
        out["kitti_flow_bgr"].append(torch.from_numpy(bgr.astype(np.int32)))
    for d in discs:
        out["disp"].append(torch.from_numpy(d.copy()))
        out["kitti_disp_u16"].append(torch.from_numpy((d * 256.).astype(np.uint16).astype(np.int32)))
        write_pfm(os.path.join(tmp, "a.pfm"), d)
        out["pfm_bytes"].append(torch.frombuffer(bytearray(_read(os.path.join(tmp, "a.pfm"))), dtype=torch.uint8))

    # resize back: (inference size, original size) with align-corners weights in multiples of 1/8
    out["resize"] = []
    for (hi, wi), (ho, wo) in (((5, 9), (9, 17)), ((3, 5), (17, 33)), ((9, 17), (9, 17)), ((5, 5), (33, 9))):
        x = (rng.integers(-4096, 4096, (1, 2, hi, wi)) / 16.0).astype(np.float32)
        flow_pr = F.interpolate(torch.from_numpy(x), size=(ho, wo), mode="bilinear", align_corners=True)
        interp = flow_pr.clone()
        flow_pr[:, 0] = flow_pr[:, 0] * wo / wi
        flow_pr[:, 1] = flow_pr[:, 1] * ho / hi
        disp = F.interpolate(torch.from_numpy(x[:, :1]), size=(ho, wo), mode="bilinear", align_corners=True).squeeze(1)[0]
        disp = disp * wo / float(wi)
        out["resize"].append({"pred": torch.from_numpy(x[0]), "interp": interp[0], "flow": flow_pr[0], "disp": disp})
    torch.save(out, os.path.join(HERE, "golden_submission.pt"))
    print("wrote golden_submission.pt")


if __name__ == "__main__":
    main()
