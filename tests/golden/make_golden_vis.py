"""Generate tests/golden/golden_vis.pt by running the REFERENCE's flow visualisation (build container only).

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_vis.py

`flow_to_image` (utils/flow_viz.py:240-275, what the video driver paints, evaluate_flow.py:768) is imported from
`/root/reference` read-only and run on seeded float32 flows: random fields of several magnitudes, one with 1e9 unknown-flow
markers, an all-zero field and an odd size.  The oracle restatement (oracle/flow_viz.py) must equal it byte for byte; the
flows and the reference pictures are stored for the box where the reference does not exist.
"""
import os
import sys
import warnings

import numpy as np
import torch

warnings.filterwarnings("ignore")
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, "/root/reference")

from oracle import flow_viz as OV  # noqa: E402
from utils.flow_viz import flow_to_image  # noqa: E402


def cases():
    """name -> planar float32 flow [N, 2, H, W]"""
    g = torch.Generator().manual_seed(2024)
    out = {}
    for name, (n, h, w, scale) in {"small": (3, 24, 40, 0.5), "medium": (3, 48, 64, 8.0), "large": (2, 40, 72, 150.0),
                                  "odd_37x53": (4, 37, 53, 5.0)}.items():
        out[name] = (torch.randn((n, 2, h, w), generator=g) * scale).float()
    smooth = torch.randn((2, 2, 6, 10), generator=g) * 20.0                 # smooth fields: every hue of the wheel
    out["smooth"] = torch.nn.functional.interpolate(smooth, size=(45, 75), mode="bilinear", align_corners=True).float()
    unk = (torch.randn((2, 2, 32, 48), generator=g) * 6.0).float()
    mask = torch.rand((2, 32, 48), generator=g) < 0.1
    unk[:, 0][mask] = 1e9                                                     # .flo unknown-flow markers
    unk[1, 1][torch.rand((32, 48), generator=g) < 0.05] = -1e9
    out["unknown"] = unk
    out["zero"] = torch.zeros((1, 2, 16, 24))
    axes = torch.zeros((1, 2, 8, 8))                                          # pure +-u / +-v: signed zeros in arctan2
    axes[0, 0, :2], axes[0, 0, 2:4], axes[0, 1, 4:6], axes[0, 1, 6:] = 3.0, -3.0, 2.0, -2.0
    out["axes"] = axes
    return out


def main():
    res = {}
    for name, flow in cases().items():
        ref = np.stack([flow_to_image(f.permute(1, 2, 0).numpy().copy()) for f in flow], 0)
        got = OV.flow_to_image_batch(flow.numpy())
        assert ref.dtype == np.uint8 and got.dtype == np.uint8 and ref.shape == got.shape, name
        assert np.array_equal(ref, got), "oracle flow_to_image != reference on %s (%d bytes differ)" % (name, (ref != got).sum())
        res[name] = dict(flow=flow, image=torch.from_numpy(ref))
        print("%-10s %s  oracle == reference byte for byte" % (name, tuple(flow.shape)))
    path = os.path.join(HERE, "golden_vis.pt")
    torch.save(res, path)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
