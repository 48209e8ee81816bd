"""Generate tests/golden/golden_disp_vis.pt by running the REFERENCE's disparity visualisation (build container only).

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_disp_vis.py

`vis_disparity` (utils/visualization.py:11-16, what the stereo driver paints, evaluate_stereo.py:826, :840) is imported from
`/root/reference` read-only, with `matplotlib` / `matplotlib.cm` stubbed (import-time-only dependencies of that module), and
run with cv2 on seeded float32 disparities: odd sizes and a batch, smooth wide-range and negative fields, values whose
normalised `x * 255` lands just below an integer (a contracted or reassociated expression moves them across it), a constant
image, +-NaN, +-inf, and a disparity map of the oracle's stereo forward.  The oracle restatement (oracle/disp_viz.py) must
equal it byte for byte; the disparities and the reference pictures are stored for the box where the reference does not exist.
"""
import os
import sys
import types
import warnings

import numpy as np
import torch

warnings.filterwarnings("ignore")
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, "/root/reference")
_mpl = types.ModuleType("matplotlib")
_mpl.cm = types.ModuleType("matplotlib.cm")
_mpl.cm.get_cmap = None
sys.modules.setdefault("matplotlib", _mpl)
sys.modules.setdefault("matplotlib.cm", _mpl.cm)

from oracle import disp_viz as OD  # noqa: E402
from oracle import unimatch_oracle as O  # noqa: E402
from unimatch_b200.spec import WORKLOADS  # noqa: E402
from unimatch_b200.synthetic import BENCH_WEIGHTS, synthetic_pair, synthetic_state_dict  # noqa: E402
from utils.visualization import vis_disparity  # noqa: E402


def _smooth(g, n, h, w, lo, hi):
    x = torch.rand((n, 1, max(h // 8, 2), max(w // 8, 2)), generator=g)
    x = torch.nn.functional.interpolate(x, size=(h, w), mode="bilinear", align_corners=True)[:, 0]
    return (lo + (hi - lo) * x + 0.01 * (hi - lo) * torch.rand((n, h, w), generator=g)).float()


def _ulp_values(rng):
    """(mn, mx, values): every float32 disparity d within 4 ulps of mn + k (mx - mn) / 255, k = 1..254, whose fp32
    ((d - mn) / (mx - mn)) * 255 truncates below the integer that a reassociated form (d - mn) * (255 / (mx - mn)), or the
    exact value, reaches (or above it)."""
    f = np.float32
    mn, mx = f(rng.uniform(-40, 10)), f(rng.uniform(60, 400))
    rng_ = f(mx - mn)
    scale = f(f(255.0) / rng_)
    found = set()
    for k in range(1, 255):
        d = f(mn + f(k * float(rng_) / 255.0))
        for _ in range(4):
            d = np.nextafter(d, f(-np.inf))
        for _ in range(9):                                # the 4 ulps either side of the nearest float to the integer
            q = f(f(f(d - mn) / rng_) * f(255.0))
            alt = f(f(d - mn) * scale)
            exact = (float(d) - float(mn)) / (float(mx) - float(mn)) * 255.0
            if mn < d < mx and (int(q) != int(alt) or int(q) != int(exact)):
                found.add(float(d))
            d = np.nextafter(d, f(np.inf))
    return mn, mx, rng.permutation(np.array(sorted(found), np.float32))


def cases():
    """name -> float32 disparities [N, H, W]"""
    g = torch.Generator().manual_seed(2025)
    rng = np.random.default_rng(2025)
    out = {"one_1x1": torch.tensor([[[3.5]]]),
           "odd_37x53": _smooth(g, 2, 37, 53, 0.5, 180.0),
           "batch_2x120x208": _smooth(g, 2, 120, 208, 0.0, 300.0),
           "negative": _smooth(g, 1, 24, 40, -60.0, -5.0),
           "signed": _smooth(g, 1, 24, 40, -25.0, 25.0)}
    for name in ("ulp_a", "ulp_b"):
        mn, mx, vals = _ulp_values(rng)
        assert len(vals) >= 50, (name, len(vals))
        out[name] = torch.from_numpy(np.concatenate([vals[:len(vals) // 2], [mx, mn], vals[len(vals) // 2:]]))[None, None]
    out["constant"] = torch.full((1, 16, 24), 7.25)
    for name, v in (("nan_pos", float("nan")), ("nan_neg", -float("nan")), ("inf_pos", float("inf")),
                    ("inf_neg", -float("inf"))):
        d = _smooth(g, 1, 16, 24, 1.0, 50.0)
        d[0, 5, 7] = v
        out[name] = d
    nan_neg = out["nan_neg"].numpy()
    assert np.signbit(nan_neg[0, 5, 7]) and np.isnan(nan_neg[0, 5, 7])
    cfg = WORKLOADS["gmstereo-scale2"]
    sd = synthetic_state_dict(seed=326, **BENCH_WEIGHTS, **cfg["model"])
    mk = {k: cfg["model"][k] for k in ("num_scales", "upsample_factor", "reg_refine")}
    pair = synthetic_pair("stereo", 64, 96, index=3)
    out["oracle_stereo_64x96"] = O.forward(sd, pair["img0"], pair["img1"], **mk, **cfg["call"])["flow_preds"][-1].float()
    return {k: v.float().contiguous() for k, v in out.items()}


def main():
    res = {}
    for name, disp in cases().items():
        ref = np.stack([vis_disparity(d.numpy().copy()) for d in disp], 0)
        got = OD.vis_disparity_batch(disp.numpy())
        assert ref.dtype == np.uint8 and got.dtype == np.uint8 and ref.shape == got.shape, name
        assert np.array_equal(ref, got), "oracle vis_disparity != reference on %s (%d bytes differ)" % (name, (ref != got).sum())
        res[name] = dict(disp=disp, image=torch.from_numpy(ref))
        print("%-20s %s  oracle == reference byte for byte" % (name, tuple(disp.shape)))
    path = os.path.join(HERE, "golden_disp_vis.pt")
    torch.save(res, path)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
