"""Generate tests/golden/golden_eval.pt by running the REFERENCE's own validation loops (build container only).

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_eval.py

evaluate_flow.validate_{chairs,things,sintel,kitti}, evaluate_stereo.validate_{things,kitti15,eth3d,middlebury} and
evaluate_depth.validate_{scannet,demon} are imported from `/root/reference` read-only and run unchanged, with
  * each function's dataset class rebound to a small seeded in-memory dataset from eval_samples.py (64x96 to 75x130 images, a
    few samples, two shapes for KITTI), with empty masks, zero-magnitude GT and errors exactly on the thresholds;
  * `torch.Tensor.cuda` rebound to the identity (everything runs on the CPU) and imageio / skimage / matplotlib stubbed;
  * `eval_samples.STUB` as the model: an elementwise function of the padded inputs, so the same fp32 predictions come out of
    a batch of one in the reference and of a batch of B in the drivers.
Stored per case: its name, task, driver options, the digest of its samples (the tests rebuild them from eval_samples.py,
which keeps the file small) and the reference's results dict.  The samples come from torch's CPU generator; should a torch
release change its streams, the digest check fails and this script has to be rerun.
"""
import os
import sys
import types
import warnings

import torch

warnings.filterwarnings("ignore")
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, "/root/reference")

for name in ("imageio", "skimage", "skimage.io", "matplotlib", "matplotlib.cm", "matplotlib.colors"):
    mod = types.ModuleType(name)
    mod.get_cmap = lambda *a, **k: None
    sys.modules.setdefault(name, mod)
sys.modules["skimage"].io = sys.modules["skimage.io"]
sys.modules["matplotlib"].cm = sys.modules["matplotlib.cm"]
torch.Tensor.cuda = lambda self, *a, **k: self

import eval_samples as E  # noqa: E402
import evaluate_depth  # noqa: E402
import evaluate_flow  # noqa: E402
import evaluate_stereo  # noqa: E402

# case name -> (reference module, function, dataset class name, the function's own keyword arguments)
REFERENCE = {
    "chairs": (evaluate_flow, "validate_chairs", "FlyingChairs", {}),
    "chairs_speed": (evaluate_flow, "validate_chairs", "FlyingChairs", dict(with_speed_metric=True)),
    "things_speed": (evaluate_flow, "validate_things", "FlyingThings3D",
                     dict(with_speed_metric=True, max_val_flow=100, padding_factor=16)),
    # validate_sintel loops over both passes with the same dataset here; the clean keys are kept
    "sintel_matched_speed": (evaluate_flow, "validate_sintel", "MpiSintel",
                             dict(with_speed_metric=True, evaluate_matched_unmatched=True)),
    "kitti": (evaluate_flow, "validate_kitti", "KITTI", dict(with_speed_metric=True)),
    "kitti_per_sample": (evaluate_flow, "validate_kitti", "KITTI", dict(with_speed_metric=True, average_over_pixels=False)),
    "stereo_things": (evaluate_stereo, "validate_things", "FlyingThings3D", {}),
    "stereo_kitti15": (evaluate_stereo, "validate_kitti15", "KITTI15", {}),
    "stereo_eth3d": (evaluate_stereo, "validate_eth3d", "ETH3DStereo", {}),
    "stereo_middlebury": (evaluate_stereo, "validate_middlebury", "MiddleburyEval3", dict(padding_factor=32)),
    "depth_scannet": (evaluate_depth, "validate_scannet", "ScannetDataset", {}),
    "depth_demon": (evaluate_depth, "validate_demon", "DemonDataset", dict(eval_min_depth=1.0, eval_max_depth=8.0)),
}


def main():
    out = []
    for name, task, options, build in E.CASES:
        samples = build()
        module, fn, cls, kw = REFERENCE[name]
        setattr(module, cls, lambda *a, _s=samples, **k: list(_s))
        res = {k: float(v) for k, v in getattr(module, fn)(E.STUB, **kw).items()}
        if name.startswith("sintel"):
            res = {k: v for k, v in res.items() if k.startswith("sintel_clean")}
        out.append(dict(name=name, task=task, options=options, digest=E.digest(samples), results=res))
        print("%-22s %d samples  %s" % (name, len(samples), res))
    path = os.path.join(HERE, "golden_eval.pt")
    torch.save(out, path)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
