"""Leaderboard submissions on the device: `um_encode_submission` against the numpy statement (oracle/submission_io.py) bit
for bit, for every format and both geometries; and each driver end to end on small synthetic datasets with a random-init
model, its decoded files against the oracle applied to the model's output on the same batches (the batch composition
changes `um_conv2d_tc`'s summation order, so the comparison runs the model on the driver's batches)."""
import os

import numpy as np
import pytest
import torch

from oracle import submission_io as S
from unimatch_b200 import ops, submission
from unimatch_b200.inference import InputPadder, _resize, disparity_to_image, flow_to_image
from unimatch_b200.synthetic import synthetic_model, workload_call

pytestmark = pytest.mark.gpu
OPS = torch.ops.unimatch_sm100
FORMATS = [ops.SUBMIT_FLO, ops.SUBMIT_KITTI_FLOW_PNG, ops.SUBMIT_KITTI_DISP_PNG, ops.SUBMIT_PFM]
SPECIALS = [np.nan, np.inf, -np.inf, 0.0, -0.0, 512.0, -512.0, 511.99, -512.01, 256.0, -256.01, 1e6, -1e6, 3e38, 1e10,
            70000.7 / 64, -70000.2 / 64, -1.5 / 64, 1.0 / 64 - 1e-3]


def _pred(seed, b, c, h, w):
    g = np.random.default_rng(seed)
    x = (g.standard_normal((b, c, h, w)) * 200).astype(np.float32)
    k = g.integers(-40000, 40000, x.shape)
    near = ((k + g.choice([1e-3, -1e-3, 0.5, 0.4999], x.shape)) / 64).astype(np.float32)
    x = np.where(g.random(x.shape) < 0.3, near, x).astype(np.float32)
    flat = x.reshape(-1)
    idx = g.choice(flat.size, size=min(flat.size, 4 * len(SPECIALS)), replace=False)
    flat[idx] = np.resize(np.array(SPECIALS, np.float32), idx.size)
    return x


def _oracle(pred, fmt, ori, resize, top, left):
    rows = []
    for p in pred:
        vals = S.resize_back(p, ori) if resize else S.crop(p, top, left, *ori)
        rows.append(np.frombuffer(S.payload(vals, fmt), np.uint8))
    return np.stack(rows)


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("b,h,w,ori,resize,top,left", [
    (1, 37, 53, (31, 47), False, 3, 2),        # odd crop, B = 1
    (3, 40, 56, (37, 53), False, 0, 1),        # bottom-only crop (KITTI mode)
    (1, 1, 1, (1, 1), False, 0, 0),
    (2, 40, 56, (37, 53), True, 0, 0),         # resize back, non-dyadic weights
    (3, 24, 40, (75, 121), True, 0, 0),        # resize up by ~3
    (2, 33, 45, (33, 45), True, 0, 0),         # resize at the same size: only the rescale rounds
])
def test_encode_matches_oracle(fmt, b, h, w, ori, resize, top, left):
    c = ops.SUBMIT_CHANNELS[fmt]
    pred = _pred(fmt * 100 + b * 10 + h, b, c, h, w)
    got = OPS.encode_submission(torch.from_numpy(pred).cuda(), fmt, ori[0], ori[1], resize, top, left).cpu().numpy()
    want = _oracle(pred, fmt, ori, resize, top, left)
    assert got.shape == want.shape == (b, ops.submission_payload_bytes(fmt, *ori))
    bad = np.argwhere(got != want)
    assert bad.size == 0, "first differing bytes (sample, offset): %s" % bad[:5].tolist()


def test_encode_rejects_bad_arguments():
    x = torch.zeros((1, 2, 8, 8), device="cuda")
    with pytest.raises(RuntimeError):
        OPS.encode_submission(x, ops.SUBMIT_PFM, 8, 8, False, 0, 0)          # PFM takes one channel
    with pytest.raises(RuntimeError):
        OPS.encode_submission(x, ops.SUBMIT_FLO, 8, 8, False, 1, 0)          # crop outside the prediction


# --------------------------------------------------------------------------------------------------- drivers end to end
def _model_inputs(images, geom, padding_factor, mode):
    """The driver's model inputs for stacked device images, restated: InputPadder or the resize."""
    if geom[0] == "pad":
        return InputPadder(images[0].shape, mode=mode, padding_factor=padding_factor).pad(*images)
    if geom[0] == "resize":
        return [_resize(x, geom[1]) for x in images]
    return images


def _read(path):
    with open(path, "rb") as f:
        return f.read()


@torch.no_grad()
def test_flow_drivers_end_to_end(tmp_path):
    model, kw = synthetic_model("gmflow-scale1"), workload_call("gmflow-scale1", drop=("task",))
    g = torch.Generator().manual_seed(5)
    sizes = [(60, 90), (60, 90), (52, 100), (60, 90)]
    sintel = [(torch.rand((3, h, w), generator=g) * 255, torch.rand((3, h, w), generator=g) * 255, ("seq%d" % (i % 2), i))
              for i, (h, w) in enumerate(sizes)]
    kitti = [(a, b, ("%06d_10.png" % i,)) for i, (a, b, _) in enumerate(sintel)]
    for protocol, data, inference_size in (("sintel", sintel, None), ("kitti", kitti, None), ("sintel", sintel, (48, 80))):
        out = tmp_path / ("%s_%s" % (protocol, inference_size is not None))
        submission.create_flow_submission(model, data, protocol=protocol, output_path=str(out), batch=2, padding_factor=16,
                                          inference_size=inference_size, save_vis_flow=protocol == "sintel", **kw)
        mode = "kitti" if protocol == "kitti" else "sintel"
        for items in submission._batches(data, 2, lambda s: tuple(s[0].shape)):
            ori = tuple(items[0][0].shape[-2:])
            geom = S.geometry("flow", protocol, ori, 16, inference_size)
            imgs = [torch.stack([s[k] for s in items]).cuda() for k in (0, 1)]
            pred = model(*_model_inputs(imgs, geom, 16, mode), task="flow", **kw)["flow_preds"][-1].cpu().numpy()
            for s, p in zip(items, pred):
                flow = S.to_original(p, geom, ori)
                if protocol == "sintel":
                    path = out / "clean" / s[2][0] / ("frame%04d.flo" % (s[2][1] + 1))
                    assert _read(path) == S.flo_header(*ori) + S.payload(flow, S.FLO)
                    pic = flow_to_image(torch.from_numpy(flow)[None].cuda())[0].cpu().numpy()
                    assert np.array_equal(S.decode_png(_read(str(path).replace(".flo", ".png"))), pic)
                else:
                    assert np.array_equal(S.decode_png(_read(out / s[2][0])), S.kitti_flow_pixels(flow))


@torch.no_grad()
def test_stereo_drivers_end_to_end(tmp_path):
    g = torch.Generator().manual_seed(6)
    for workload, protocol, sizes, inference_size, vis in (
            ("gmstereo-scale2", "kitti", [(70, 100), (70, 100), (64, 96)], None, False),
            ("gmstereo-scale2", "kitti", [(70, 100), (64, 96)], (64, 96), False),
            ("gmstereo-scale2", "eth3d", [(70, 100), (64, 96), (70, 100)], None, False),       # resize, then none
            ("gmstereo-scale2", "eth3d", [(70, 100)], None, True),
            ("gmstereo-scale2-regrefine3", "middlebury", [(70, 100), (70, 100), (70, 100)], None, False)):
        model, kw = synthetic_model(workload), workload_call(workload, drop=("task",))
        data = [{"left": torch.randn((3, h, w), generator=g), "right": torch.randn((3, h, w), generator=g),
                 "left_name": "scenes/scene%d/im0.png" % i if protocol != "kitti" else "%06d_10.png" % i}
                for i, (h, w) in enumerate(sizes)]
        out = tmp_path / ("%s_%s_%s" % (protocol, inference_size is not None, vis))
        submission.create_stereo_submission(model, data, protocol=protocol, output_path=str(out), batch=2, padding_factor=32,
                                            inference_size=inference_size, save_vis_disp=vis, **kw)
        fwd = {k: v for k, v in kw.items() if not (protocol == "middlebury" and k == "num_reg_refine")}
        for items in submission._batches(data, 2, lambda s: tuple(s["left"].shape)):
            ori = tuple(items[0]["left"].shape[-2:])
            geom = S.geometry("stereo", protocol, ori, 32, inference_size)
            imgs = [torch.stack([s[k] for s in items]).cuda() for k in ("left", "right")]
            pred = model(*_model_inputs(imgs, geom, 32, "sintel"), task="stereo", **fwd)["flow_preds"][-1]
            for s, p in zip(items, pred.unsqueeze(1).cpu().numpy()):
                disp = S.to_original(p, geom, ori)[0]
                scene = os.path.basename(os.path.dirname(s["left_name"]))
                if protocol == "kitti":
                    assert np.array_equal(S.decode_png(_read(out / s["left_name"])), S.kitti_disp_pixels(disp))
                elif vis:
                    pic = disparity_to_image(torch.from_numpy(disp).cuda()).cpu().numpy()[..., ::-1]
                    assert np.array_equal(S.decode_png(_read(out / (scene + ".png"))), pic)
                else:
                    pfm = out / (scene + ".pfm") if protocol == "eth3d" else out / scene / "disp0GMStereo.pfm"
                    assert _read(pfm) == S.pfm_header(*ori) + S.payload(disp[None], S.PFM)
                    txt = out / (scene + ".txt") if protocol == "eth3d" else out / scene / "timeGMStereo.txt"
                    assert float(_read(txt).decode().split()[-1]) > 0
