"""Leaderboard submissions without a GPU: the numpy statement (oracle/submission_io.py) against the reference's writers
(tests/golden/golden_submission.pt, made by make_golden_submission.py), the stdlib PNG writer read back by a stdlib decoder
and by cv2, and the drivers' file layout, runtime files and writer-error propagation on a stub model, with the device encode
replaced by the oracle."""
import os
import re

import numpy as np
import pytest
import torch

from oracle import submission_io as S
from unimatch_b200 import ops, submission

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = torch.load(os.path.join(HERE, "golden", "golden_submission.pt"))


# ---------------------------------------------------------------------------------------------------- oracle vs reference
def test_cast_rule_examples():
    x = np.array([-1.5, -0.5, 65536, 70000.7, -70000.2, 1e10, np.nan, np.inf, -np.inf, 65535.9, -2147483648.0, 2147483648.0])
    want = [65535, 0, 0, 4464, 61072, 0, 0, 0, 0, 65535, 0, 0]
    assert S.numpy_u16(x).tolist() == want
    assert S.numpy_u16(x.astype(np.float32)).tolist() == want


def test_flo_bytes_match_write_flow():
    for f, b in zip(GOLD["flow"], GOLD["flo_bytes"]):
        f = f.numpy()
        assert S.flo_header(*f.shape[1:]) + S.payload(f, S.FLO) == bytes(b.numpy())


def test_kitti_flow_pixels_match_write_flow_kitti():
    for f, bgr in zip(GOLD["flow"], GOLD["kitti_flow_bgr"]):
        assert np.array_equal(S.kitti_flow_pixels(f.numpy())[..., ::-1].astype(np.int32), bgr.numpy())
    assert any(f.numel() >= 2 * 4096 for f in GOLD["flow"])


def test_kitti_disparity_matches_reference_expression():
    for d, u in zip(GOLD["disp"], GOLD["kitti_disp_u16"]):
        assert np.array_equal(S.kitti_disp_pixels(d.numpy()).astype(np.int32), u.numpy())


def test_pfm_bytes_match_write_pfm():
    for d, b in zip(GOLD["disp"], GOLD["pfm_bytes"]):
        d = d.numpy()
        assert S.pfm_header(*d.shape) + S.payload(d[None], S.PFM) == bytes(b.numpy())
        assert submission.pfm_header(*d.shape) == S.pfm_header(*d.shape)


def test_resize_back_matches_reference():
    differs = 0
    for r in GOLD["resize"]:
        p, ori = r["pred"].numpy(), tuple(r["flow"].shape[-2:])
        assert np.array_equal(S.bilinear_align_corners(p, *ori).view(np.uint32), r["interp"].numpy().view(np.uint32))
        assert np.array_equal(S.resize_back(p, ori).view(np.uint32), r["flow"].numpy().view(np.uint32))
        assert np.array_equal(S.resize_back(p[:1], ori)[0].view(np.uint32), r["disp"].numpy().view(np.uint32))
        ratio = (r["interp"][0].numpy() * np.float32(ori[1] / p.shape[2])).astype(np.float32)
        differs += int((ratio != r["flow"][0].numpy()).sum())
    assert differs > 0, "the maps must tell the two-step rescale from the ratio"


def test_fma32_is_a_single_rounding():
    rng = np.random.default_rng(3)
    a, b, c = (rng.standard_normal(20000).astype(np.float32) for _ in range(3))
    exact = [float(np.float32(float(x) * float(y) + float(z))) for x, y, z in zip(a[:50], b[:50], c[:50])]
    assert np.array_equal(S.fma32(a[:50], b[:50], c[:50]), np.float32(exact))
    # a case where a float64 sum rounds to a float32 tie: double rounding would be wrong
    x, y, z = np.float32(1 + 2 ** -12), np.float32(1 + 2 ** -12), np.float32(-(2 ** -24) * 2 ** -30)
    assert S.fma32(x, y, z) == np.float32(1 + 2 ** -11)


# ------------------------------------------------------------------------------------------------------------- PNG writer
def _png_cases():
    for f, bgr in zip(GOLD["flow"], GOLD["kitti_flow_bgr"]):
        yield S.kitti_flow_pixels(f.numpy()), 2, bgr.numpy()[..., ::-1]
    for d, u in zip(GOLD["disp"], GOLD["kitti_disp_u16"]):
        yield S.kitti_disp_pixels(d.numpy()), 0, u.numpy()


def test_png_writer_round_trips_through_stdlib_decoder(tmp_path):
    for px, ctype, want in _png_cases():
        data = submission.png_bytes(S.png_scanlines(px), px.shape[0], px.shape[1], 16, ctype)
        assert np.array_equal(S.decode_png(data).astype(np.int32), want)
    rgb = np.random.default_rng(0).integers(0, 256, (13, 17, 3), dtype=np.uint8)
    data = submission.png_bytes(submission.picture_scanlines(rgb), 13, 17, 8, 2)
    assert np.array_equal(S.decode_png(data), rgb)


def test_png_writer_round_trips_through_cv2(tmp_path):
    cv2 = pytest.importorskip("cv2")
    for k, (px, ctype, want) in enumerate(_png_cases()):
        path = str(tmp_path / ("%d.png" % k))
        submission._write_png(path, S.png_scanlines(px), px.shape[0], px.shape[1], 16, ctype)
        got = cv2.imread(path, cv2.IMREAD_ANYDEPTH | (cv2.IMREAD_COLOR if ctype == 2 else 0))
        assert np.array_equal(got[..., ::-1] if ctype == 2 else got, want.astype(np.uint16))


# ----------------------------------------------------------------------------------------- drivers on a stub model (CPU)
def _cpu_encode(pred, fmt, ori, enc):
    """The device encode as the oracle states it (the op itself only runs on CUDA)."""
    resize, top, left = enc
    rows = []
    for p in pred.float().numpy():
        vals = S.resize_back(p, ori) if resize else S.crop(p, top, left, *ori)
        rows.append(np.frombuffer(S.payload(vals, fmt), np.uint8))
    return torch.from_numpy(np.stack(rows))


class StubModel:
    """flow = channels 0, 1 of image1 scaled, disparity = channel 0 of left; records every call's keyword arguments."""

    def __init__(self):
        self.calls = []

    def __call__(self, a, b, **kw):
        self.calls.append(dict(kw, batch=a.shape[0], shape=tuple(a.shape[-2:])))
        if kw["task"] == "flow":
            return {"flow_preds": [a[:, :2] * 0.37 - b[:, 1:3] * 2.1]}
        return {"flow_preds": [a[:, 0] * 11.3 + b[:, 2]]}


@pytest.fixture
def cpu_encode(monkeypatch):
    monkeypatch.setattr(submission, "_encode", _cpu_encode)


def _img(g, h, w, scale=255.0):
    return torch.rand((3, h, w), generator=g) * scale


def _files(root):
    return sorted(os.path.relpath(os.path.join(d, f), root) for d, _, fs in os.walk(root) for f in fs)


def _expected(model_out, geom, ori, fmt):
    return S.payload(S.to_original(model_out, geom, ori), fmt)


def test_sintel_layout_and_payloads(tmp_path, cpu_encode):
    g = torch.Generator().manual_seed(0)
    data = [(_img(g, 13, 22), _img(g, 13, 22), ("alley_1", 0)), (_img(g, 16, 24), _img(g, 16, 24), ("alley_1", 1)),
            (_img(g, 13, 22), _img(g, 13, 22), ("market_5", 9))]
    model = StubModel()
    stats = submission.create_flow_submission(model, data, protocol="sintel", output_path=str(tmp_path), dstype="final",
                                              batch=2, device="cpu", writers=3, attn_type="swin")
    assert _files(tmp_path) == ["final/alley_1/frame0001.flo", "final/alley_1/frame0002.flo", "final/market_5/frame0010.flo"]
    assert stats["samples"] == 3 and stats["batches"] == 2
    assert [c["batch"] for c in model.calls] == [2, 1] and all(c["attn_type"] == "swin" for c in model.calls)
    for img1, img2, (seq, frame) in data:
        ori = tuple(img1.shape[-2:])
        geom = S.geometry("flow", "sintel", ori, 8)
        padded = [torch.nn.functional.pad(x[None], (geom[2], geom[3][1] - ori[1] - geom[2], geom[1],
                                                    geom[3][0] - ori[0] - geom[1]), mode="replicate") for x in (img1, img2)]
        out = StubModel()(*padded, task="flow")["flow_preds"][-1][0].numpy()
        data_ = open(tmp_path / "final" / seq / ("frame%04d.flo" % (frame + 1)), "rb").read()
        assert data_ == S.flo_header(*ori) + _expected(out, geom, ori, S.FLO)


def test_kitti_flow_layout_and_payloads(tmp_path, cpu_encode):
    g = torch.Generator().manual_seed(1)
    data = [(_img(g, 11, 20), _img(g, 11, 20), ("%06d_10.png" % i,)) for i in range(3)]
    submission.create_flow_submission(StubModel(), data, protocol="kitti", output_path=str(tmp_path), batch=8, device="cpu")
    assert _files(tmp_path) == ["000000_10.png", "000001_10.png", "000002_10.png"]
    for img1, img2, (name,) in data:
        geom = S.geometry("flow", "kitti", (11, 20), 8)
        assert geom[1] == 0                                     # mode 'kitti': bottom-only padding in height
        padded = [torch.nn.functional.pad(x[None], (geom[2], geom[3][1] - 20 - geom[2], 0, geom[3][0] - 11),
                                          mode="replicate") for x in (img1, img2)]
        out = StubModel()(*padded, task="flow")["flow_preds"][-1][0].numpy()
        got = S.decode_png(open(tmp_path / name, "rb").read())
        assert np.array_equal(got, S.kitti_flow_pixels(S.to_original(out, geom, (11, 20))))


def _stereo_data(g, sizes, names):
    return [{"left": _img(g, h, w, 2.0), "right": _img(g, h, w, 2.0), "left_name": n} for (h, w), n in zip(sizes, names)]


def test_stereo_layouts(tmp_path, cpu_encode):
    g = torch.Generator().manual_seed(2)
    kitti = _stereo_data(g, [(20, 33)] * 2, ["000000_10.png", "000001_10.png"])
    submission.create_stereo_submission(StubModel(), kitti, protocol="kitti", output_path=str(tmp_path / "k"), device="cpu")
    assert _files(tmp_path / "k") == ["000000_10.png", "000001_10.png"]
    for s in kitti:
        geom = S.geometry("stereo", "kitti", (20, 33), 16)
        top, left, (ph, pw) = geom[1], geom[2], geom[3]
        padded = [torch.nn.functional.pad(s[k][None], (left, pw - 33 - left, top, ph - 20 - top), mode="replicate")
                  for k in ("left", "right")]
        out = StubModel()(*padded, task="stereo")["flow_preds"][-1].numpy()
        got = S.decode_png(open(tmp_path / "k" / s["left_name"], "rb").read())
        assert np.array_equal(got, S.kitti_disp_pixels(S.to_original(out, geom, (20, 33))[0]))

    # ETH3D at a size that is already a multiple: no resize, the model sees the pair as it is
    eth = _stereo_data(g, [(32, 48), (32, 48)], ["two_view_test/delivery_area_1l/im0.png", "two_view_test/lakeside_1l/im0.png"])
    model = StubModel()
    submission.create_stereo_submission(model, eth, protocol="eth3d", output_path=str(tmp_path / "e"), batch=2, device="cpu",
                                        padding_factor=16, num_reg_refine=3)
    assert _files(tmp_path / "e") == ["delivery_area_1l.pfm", "delivery_area_1l.txt", "lakeside_1l.pfm", "lakeside_1l.txt"]
    assert len(model.calls) == submission.WARMUP_FORWARDS + 1 and all(c["num_reg_refine"] == 3 for c in model.calls)
    for s in eth:
        scene = os.path.basename(os.path.dirname(s["left_name"]))
        out = StubModel()(s["left"][None], s["right"][None], task="stereo")["flow_preds"][-1].numpy()
        want = S.pfm_header(32, 48) + _expected(out, ("none",), (32, 48), S.PFM)
        assert open(tmp_path / "e" / (scene + ".pfm"), "rb").read() == want
        text = open(tmp_path / "e" / (scene + ".txt")).read()
        assert re.fullmatch(r"runtime \d+\.\d+(e-\d+)?", text) and float(text.split()[1]) >= 0

    # Middlebury: the saved forward goes without num_reg_refine (the model's default), the warm-up forwards pass it
    mid = _stereo_data(g, [(20, 30), (24, 30), (20, 30)], ["MiddEval3/testF/Australia/im0.png", "MiddEval3/testF/Bicycle2/im0.png",
                                                          "MiddEval3/testF/Crusade/im0.png"])
    model = StubModel()
    submission.create_stereo_submission(model, mid, protocol="middlebury", output_path=str(tmp_path / "m"), batch=2,
                                        device="cpu", num_reg_refine=3)
    assert _files(tmp_path / "m") == ["Australia/disp0GMStereo.pfm", "Australia/timeGMStereo.txt", "Bicycle2/disp0GMStereo.pfm",
                                      "Bicycle2/timeGMStereo.txt", "Crusade/disp0GMStereo.pfm", "Crusade/timeGMStereo.txt"]
    warm, timed = model.calls[:submission.WARMUP_FORWARDS], model.calls[submission.WARMUP_FORWARDS:]
    assert all(c["num_reg_refine"] == 3 for c in warm) and all("num_reg_refine" not in c for c in timed)
    assert [c["batch"] for c in timed] == [2, 1]
    for s in mid:
        scene = os.path.basename(os.path.dirname(s["left_name"]))
        text = open(tmp_path / "m" / scene / "timeGMStereo.txt").read()
        assert re.fullmatch(r"\d+\.\d+(e-\d+)?", text)


def test_argument_checks(tmp_path):
    with pytest.raises(ValueError):
        submission.create_flow_submission(StubModel(), [], protocol="chairs", output_path=str(tmp_path), device="cpu")
    with pytest.raises(ValueError):
        submission.create_stereo_submission(StubModel(), [], protocol="kitti", output_path=str(tmp_path), device="cpu",
                                            save_vis_disp=True)
    with pytest.raises(ValueError):
        submission.create_stereo_submission(StubModel(), [], protocol="eth3d", output_path=str(tmp_path), device="cpu",
                                            task="flow")
    with pytest.raises(RuntimeError):
        ops.submission_payload_bytes(7, 2, 2)


def test_writer_errors_reach_the_caller(tmp_path, cpu_encode):
    g = torch.Generator().manual_seed(4)
    data = [(_img(g, 8, 8), _img(g, 8, 8), ("seq", i)) for i in range(5)]
    (tmp_path / "clean").mkdir()
    (tmp_path / "clean" / "seq").write_text("a file where the sequence directory goes")
    with pytest.raises(OSError):
        submission.create_flow_submission(StubModel(), data, protocol="sintel", output_path=str(tmp_path), batch=2,
                                          device="cpu", writers=2)


def test_batches_group_by_size_and_flush_at_the_end():
    items = [(0, "a"), (1, "b"), (2, "a"), (3, "a"), (4, "b"), (5, "c")]
    got = [[i for i, _ in b] for b in submission._batches(items, 2, lambda s: s[1])]
    assert got == [[0, 2], [1, 4], [3], [5]]
