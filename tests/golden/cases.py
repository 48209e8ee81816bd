"""Golden-vector case table shared by `make_golden.py` (runs the REFERENCE, build container only)
and `tests/test_oracle_golden.py` (runs the ORACLE against the stored reference outputs, anywhere).

Every case: seeded inputs (regenerated, never stored) -> reference output (stored in golden.pt).
"""
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import unimatch_oracle as O  # noqa: E402
from unimatch_b200.spec import WORKLOADS  # noqa: E402
from unimatch_b200.synthetic import BENCH_WEIGHTS, synthetic_batch, synthetic_state_dict  # noqa: E402

C = 128


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _feat(g, b, h, w, scale=1.0):
    return torch.randn((b, C, h, w), generator=g) * scale


def _tok(g, b, l, scale=1.0):
    return torch.randn((b, l, C), generator=g) * scale


# ---- op-level cases: name -> (input builder, oracle call) ---------------------------------------
def in_attn2d(seed, b, h, w):
    g = _g(seed)
    return dict(q=_tok(g, b, h * w, 2.0), k=_tok(g, b, h * w, 2.0), v=_tok(g, b, h * w), h=h, w=w)


def in_feats(seed, b, h, w, scale=1.5):
    g = _g(seed)
    return dict(f0=_feat(g, b, h, w, scale), f1=_feat(g, b, h, w, scale))


def in_feats_flow(seed, b, h, w, fc=2, mag=3.0):
    g = _g(seed)
    d = dict(f0=_feat(g, b, h, w, 1.5), f1=_feat(g, b, h, w, 1.5))
    d["flow"] = torch.randn((b, fc, h, w), generator=g) * mag
    return d


def in_depth(seed, b, h, w, d=16):
    g = _g(seed)
    x = dict(f0=_feat(g, b, h, w), f1=_feat(g, b, h, w))
    K = torch.tensor([[0.9 * w, 0.0, w / 2.0], [0.0, 0.9 * w, h / 2.0], [0.0, 0.0, 1.0]]).view(1, 3, 3).repeat(b, 1, 1)
    pose = torch.eye(4).view(1, 4, 4).repeat(b, 1, 1)
    pose[:, 0, 3] = 0.1
    pose[:, 2, 3] = 0.02
    x["K"], x["pose"] = K, pose
    x["cand"] = torch.linspace(0.1, 2.0, d).view(1, d, 1, 1).repeat(b, 1, h, w)
    return x


def in_update(seed, b, h, w, fd=2):
    g = _g(seed)
    return dict(net=torch.tanh(torch.randn((b, 128, h, w), generator=g)),
                inp=torch.relu(torch.randn((b, 128, h, w), generator=g)),
                corr=torch.randn((b, 81, h, w), generator=g) * 4,
                flow=torch.randn((b, fd, h, w), generator=g) * 2)


SD_FLOW_RR = dict(num_scales=2, upsample_factor=4, reg_refine=True, task="flow")
SD_DEPTH_RR = dict(num_scales=1, upsample_factor=8, reg_refine=True, task="depth")

OP_CASES = {
    # attention.py
    "attn_full": (lambda: in_attn2d(1, 2, 6, 8),
                  lambda x, sd: O.attn_full(x["q"], x["k"], x["v"])),
    "attn_full_1d": (lambda: in_attn2d(2, 2, 6, 8),
                     lambda x, sd: O.attn_full_1d(x["q"], x["k"], x["v"], x["h"], x["w"])),
    "attn_window_2d": (lambda: in_attn2d(3, 2, 12, 16),
                       lambda x, sd: O.attn_window_2d(x["q"], x["k"], x["v"], 2, False, x["h"], x["w"], None)),
    "attn_window_2d_shift": (lambda: in_attn2d(4, 2, 12, 16),
                             lambda x, sd: O.attn_window_2d(
                                 x["q"], x["k"], x["v"], 2, True, x["h"], x["w"],
                                 O.shift_mask_2d(x["h"], x["w"], x["h"] // 2, x["w"] // 2, x["h"] // 4, x["w"] // 4, "cpu"))),
    "attn_window_2d_shift_k4": (lambda: in_attn2d(5, 1, 16, 24),
                                lambda x, sd: O.attn_window_2d(
                                    x["q"], x["k"], x["v"], 4, True, x["h"], x["w"],
                                    O.shift_mask_2d(x["h"], x["w"], 4, 6, 2, 3, "cpu"))),
    "attn_window_1d_shift": (lambda: in_attn2d(6, 2, 5, 24),
                             lambda x, sd: O.attn_window_1d(
                                 x["q"], x["k"], x["v"], 4, True, x["h"], x["w"], O.shift_mask_1d(24, 6, 3, "cpu"))),
    "attn_window_1d": (lambda: in_attn2d(7, 2, 5, 24),
                       lambda x, sd: O.attn_window_1d(x["q"], x["k"], x["v"], 4, False, x["h"], x["w"], None)),
    # utils.py / position.py
    "add_position_k2": (lambda: in_feats(8, 2, 8, 12),
                        lambda x, sd: torch.stack(O.add_position(x["f0"], x["f1"], 2))),
    "add_position_k1": (lambda: in_feats(9, 1, 6, 10),
                        lambda x, sd: torch.stack(O.add_position(x["f0"], x["f1"], 1))),
    # transformer.py
    "transformer_swin_k2": (lambda: in_feats(10, 1, 8, 12, 1.0),
                            lambda x, sd: torch.stack(O.feature_transformer(sd, x["f0"], x["f1"], "swin", 2))),
    "transformer_swin_k1": (lambda: in_feats(11, 1, 6, 8, 1.0),
                            lambda x, sd: torch.stack(O.feature_transformer(sd, x["f0"], x["f1"], "swin", 1))),
    "transformer_stereo_k2": (lambda: in_feats(12, 1, 8, 12, 1.0),
                              lambda x, sd: torch.stack(O.feature_transformer(
                                  sd, x["f0"], x["f1"], "self_swin2d_cross_swin1d", 2))),
    "transformer_stereo_k1": (lambda: in_feats(13, 1, 6, 8, 1.0),
                              lambda x, sd: torch.stack(O.feature_transformer(
                                  sd, x["f0"], x["f1"], "self_swin2d_cross_1d", 1))),
    # matching.py
    "global_corr": (lambda: in_feats(14, 2, 7, 9),
                    lambda x, sd: O.global_corr_flow(x["f0"], x["f1"], False)),
    "global_corr_bidir": (lambda: in_feats(15, 1, 7, 9),
                          lambda x, sd: O.global_corr_flow(x["f0"], x["f1"], True)),
    "local_corr_r4": (lambda: in_feats(16, 2, 11, 13),
                      lambda x, sd: O.local_corr_flow(x["f0"], x["f1"], 4)),
    "local_corr_volume": (lambda: in_feats_flow(17, 2, 11, 13),
                          lambda x, sd: O.local_corr_volume(x["f0"], x["f1"], x["flow"], 4)),
    "global_corr_stereo": (lambda: in_feats(18, 2, 5, 14),
                           lambda x, sd: O.global_corr_disp(x["f0"], x["f1"])),
    "local_corr_stereo_r4": (lambda: in_feats(19, 2, 5, 14),
                             lambda x, sd: O.local_corr_disp(x["f0"], x["f1"], 4)),
    "depth_corr": (lambda: in_depth(20, 2, 8, 10),
                   lambda x, sd: O.depth_corr(x["f0"], x["f1"], x["K"], x["pose"], x["cand"])),
    "depth_corr_bidir_argmax": (lambda: in_depth(21, 1, 8, 10),
                                lambda x, sd: O.depth_corr(x["f0"], x["f1"], x["K"], x["pose"], x["cand"], True, True)),
    # geometry.py
    "flow_warp": (lambda: in_feats_flow(22, 2, 9, 12, mag=4.0),
                  lambda x, sd: O.warp_by_flow(x["f1"], x["flow"])),
    "rigid_flow": (lambda: in_depth(23, 2, 8, 10),
                   lambda x, sd: O.rigid_flow_from_depth(1.0 / x["cand"][:, 3], x["K"], x["pose"])),
    # attention.py SelfAttnPropagation
    "prop_global": (lambda: in_feats_flow(24, 2, 7, 9),
                    lambda x, sd: O.propagate_global(sd, x["f0"], x["flow"])),
    "prop_local_r1": (lambda: in_feats_flow(25, 2, 7, 9),
                      lambda x, sd: O.propagate_local(sd, x["f0"], x["flow"], 1)),
    "prop_local_r1_disp": (lambda: in_feats_flow(26, 2, 7, 9, fc=1),
                           lambda x, sd: O.propagate_local(sd, x["f0"], x["flow"], 1)),
    # utils.py convex upsampling
    "convex_upsample": (lambda: dict(flow=torch.randn((2, 2, 6, 7), generator=_g(27)),
                                     mask=torch.randn((2, 144, 6, 7), generator=_g(28)) * 3),
                        lambda x, sd: O.convex_upsample(x["flow"], x["mask"], 4)),
    # reg_refine.py
    "update_block_flow": (lambda: in_update(29, 1, 8, 10, 2),
                          lambda x, sd: torch.cat([t for t in O.update_block(sd, x["net"], x["inp"], x["corr"], x["flow"])
                                                   if t is not None], dim=1)),
    # backbone.py
    "backbone_s2": (lambda: dict(img=torch.randn((2, 3, 32, 48), generator=_g(30))),
                    lambda x, sd: torch.cat([t.flatten(1) for t in O.backbone(sd, x["img"], 2)], dim=1)),
}

OP_CASE_WEIGHTS = {name: SD_FLOW_RR for name in OP_CASES}


# ---- end-to-end cases -------------------------------------------------------------------------------
# (workload, batch, H, W, extra forward kwargs)
E2E_CASES = {
    "e2e_gmflow_s1_256x320": ("gmflow-scale1", 1, 256, 320, {}),                  # BASELINE configs[0]
    "e2e_gmflow_s1_bidir": ("gmflow-scale1", 1, 64, 96, dict(pred_bidir_flow=True)),
    "e2e_gmflow_s2": ("gmflow-scale2", 1, 128, 192, {}),
    "e2e_gmflow_s2_rr6": ("gmflow-scale2-regrefine6", 2, 128, 192, {}),
    "e2e_gmflow_s2_rr6_bidir": ("gmflow-scale2-regrefine6", 1, 64, 128, dict(pred_bidir_flow=True)),
    "e2e_gmstereo_s2": ("gmstereo-scale2", 1, 128, 192, {}),
    "e2e_gmstereo_s2_rr3": ("gmstereo-scale2-regrefine3", 1, 128, 192, {}),
    "e2e_gmdepth_s1": ("gmdepth-scale1", 1, 128, 192, {}),
    "e2e_gmdepth_s1_rr1": ("gmdepth-scale1-regrefine1", 2, 128, 192, {}),
    "e2e_gmdepth_s1_rr1_bidir": ("gmdepth-scale1-regrefine1", 1, 96, 128, dict(pred_bidir_depth=True)),
}

E2E_DAMP = 0.5   # transformer matrices x0.5: keeps the random-init network out of its chaotic regime


def e2e_setup(name):
    wl, b, h, w, extra = E2E_CASES[name]
    cfg = WORKLOADS[wl]
    sd = synthetic_state_dict(seed=326, damp=E2E_DAMP, **cfg["model"])
    batch = synthetic_batch(cfg["model"]["task"], b, h, w)
    call = dict(cfg["call"])
    call.update(extra)
    return cfg, sd, batch, call


def e2e_oracle(name, taps=None):
    cfg, sd, batch, call = e2e_setup(name)
    mk = {k: cfg["model"][k] for k in ("num_scales", "upsample_factor", "reg_refine")}
    return O.forward(sd, batch["img0"], batch["img1"], intrinsics=batch.get("intrinsics"), pose=batch.get("pose"),
                     taps=taps, **mk, **call)["flow_preds"][-1]


# ---- end-to-end tolerances ---------------------------------------------------------------------------
# Measured self-noise of the REFERENCE algorithm (oracle == reference bit-for-bit): mean end-point
# error (flow) / mean |diff| (disparity, depth) between a 1-thread and an 8-thread CPU run of the same
# fp32 code on the same inputs and weights (damp 0.5, refine_gain 0.02).  It is the floor below which
# two correct fp32 implementations cannot be told apart.
E2E_NOISE = {
    "e2e_gmflow_s1_256x320": 3.1e-4,
    "e2e_gmflow_s1_bidir": 1.7e-4,
    "e2e_gmflow_s2": 6.2e-3,
    "e2e_gmflow_s2_rr6": 3.7e-2,
    "e2e_gmflow_s2_rr6_bidir": 6.9e-3,
    "e2e_gmstereo_s2": 6.3e-4,
    "e2e_gmstereo_s2_rr3": 3.4e-3,
    "e2e_gmdepth_s1": 1e-6,
    "e2e_gmdepth_s1_rr1": 1e-6,
    "e2e_gmdepth_s1_rr1_bidir": 1e-6,
}
E2E_NOISE_FACTOR = 8.0    # stated tolerance: mean error <= 8 x self-noise (+ 1e-4 absolute)


def e2e_tolerance(name):
    return E2E_NOISE_FACTOR * E2E_NOISE[name] + 1e-4


def distinct_cameras(B, h, w, seed=5):
    """Per-pair cameras for images of h x w: intrinsics [B,3,3] whose focal length, aspect ratio and principal point all
    differ between pairs, and relative poses [B,4,4] with a rotation about all three axes (up to 3 degrees each) and a
    translation, different for every pair."""
    g = _g(seed)
    K, pose = torch.zeros((B, 3, 3)), torch.eye(4).repeat(B, 1, 1)
    for b in range(B):
        r = torch.rand(4, generator=g)
        fx = w * (0.7 + 0.5 * r[0].item())
        K[b] = torch.tensor([[fx, 0.0, w * (0.4 + 0.2 * r[2].item())],
                             [0.0, fx * (0.85 + 0.3 * r[1].item()), h * (0.4 + 0.2 * r[3].item())], [0.0, 0.0, 1.0]])
        ax, ay, az = ((torch.rand(3, generator=g) * 2 - 1) * 0.05).tolist()
        rx = torch.tensor([[1.0, 0, 0], [0, math.cos(ax), -math.sin(ax)], [0, math.sin(ax), math.cos(ax)]])
        ry = torch.tensor([[math.cos(ay), 0, math.sin(ay)], [0, 1.0, 0], [-math.sin(ay), 0, math.cos(ay)]])
        rz = torch.tensor([[math.cos(az), -math.sin(az), 0], [math.sin(az), math.cos(az), 0], [0, 0, 1.0]])
        pose[b, :3, :3] = rz @ ry @ rx
        pose[b, :3, 3] = torch.tensor([0.05 + 0.1 * b / max(B - 1, 1), 0.0, 0.0]) + (torch.rand(3, generator=g) * 2 - 1) * 0.03
    return K, pose


# ---- batch 3 cases: distinct pairs, bidirectional modes and per-pair cameras ------------------------------------------
# (workload, H, W, extra forward kwargs); the depth cases get the cameras of `distinct_cameras`
BATCH3_CASES = {
    "b3_gmflow_s1_bidir": ("gmflow-scale1", 64, 96, dict(pred_bidir_flow=True)),
    "b3_gmflow_s2_rr6_bidir": ("gmflow-scale2-regrefine6", 64, 128, dict(pred_bidir_flow=True)),
    "b3_gmstereo_s2": ("gmstereo-scale2", 128, 192, {}),
    "b3_gmstereo_s2_rr3": ("gmstereo-scale2-regrefine3", 128, 192, {}),
    "b3_gmdepth_s1": ("gmdepth-scale1", 128, 192, {}),
    "b3_gmdepth_s1_rr1": ("gmdepth-scale1-regrefine1", 128, 192, {}),
    "b3_gmdepth_s1_bidir": ("gmdepth-scale1", 96, 128, dict(pred_bidir_depth=True)),
    "b3_gmdepth_s1_rr1_bidir": ("gmdepth-scale1-regrefine1", 96, 128, dict(pred_bidir_depth=True)),
    "b3_gmdepth_s1_argmax": ("gmdepth-scale1", 96, 128, dict(depth_from_argmax=True)),
}

# Self-noise of the reference on these batches (tools/self_noise.py's `threads` probe: 1 against 8 CPU threads), largest
# per-pair mean error; the tolerance of a pair is E2E_NOISE_FACTOR x this + 1e-4, as for E2E_CASES.
BATCH3_NOISE = {
    "b3_gmflow_s1_bidir": 9.7e-5,
    "b3_gmflow_s2_rr6_bidir": 1.5e-2,
    "b3_gmstereo_s2": 4.9e-4,
    "b3_gmstereo_s2_rr3": 2.5e-3,
    "b3_gmdepth_s1": 3.4e-6,
    "b3_gmdepth_s1_rr1": 2.6e-6,
    "b3_gmdepth_s1_bidir": 3.8e-6,
    "b3_gmdepth_s1_rr1_bidir": 3.3e-6,
    "b3_gmdepth_s1_argmax": 5.8e-6,
}


def batch3_setup(name, h=None, w=None):
    """(cfg, state_dict, batch of 3 distinct pairs, call kwargs) of a BATCH3_CASES entry, optionally at another size."""
    wl, h0, w0, extra = BATCH3_CASES[name]
    h, w = h or h0, w or w0
    cfg = WORKLOADS[wl]
    sd = synthetic_state_dict(seed=326, damp=E2E_DAMP, **cfg["model"])
    batch = synthetic_batch(cfg["model"]["task"], 3, h, w, first_index=7)
    if cfg["model"]["task"] == "depth":
        batch["intrinsics"], batch["pose"] = distinct_cameras(3, h, w)
    call = dict(cfg["call"])
    call.update(extra)
    return cfg, sd, batch, call


def oracle_forward(cfg, sd, batch, call):
    mk = {k: cfg["model"][k] for k in ("num_scales", "upsample_factor", "reg_refine")}
    return O.forward(sd, batch["img0"], batch["img1"], intrinsics=batch.get("intrinsics"), pose=batch.get("pose"),
                     **mk, **call)["flow_preds"][-1]


def epe(a, b):
    d = (a - b).norm(dim=1) if a.dim() == 4 else (a - b).abs()
    return d.mean().item(), d.max().item()


# ---- post-processing around the path (SURVEY.md section 8f rows 3-4) ------------------------------------
def fb_inputs(seed=77, b=2, h=37, w=53):
    """A forward / backward flow pair that is mostly consistent (bwd ~ -fwd warped) with an inconsistent blob and flows
    that leave the image, so that both outcomes of the occlusion test and the zero-padding branch occur."""
    gen = torch.Generator().manual_seed(seed)
    base = torch.randn((b, 2, 3, 4), generator=gen) * 1.5 + 2.0
    fwd = torch.nn.functional.interpolate(base, size=(h, w), mode="bilinear", align_corners=True)
    bwd = -fwd + 0.25 * torch.randn((b, 2, h, w), generator=gen)
    bwd[:, :, 10:18, 20:33] += 3.0                       # an "occluded" region
    return fwd.contiguous(), bwd.contiguous()


PADDER_CASES = [((1, 3, 436, 1024), "sintel", 32), ((1, 3, 375, 1242), "kitti", 16), ((2, 3, 480, 832), "sintel", 32),
                ((1, 3, 37, 53), "sintel", 8), ((1, 3, 100, 64), "kitti", 32)]


# ---- BASELINE.json configs at their real H x W (one pair each), well-conditioned weight set ---------------------------
# name -> (workload, H, W, mean tolerance, max tolerance, measured self-noise of the reference (mean, max)).
# Self-noise = tools/self_noise.py --bench-set (inputs scaled by 1 + 1e-7); units: px (flow, disparity) / depth units.
# Stated tolerance: mean error <= 1e-2 px (flow), 2e-2 px (disparities of up to several hundred px), 1e-4 (depth ~ 1).
FULL_CASES = {
    "full_gmflow_s1_480x832": ("gmflow-scale1", 480, 832, 1e-2, 1e-1, (7.9e-6, 3.6e-5)),                 # configs[1]
    "full_gmstereo_s2_544x960": ("gmstereo-scale2", 544, 960, 2e-2, 2e-1, (2.0e-5, 1.8e-4)),             # configs[2]
    "full_gmflow_s2_rr6_480x832": ("gmflow-scale2-regrefine6", 480, 832, 1e-2, 1e-1, (2.0e-5, 1.3e-4)),  # configs[3]
    "full_gmdepth_s1_rr1_384x512": ("gmdepth-scale1-regrefine1", 384, 512, 1e-4, 1e-3, (1.0e-7, 8.3e-7)),  # configs[4]
    # token rows not a multiple of 16 (2 x 46 x 62 = 5704) on the tensor-core attention path: the GEMM row padding
    "odd_gmflow_s1_368x496": ("gmflow-scale1", 368, 496, 1e-2, 1e-1, None),
    "odd_gmflow_s1_48x80": ("gmflow-scale1", 48, 80, 1e-2, 1e-1, None),
}


def full_setup(name, batch=1):
    wl, h, w = FULL_CASES[name][:3]
    cfg = WORKLOADS[wl]
    sd = synthetic_state_dict(seed=326, **BENCH_WEIGHTS, **cfg["model"])
    data = synthetic_batch(cfg["model"]["task"], batch, h, w)
    return cfg, sd, data, dict(cfg["call"])


def full_oracle(name, batch=1):
    cfg, sd, data, call = full_setup(name, batch)
    mk = {k: cfg["model"][k] for k in ("num_scales", "upsample_factor", "reg_refine")}
    return O.forward(sd, data["img0"], data["img1"], intrinsics=data.get("intrinsics"), pose=data.get("pose"),
                     **mk, **call)["flow_preds"][-1]
