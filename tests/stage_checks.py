"""Teacher-forced stage parity of `unimatch_b200.UniMatch` against the oracle (== reference, tests/golden), for every workload
of `spec.WORKLOADS` and both bidirectional modes.

The oracle's forward records its intermediate tensors (`taps`: encoder features, warped / transformed features, the estimate
after correlation and after propagation, after every refinement iteration, the upsampling mask).  Each stage of the module
(`UniMatch._stage_*`, with the glue of `UniMatch._forward_encoded` around it) is then run ON THE ORACLE'S INPUTS for that stage
and compared with the oracle's output for it, so an error cannot hide behind -- or be blamed on -- the amplification of earlier
stages (unimatch/unimatch.py:136-354).  The harness calls the ops through `unimatch_b200.unimatch._OPS`, the table the module
calls, so a test that wraps that table reaches the harness's own launches too.

Used at the bench resolutions on the GPU (tests/test_stages_gpu.py, the CUDA kernels) and at small shapes on the CPU
(tests/test_stages_cpu.py, oracle-backed kernels of tests/refops*.py: checks this harness and the host orchestration).

Tolerances (stated per stage, asserted; every report line prints the error, the tolerance and their ratio, the headroom):
  * feature stages : max |diff| <= FEAT_TOL (encoder, warp) or TRANSFORMER_TOL x max |ref|
  * estimates      : mean and max error at the stage's own resolution, in the estimate's own unit -- flow: end-point error in
                     px (FLOW_*); disparity: |diff| in px (DISP_*); inverse depth: |diff|, the tolerance a fraction of
                     max_depth - min_depth (DEPTH_*)
  * rigid flow     : end-point error in px of the refinement's flow from depth and pose (RIGID_*)
  * upsampling     : the learned upsampler at the input resolution (UPSAMPLE_*, per task, same units); the convex upsampling
                     of the refinement workloads at the estimate's tolerance x the upsampling factor
  * end to end     : the tolerance bench.py's BENCH_WORKLOADS states for the workload, or else for its task
"""
import time

import torch

import unimatch_b200.unimatch as um
from bench import BENCH_WORKLOADS
from oracle import unimatch_oracle as O
from unimatch_b200 import UniMatch
from unimatch_b200.spec import WORKLOADS
from unimatch_b200.synthetic import BENCH_WEIGHTS, synthetic_batch, synthetic_state_dict, workload_call

FEAT_TOL = 3e-5          # encoder, warp: one pass of fp32-faithful arithmetic
TRANSFORMER_TOL = 1e-4   # six blocks (24 GEMMs, 12 attention calls, 18 LayerNorms) in sequence
FLOW_MEAN, FLOW_MAX = 2e-4, 5e-3     # px, per stage, teacher-forced
E2E_MEAN, E2E_MAX = 1e-2, 1e-1       # px at full resolution, free-running end to end (= bench.py's tolerance)
# Stereo and depth stages, the refinement's rigid flow and the learned upsampler.  "measured": the largest error of any
# stage the constant covers over the bench-resolution cases of tests/test_stages_gpu.py, one run on an H100 80GB HBM3 (SXM),
# mean / max, and the stage it came from.  Each tolerance leaves at least 5x headroom and is tighter than the flow constant.
DISP_MEAN, DISP_MAX = 5e-5, 5e-4     # px |disparity error|; measured 9.5e-6 / 8.0e-5 px (s1.correlation, 544x960)
DEPTH_MEAN, DEPTH_MAX = 2e-6, 5e-6   # |inverse depth error| / (max_depth - min_depth); measured 2.6e-7 / 8.8e-7 (refine0)
RIGID_MEAN, RIGID_MAX = 1e-5, 1e-4   # px EPE of `_rigid_flow` against the oracle's on the same inverse depth; measured 0 / 0
UPSAMPLE_FLOW = (2e-5, 1e-4)         # px EPE at the input resolution; measured 2.3e-6 / 1.6e-5 (gmflow-scale2)
UPSAMPLE_DISP = (1e-4, 1e-3)         # px |disparity error| at the input resolution; measured 1.5e-5 / 1.1e-4
UPSAMPLE_DEPTH = (3e-7, 2e-6)        # |inverse depth error| / (max_depth - min_depth) at the input resolution;
                                     # measured 3.6e-8 / 2.5e-7

UNIT = {"flow": "px EPE", "stereo": "px |disp|", "depth": "|inv depth|"}

# (workload, bidirectional): every workload, and the bidirectional modes of flow (pred_bidir_flow) and depth (pred_bidir_depth)
CASES = [(wl, False) for wl in WORKLOADS] + [("gmflow-scale2-regrefine6", True), ("gmdepth-scale1-regrefine1", True)]
BENCH_HW = {"flow": (480, 832), "stereo": (544, 960), "depth": (384, 512)}     # bench.py's resolution of each task


def estimate_tol(task):
    """(mean, max) per-stage tolerance of the task's estimate, as a fraction of the depth range for depth."""
    return {"flow": (FLOW_MEAN, FLOW_MAX), "stereo": (DISP_MEAN, DISP_MAX), "depth": (DEPTH_MEAN, DEPTH_MAX)}[task]


def upsample_tol(task):
    return {"flow": UPSAMPLE_FLOW, "stereo": UPSAMPLE_DISP, "depth": UPSAMPLE_DEPTH}[task]


def e2e_tol(workload):
    """(mean, max, unit) bench.py states for `workload`, or for the first bench workload of the same task."""
    task = WORKLOADS[workload]["model"]["task"]
    rows = [(wl, tol) for wl, *_, tol in BENCH_WORKLOADS.values()]
    return ([tol for wl, tol in rows if wl == workload] or [tol for wl, tol in rows if WORKLOADS[wl]["model"]["task"] == task])[0]


def cl(t, dev):
    """oracle NCHW -> channel-last on `dev`, with the strides of a contiguous tensor: `contiguous()` may leave a 1-channel
    map's channel stride at h * w, and the ops require a channel stride of 1"""
    return t.to(dev).permute(0, 2, 3, 1).clone(memory_format=torch.contiguous_format)


def feat_err(got, ref_nchw):
    ref = ref_nchw.permute(0, 2, 3, 1)
    got = got.detach().float().cpu().reshape(ref.shape)
    return (got - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30)


def flow_err(got_cl, ref_nchw):
    """(mean, max) over pixels of the channel norm of the difference: EPE of a flow, |diff| of a disparity or depth."""
    ref = ref_nchw.permute(0, 2, 3, 1)
    d = (got_cl.detach().float().cpu().reshape(ref.shape) - ref).norm(dim=-1)
    return d.mean().item(), d.max().item()


def run(dev, workload="gmflow-scale2-regrefine6", H=480, W=832, bidir=False, weights=None, report=print, res=None):
    """Returns {stage: headroom}, headroom = error / tolerance (the larger of mean and max for estimates); raises an
    AssertionError whose message starts with the first stage outside its tolerance.  `bidir` sets pred_bidir_flow (flow) or
    pred_bidir_depth (depth).  `res`, if given, is the dict filled stage by stage, so a caller that catches the AssertionError
    still sees the stages checked before it."""
    cfg = WORKLOADS[workload]
    task = cfg["model"]["task"]
    call = workload_call(workload)
    if bidir:
        assert task in ("flow", "depth"), "the stereo task has no bidirectional mode here"
        call["pred_bidir_flow" if task == "flow" else "pred_bidir_depth"] = True
    sd = synthetic_state_dict(seed=326, **(weights or BENCH_WEIGHTS), **cfg["model"])
    batch = synthetic_batch(task, 1, H, W)
    intr, pose = batch.get("intrinsics"), batch.get("pose")
    taps = {}
    mk = {k: cfg["model"][k] for k in ("num_scales", "upsample_factor", "reg_refine")}
    t_oracle = time.perf_counter()
    ref_out = O.forward(sd, batch["img0"], batch["img1"], intrinsics=intr, pose=pose, taps=taps, **mk, **call)["flow_preds"][-1]
    t_oracle = time.perf_counter() - t_oracle

    m = UniMatch(**cfg["model"]).eval()
    m.load_state_dict(sd, strict=True)
    m = m.to(dev)
    ops = um._OPS
    res = {} if res is None else res
    unit = UNIT[task]
    scale = call["max_depth"] - call["min_depth"] if task == "depth" else 1.0     # depth tolerances: fractions of the range
    est_tol = tuple(t * scale for t in estimate_tol(task))
    report("%s %dx%d%s: oracle forward %.1f s on the CPU" % (workload, H, W, " bidirectional" if bidir else "", t_oracle))

    def check_feat(name, got, ref, tol):
        e = feat_err(got, ref)
        res[name] = e / tol
        report("%-22s rel max err %.3e (tol %.1e)  headroom %.3f" % (name, e, tol, e / tol))
        assert e <= tol, "%s: rel max err %.3e > %.1e" % (name, e, tol)

    def check_est(name, err, tol, what=unit):
        (mean, mx), (mean_tol, max_tol) = err, tol
        res[name] = max(mean / mean_tol, mx / max_tol)
        report("%-22s %s mean %.3e max %.3e (tol %.1e / %.1e)  headroom %.3f"
               % (name, what, mean, mx, mean_tol, max_tol, res[name]))
        assert mean <= mean_tol and mx <= max_tol, "%s: %s mean %.3e max %.3e (tol %.1e / %.1e)" % (
            name, what, mean, mx, mean_tol, max_tol)

    def full_err(got_nchw, ref_nchw):
        d = (got_nchw.detach().float().cpu() - ref_nchw.reshape(got_nchw.shape)).norm(dim=1)
        return d.mean().item(), d.max().item()

    with torch.no_grad():
        P = m._prepared()
        img0, img1 = batch["img0"].to(dev), batch["img1"].to(dev)
        cams = None
        if task == "depth":
            cams = m.depth_cameras(intr.to(dev), pose.to(dev), m.upsample_factor, call["min_depth"], call["max_depth"],
                                   call["num_depth_candidates"], bidir)
        # ---- encoder (backbone.py:104-133, trident_conv.py:64-70); stereo and depth images come normalised
        feats = m._stage_backbone(P, img0, img1, task == "flow")
        for s, f in enumerate(feats):
            check_feat("s%d.encoder.view0" % s, f[:1], taps["s%d.f0_ori" % s][:1], FEAT_TOL)
            check_feat("s%d.encoder.view1" % s, f[1:], taps["s%d.f1_ori" % s][:1], FEAT_TOL)
        for s in range(mk["num_scales"]):
            f0_ori, f1_ori = cl(taps["s%d.f0_ori" % s], dev), cl(taps["s%d.f1_ori" % s], dev)
            Bp, h, wd, c = f0_ori.shape                    # 2 streams at scale > 0 with pred_bidir_flow
            splits, prop_r = call["attn_splits_list"][s], call["prop_radius_list"][s]
            radius = None if task == "depth" else call["corr_radius_list"][s]
            flow_up = None
            if s > 0:
                # ---- x2 upsampling + warp (unimatch.py:154-168, geometry.py:65-72); a disparity warps as (-d, 0) in-kernel
                flow_up = ops.upsample2x(cl(taps["s%d.flow_prop" % (s - 1)], dev), 2.0)
                warped = ops.flow_warp(f1_ori, flow_up, h, wd)
                check_feat("s%d.warp" % s, warped, taps["s%d.f1_in" % s], FEAT_TOL)
            # ---- position + transformer (utils.py:111-131, transformer.py:226-294) on the oracle's inputs
            tok = m._stage_features(cl(taps["s%d.f0_in" % s], dev), cl(taps["s%d.f1_in" % s], dev), None, h, wd, splits)
            tok_out, _ = m._stage_transformer(P, tok, h, wd, call["attn_type"], splits, "s%d" % s)
            check_feat("s%d.transformer.view0" % s, tok_out[:Bp], taps["s%d.f0_tr" % s], TRANSFORMER_TOL)
            check_feat("s%d.transformer.view1" % s, tok_out[Bp:], taps["s%d.f1_tr" % s], TRANSFORMER_TOL)
            # ---- correlation + softmax (matching.py:7-282) on the oracle's transformer outputs, then the glue of
            # _forward_encoded: + the upsampled estimate, clamp(min=0) of a disparity
            tok_ref = torch.cat((cl(taps["s%d.f0_tr" % s], dev), cl(taps["s%d.f1_tr" % s], dev)), 0).view(2 * Bp, h * wd, c)
            dargs = (cams, False, bidir) if task == "depth" else None
            pred = m._stage_correlation(tok_ref, Bp, h, wd, task, radius, call.get("pred_bidir_flow", False), dargs)
            flow = pred if flow_up is None else flow_up + pred
            if task == "stereo":
                flow = flow.clamp(min=0)
            check_est("s%d.correlation" % s, flow_err(flow, taps["s%d.flow_corr" % s]), est_tol)
            # ---- propagation (attention.py:184-253) on the oracle's features and estimate; both views' streams when
            # bidirectional at scale 0 (cat(feature0, feature1), unimatch.py:230-237)
            nb = 2 * Bp if bidir and s == 0 else Bp
            rows = 2 * Bp * h * wd
            x_s = torch.zeros((2, (rows + 15) // 16 * 16, c), device=dev, dtype=torch.float16)
            ops.split_planes(tok_ref.view(rows, c), x_s, 0)
            flow = m._stage_propagation(P, x_s, cl(taps["s%d.flow_corr" % s], dev), nb, h, wd, prop_r)
            check_est("s%d.propagation" % s, flow_err(flow, taps["s%d.flow_prop" % s]), est_tol)
        s = mk["num_scales"] - 1
        feat0 = tok_ref[:nb].reshape(nb, h, wd, c)
        final = "s%d.flow_prop" % s
        F = mk["upsample_factor"]
        if mk["reg_refine"]:
            # ---- refinement iterations (unimatch.py:272-354, reg_refine.py:106-119), each from the oracle's previous estimate
            g0, g1 = f0_ori, f1_ori
            drefine = None
            if task == "depth":
                if bidir:
                    g0, g1 = torch.cat((g0, g1), 0), torch.cat((g1, g0), 0)
                drefine = (cams, call["min_depth"], call["max_depth"])
                Ks = intr.clone()                                    # the oracle's cameras, built as the oracle builds them
                Ks[:, :2] = Ks[:, :2] / F
                Ks, pose_ref = (Ks.repeat(2, 1, 1), torch.cat((pose, torch.inverse(pose)), 0)) if bidir else (Ks, pose)
            rst = m._stage_refine_setup(P, feat0.contiguous(), nb, h, wd)
            n_it = call["num_reg_refine"]
            mask = None
            for it in range(n_it):
                fin = taps[final] if it == 0 else taps["refine%d.flow" % (it - 1)]
                if task == "depth":
                    # ---- flow from inverse depth and pose (geometry.py:99-195), the refinement's correlation offsets
                    rigid = m._rigid_flow(cl(fin, dev), cams["K"], cams["K_inv"], cams["pose"], h, wd)
                    check_est("rigid_flow%d" % it, flow_err(rigid, O.rigid_flow_from_depth(1.0 / fin.squeeze(1), Ks, pose_ref)),
                              (RIGID_MEAN, RIGID_MAX), "px EPE")
                fout, mask = m._stage_refine_iter(P, rst, g0, g1, cl(fin, dev), task, it == n_it - 1, drefine)
                check_est("refine%d" % it, flow_err(fout, taps["refine%d.flow" % it]), est_tol)
            final = "refine%d.flow" % (n_it - 1)
            if task != "depth":
                check_feat("refine.mask", mask, taps["refine%d.mask" % (n_it - 1)], 1e-4)
                # ---- convex upsampling (utils.py:134-152) of the oracle's final estimate with the oracle's mask
                up = ops.convex_upsample(cl(taps[final], dev), cl(taps["refine%d.mask" % (n_it - 1)], dev), F, float(F))
                check_est("convex_upsample", full_err(up, ref_out), tuple(F * t for t in est_tol))
        if task == "depth" or not mk["reg_refine"]:
            # ---- learned upsampler (unimatch.py:81-93, :246-264) on the oracle's final estimate and feature0, with the
            # task's transforms: a disparity goes in and comes out negated, depth upsamples with mult 1 and is clamped
            est, f0_nchw = taps[final], feat0.cpu().permute(0, 3, 1, 2)
            pad = lambda t: torch.cat((t, torch.zeros_like(t)), 1)
            if task == "flow":
                got = m._stage_upsample_learned(P, cl(est, dev), feat0, F, F)
                ref = O._upsampler(sd, est, f0_nchw, F)
            elif task == "stereo":
                got = -m._stage_upsample_learned(P, cl(pad(-est), dev), feat0, F, F)[:, :1]
                ref = -O._upsampler(sd, pad(-est), f0_nchw, F)[:, :1]
            else:
                lo, hi = call["min_depth"], call["max_depth"]
                got = m._stage_upsample_learned(P, cl(pad(est), dev), feat0, F, 1).clamp(min=lo, max=hi)[:, :1]
                ref = O._upsampler(sd, pad(est), f0_nchw, F, True).clamp(min=lo, max=hi)[:, :1]
            check_est("upsample", full_err(got, ref), tuple(t * scale for t in upsample_tol(task)))
        # ---- and free-running end to end, in the output's unit, at bench.py's tolerance
        kw = dict(intrinsics=intr.to(dev), pose=pose.to(dev)) if task == "depth" else {}
        out = m(img0, img1, **kw, **call)["flow_preds"][-1]
        e2e_mean, e2e_max, e2e_unit = e2e_tol(workload)
        check_est("e2e", full_err(out if task == "flow" else out.unsqueeze(1), ref_out), (e2e_mean, e2e_max), e2e_unit)
        mag = ref_out.norm(dim=1) if task == "flow" else ref_out.abs()
        report("%-22s mean %.3e" % ("|reference output|", mag.mean().item()))
    return res
