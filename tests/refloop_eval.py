"""The reference's validation loops restated around a model, sample by sample (test infrastructure; tools/eval_bench.py times
it): evaluate_flow.py:160-638, evaluate_stereo.py:302-708 and evaluate_depth.py:22-293 with the dataset, `.to(device)` and the
printing taken out.  One sample per `model(...)` call, `InputPadder` in the mode each reference function uses (or the
`inference_size` resize, resize-back and rescale), the masks, the metrics in torch / numpy as the reference computes them
(flow on host copies, stereo on the device, depth in numpy), and the reference's own aggregation.  Nothing here calls the
validation drivers or `eval_stats`, so the drivers can be compared against it."""
import numpy as np
import torch
import torch.nn.functional as F

from unimatch_b200.inference import InputPadder


def _in_image(flow_gt):
    """utils/utils.py:compute_out_of_boundary_mask of one GT flow [2, H, W]"""
    _, h, w = flow_gt.shape
    ys, xs = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    corres = torch.stack((xs, ys), 0).float() + flow_gt
    m = (corres[0] >= 0) & (corres[0] <= w - 1) & (corres[1] >= 0) & (corres[1] <= h - 1)
    return m & (flow_gt[0].abs() <= w - 1) & (flow_gt[1].abs() <= h - 1)


@torch.no_grad()
def flow_loop(model, samples, *, protocol, device="cuda", dstype="clean", padding_factor=8, with_speed_metric=False,
              evaluate_matched_unmatched=False, average_over_pixels=True, max_val_flow=400, **model_kwargs):
    """validate_chairs / validate_things / validate_sintel / validate_kitti on `samples`"""
    model_kwargs["task"] = "flow"
    epe_list, out_list, bins, matched, unmatched = [], [], ([], [], []), [], []
    for s in samples:
        image1, image2, flow_gt = s[0][None].to(device), s[1][None].to(device), s[2]
        if protocol == "chairs":
            flow = model(image1, image2, **model_kwargs)["flow_preds"][-1][0].cpu()
        else:
            padder = InputPadder(image1.shape, mode="kitti" if protocol == "kitti" else "sintel", padding_factor=padding_factor)
            image1, image2 = padder.pad(image1, image2)
            flow = padder.unpad(model(image1, image2, **model_kwargs)["flow_preds"][-1][0]).cpu()
        epe = torch.sum((flow - flow_gt) ** 2, dim=0).sqrt()
        mag = torch.sum(flow_gt ** 2, dim=0).sqrt()
        if protocol == "things":
            val = (s[3] * (mag < max_val_flow)) >= 0.5
        elif protocol == "kitti":
            val = s[3] >= 0.5
        else:
            val = torch.ones_like(epe, dtype=torch.bool)
        if protocol == "kitti" and not average_over_pixels:
            epe_list.append(epe[val].mean().item())
        else:
            epe_list.append(epe[val].numpy())
        if protocol == "kitti":
            out_list.append(((epe > 3.0) & ((epe / mag) > 0.05)).float()[val].numpy())
        for lst, m in zip(bins, (mag < 10, (mag >= 10) * (mag <= 40), mag > 40)):
            m = m & val
            if m.max() > 0:
                lst.append((epe * m).sum() / m.sum() if protocol == "kitti" and not average_over_pixels else epe[m].numpy())
        if protocol == "sintel" and evaluate_matched_unmatched:
            mm = (s[4] > 0.5) & (_in_image(flow_gt) > 0.5)
            if mm.max() > 0:
                matched.append(epe[mm].numpy())
                unmatched.append(epe[~mm].numpy())
    prefix = {"sintel": "sintel_" + dstype, "things": "things_" + dstype}.get(protocol, protocol)
    per_sample = protocol == "kitti" and not average_over_pixels
    all_epe = np.array(epe_list) if per_sample else np.concatenate(epe_list)
    res = {prefix + "_epe": np.mean(all_epe)}
    if protocol in ("chairs", "sintel"):
        for t in (1, 3, 5):
            res["%s_%dpx" % (prefix, t)] = np.mean(all_epe > t)
    if protocol == "kitti":
        res["kitti_f1"] = 100 * np.mean(np.concatenate(out_list))
    if with_speed_metric:
        for key, lst in zip(("_s0_10", "_s10_40", "_s40+"), bins):
            res[prefix + key] = (sum(lst) / len(lst)).item() if per_sample else np.mean(np.concatenate(lst))
    if matched:
        res[prefix + "_matched"] = np.mean(np.concatenate(matched))
        res[prefix + "_unmatched"] = np.mean(np.concatenate(unmatched))
    return {k: float(v) for k, v in res.items()}


@torch.no_grad()
def stereo_loop(model, samples, *, protocol, device="cuda", padding_factor=16, inference_size=None, max_disp=400,
                **model_kwargs):
    """validate_things / validate_kitti15 / validate_eth3d / validate_middlebury on `samples`"""
    model_kwargs["task"] = "stereo"
    names = {"things": ("d1",), "kitti15": ("d1", "3px"), "eth3d": ("1px",), "middlebury": ("2px",)}[protocol]
    sums = dict.fromkeys(("epe",) + names, 0.0)
    valid_samples = 0
    for s in samples:
        left, right, gt_disp = s["left"][None].to(device), s["right"][None].to(device), s["disp"].to(device)
        if inference_size is None:
            padder = InputPadder(left.shape, padding_factor=padding_factor)
            left, right = padder.pad(left, right)
        else:
            ori_size = left.shape[-2:]
            left = F.interpolate(left, size=inference_size, mode="bilinear", align_corners=True)
            right = F.interpolate(right, size=inference_size, mode="bilinear", align_corners=True)
        mask = (gt_disp > 0) & (gt_disp < max_disp) if protocol == "things" else gt_disp > 0
        if not mask.any():
            continue
        valid_samples += 1
        pred_disp = model(left, right, **model_kwargs)["flow_preds"][-1]
        if inference_size is None:
            pred_disp = padder.unpad(pred_disp)[0]
        else:
            pred_disp = F.interpolate(pred_disp.unsqueeze(1), size=ori_size, mode="bilinear", align_corners=True).squeeze(1)[0]
            pred_disp = pred_disp * ori_size[-1] / float(inference_size[-1])
        d_est, d_gt = pred_disp[mask], gt_disp[mask]
        e = torch.abs(d_gt - d_est)
        sums["epe"] += F.l1_loss(d_gt, d_est, reduction="mean").item()
        metric = {"d1": (e > 3) & (e / d_gt > 0.05), "1px": e > 1.0, "2px": e > 2.0, "3px": e > 3.0}
        for k in names:
            sums[k] += torch.mean(metric[k].float()).item()
    return {"%s_%s" % (protocol, k): v / valid_samples for k, v in sums.items()}


@torch.no_grad()
def depth_loop(model, samples, *, protocol, device="cuda", padding_factor=16, inference_size=None, num_depth_candidates=64,
               eval_min_depth=0.5, eval_max_depth=10, min_depth=0.5, max_depth=10, **model_kwargs):
    """validate_scannet / validate_demon on `samples` (`protocol` only names the loop: both are the same)"""
    model_kwargs["task"] = "depth"
    names = ("abs_rel", "sq_rel", "rmse", "rmse_log", "a1", "a2", "a3")
    error_sum = [0.0] * len(names)
    for s in samples:
        img_ref, img_tgt = s["img_ref"][None].to(device), s["img_tgt"][None].to(device)
        gt_depth = s["depth"].to(device)
        if inference_size is None:
            padder = InputPadder(img_ref.shape, padding_factor=padding_factor, mode="kitti")
            img_ref, img_tgt = padder.pad(img_ref, img_tgt)
        else:
            ori_size = img_ref.shape[-2:]
            img_ref = F.interpolate(img_ref, size=inference_size, mode="bilinear", align_corners=True)
            img_tgt = F.interpolate(img_tgt, size=inference_size, mode="bilinear", align_corners=True)
        mask = (gt_depth > eval_min_depth) & (gt_depth < eval_max_depth) & (s["valid"].to(device) > 0.5)
        if not mask.any():
            continue
        pred_depth = model(img_ref, img_tgt, intrinsics=s["intrinsics"][None].to(device), pose=s["pose"][None].to(device),
                           min_depth=1. / max_depth, max_depth=1. / min_depth, num_depth_candidates=num_depth_candidates,
                           **model_kwargs)["flow_preds"][-1]
        if inference_size is None:
            pred_depth = padder.unpad(pred_depth)[0]
        else:
            pred_depth = F.interpolate(pred_depth.unsqueeze(1), size=ori_size, mode="bilinear", align_corners=True).squeeze(1)[0]
        mask = mask.cpu().numpy()
        gt, pred = gt_depth.cpu().numpy()[mask], pred_depth.cpu().numpy()[mask]
        thresh = np.maximum((gt / pred), (pred / gt))                      # loss/depth_loss.py:compute_errors
        metrics = [np.mean(np.abs(gt - pred) / gt), np.mean(((gt - pred) ** 2) / gt), np.sqrt(((gt - pred) ** 2).mean()),
                   np.sqrt(((np.log(gt) - np.log(pred)) ** 2).mean()), (thresh < 1.25).mean(), (thresh < 1.25 ** 2).mean(),
                   (thresh < 1.25 ** 3).mean()]
        error_sum = [a + b for a, b in zip(error_sum, metrics)]
    return {k: float(v / len(samples)) for k, v in zip(names, error_sum)}


LOOPS = {"flow": flow_loop, "stereo": stereo_loop, "depth": depth_loop}
