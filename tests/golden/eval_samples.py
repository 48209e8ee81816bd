"""Seeded in-memory validation samples and the deterministic stub model of the evaluation goldens (tests/golden/golden_eval.pt,
written by make_golden_eval.py from the reference's own validate_* loops).  Plain torch, no reference import: the tests rebuild
the samples from here and check them against the digests stored in the golden file, which keeps that file at a few kB instead
of 12 MB.  The samples come from torch's CPU generator (`torch.Generator`, randint / randn / rand): a torch release that changes
those streams makes the digest check fail loudly, and the golden file then has to be regenerated with make_golden_eval.py where
the reference is available."""
import hashlib

import torch


class Stub:
    """Deterministic model: an elementwise function of the (padded) inputs.  Flow: (u, v) = (img1[0] - img2[1], img1[2] -
    img2[0]) / 8 on [0, 255] integer images (exact multiples of 1/8); stereo: 5 |floor(10 left[0])| (multiples of 5 up to
    about 130); depth: 1 + floor(4 |ref[0]|) / 4.  Integer-grid predictions let the GT put errors exactly on the thresholds."""

    def eval(self):
        return self

    def __call__(self, a, b, task="flow", **kw):
        if task == "flow":
            return {"flow_preds": [torch.stack(((a[:, 0] - b[:, 1]) * 0.125, (a[:, 2] - b[:, 0]) * 0.125), 1)]}
        if task == "stereo":
            return {"flow_preds": [torch.floor(a[:, 0] * 10.0).abs() * 5.0]}
        return {"flow_preds": [1.0 + torch.floor(a[:, 0].abs() * 4.0) * 0.25]}


STUB = Stub()


def _img(g, h, w, normalized):
    x = torch.randint(0, 256, (3, h, w), generator=g).float()
    if normalized:
        mean = torch.tensor([0.485, 0.456, 0.406]).view(3, 1, 1)
        std = torch.tensor([0.229, 0.224, 0.225]).view(3, 1, 1)
        x = (x / 255.0 - mean) / std
    return x


def flow_samples(seed, shapes, n, sparse=False, noc=False, empty=()):
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        h, w = shapes[i % len(shapes)]
        img1, img2 = _img(g, h, w, False), _img(g, h, w, False)
        pred = STUB(img1[None], img2[None])["flow_preds"][0][0]
        kind = torch.randint(0, 6, (h, w), generator=g)
        delta = torch.randn((2, h, w), generator=g) * torch.tensor([2.0, 8.0, 30.0])[torch.randint(0, 3, (1,), generator=g)]
        delta[0][kind == 1], delta[1][kind == 1] = 1.0, 0.0          # epe exactly 1, 3, 5
        delta[0][kind == 2], delta[1][kind == 2] = 0.0, 3.0
        delta[0][kind == 3], delta[1][kind == 3] = -3.0, -4.0
        gt = pred + delta
        gt[:, :h // 6, :w // 5] = 0.0                                 # zero-magnitude GT
        gt[0, h // 2, :] = 40.0                                       # speeds exactly on the bin edges
        gt[0, h // 2 + 1, :] = 10.0
        gt[:, h // 3, :] += torch.linspace(-60, 160, w)               # fast pixels, some out of the image
        valid = (torch.rand((h, w), generator=g) < (0.4 if sparse else 0.95)).float()
        if i in empty:
            valid.zero_()
        s = [img1, img2, gt, valid]
        if noc:
            nv = (torch.rand((h, w), generator=g) < 0.8).float()
            if i in empty:
                nv.zero_()
            s.append(nv)
        out.append(tuple(s))
    return out


def stereo_samples(seed, shapes, n, empty=()):
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        h, w = shapes[i % len(shapes)]
        left, right = _img(g, h, w, True), _img(g, h, w, True)
        pred = STUB(left[None], right[None], task="stereo")["flow_preds"][0][0]
        kind = torch.randint(0, 7, (h, w), generator=g)
        gt = pred + torch.randn((h, w), generator=g) * 4.0
        for k, d in ((1, 1.0), (2, -2.0), (3, 3.0)):                   # e exactly 1, 2, 3
            gt[kind == k] = (pred + d)[kind == k]
        gt[kind == 4] = 100.0                                         # e = 5 and e / gt exactly 0.05 where pred = 95 / 105
        gt[kind == 5] = 0.0                                           # invalid
        big = (kind == 6) & (pred >= 80)
        gt[big] = (pred + 4.0)[big]                                   # e = 4 > 3 but e / gt < 0.05: 3px, not D1
        gt[0, :] = 400.0                                              # on the Things max_disp bound
        gt[1, :] = 450.0
        if i in empty:
            gt.fill_(-1.0)
        out.append({"left": left, "right": right, "disp": gt})
    return out


def depth_samples(seed, shapes, n, empty=()):
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        h, w = shapes[i % len(shapes)]
        ref, tgt = _img(g, h, w, True), _img(g, h, w, True)
        pred = STUB(ref[None], tgt[None], task="depth")["flow_preds"][0][0]
        kind = torch.randint(0, 6, (h, w), generator=g)
        gt = pred * torch.exp(torch.randn((h, w), generator=g) * 0.3)
        gt[kind == 1] = (pred * 1.25)[kind == 1]                      # ratio exactly 1.25 (and 1.5625 below)
        gt[kind == 2] = (pred * 1.5625)[kind == 2]
        gt[kind == 3] = 0.5                                           # on the eval range bounds
        gt[kind == 4] = 10.0
        gt[0, :] = 12.0
        valid = (torch.rand((h, w), generator=g) < 0.9).float()
        if i in empty:
            valid.zero_()
        K = torch.tensor([[0.9 * w, 0.0, w / 2.0], [0.0, 0.9 * w, h / 2.0], [0.0, 0.0, 1.0]])
        pose = torch.eye(4)
        pose[0, 3] = 0.1
        out.append({"img_ref": ref, "img_tgt": tgt, "intrinsics": K, "pose": pose, "depth": gt, "valid": valid})
    return out


S1, S2, S3 = (64, 96), (75, 130), (70, 101)

# (case name, task, driver options, samples); the reference function and its dataset class per case are in make_golden_eval.py
CASES = [
    ("chairs", "flow", dict(protocol="chairs"), lambda: flow_samples(21, [S1], 4)),
    ("chairs_speed", "flow", dict(protocol="chairs", with_speed_metric=True), lambda: flow_samples(21, [S1], 4)),
    ("things_speed", "flow", dict(protocol="things", with_speed_metric=True, max_val_flow=100, padding_factor=16),
     lambda: flow_samples(22, [S3], 4, empty=(1,))),
    ("sintel_matched_speed", "flow", dict(protocol="sintel", with_speed_metric=True, evaluate_matched_unmatched=True,
                                          dstype="clean"), lambda: flow_samples(23, [S2], 5, noc=True, empty=(2,))),
    ("kitti", "flow", dict(protocol="kitti", with_speed_metric=True),
     lambda: flow_samples(11, [S1, S2], 6, sparse=True, empty=(3,))),
    ("kitti_per_sample", "flow", dict(protocol="kitti", with_speed_metric=True, average_over_pixels=False),
     lambda: flow_samples(12, [S2, S1], 5, sparse=True)),
    ("stereo_things", "stereo", dict(protocol="things"), lambda: stereo_samples(31, [S1], 4, empty=(2,))),
    ("stereo_kitti15", "stereo", dict(protocol="kitti15"), lambda: stereo_samples(32, [S1, S2], 6, empty=(1,))),
    ("stereo_eth3d", "stereo", dict(protocol="eth3d"), lambda: stereo_samples(33, [S3], 3)),
    ("stereo_middlebury", "stereo", dict(protocol="middlebury", padding_factor=32), lambda: stereo_samples(34, [S2], 3)),
    ("depth_scannet", "depth", dict(protocol="scannet"), lambda: depth_samples(41, [S1, S3], 5, empty=(3,))),
    ("depth_demon", "depth", dict(protocol="demon", eval_min_depth=1.0, eval_max_depth=8.0), lambda: depth_samples(42, [S2], 3)),
]


def digest(samples):
    """sha256 over every tensor of a sample list, in order"""
    h = hashlib.sha256()
    for s in samples:
        for t in (s.values() if isinstance(s, dict) else s):
            h.update(t.contiguous().numpy().tobytes())
    return h.hexdigest()
