"""The matching-path kernels on the CUDA cores -- local correlation (stencil and gather), correlation volume, flow warp, local
propagation, the depth plane sweep, convex / x2 upsampling, the position add and the 7x7 stem / flow-encoder convolution --
at their real map sizes, tile seams, borders and coordinate edges, each against the float64 reference and per-element
error bound of tests/ref64.py (the printed `max err/bound` is the headroom).  References are evaluated on a pixel subset:
every border pixel, pixels on the tile seams and a few hundred random ones.  The `*_key` functions and `covered_keys()`
feed the launch census of tests/test_kernel_edges_gpu.py."""
import zlib

import pytest
import torch

import ref64
from test_ref64_cpu import STEM_SCALE, STEM_SHIFT, depth_setup, stem_images

pytestmark = pytest.mark.gpu
OPS = torch.ops.unimatch_sm100
C = 128


def g(name):
    return torch.Generator().manual_seed(zlib.crc32(name.encode()) % 100000)


def _feat(B, h, w, gen, scale):
    return torch.randn((B, h, w, C), generator=gen) * scale, torch.randn((B, h, w, C), generator=gen) * scale


# ---- dispatch keys (what selects a code path) ------------------------------------------------------------------------
def lcs_key(ry, rx, stereo):
    return ("local_corr_softmax", "stencil" if (not stereo and ry == 4 and rx == 4) else "gather", bool(stereo))


def corr_volume_key(fd):
    return ("local_corr_volume", fd)


def flow_warp_key(fd):
    return ("flow_warp", fd)


def propagate_key(radius, ldq, ldk, fd):
    return ("propagate_local", radius, ldq, ldk, fd)


def depth_key(n_cand, from_argmax):
    return ("depth_corr_softmax", n_cand, bool(from_argmax))


def convex_key(factor, fd, mult):
    return ("convex_upsample", factor, fd, mult == 1)


def upsample2x_key(fd):
    return ("upsample2x", fd)


def add_position_key():
    return ("add_position",)


def conv7x7_key(cin, stride, nchw, two_sources, normalised, f32, split):
    return ("conv7x7_small", cin, stride, bool(nchw), bool(two_sources), bool(normalised), bool(f32), bool(split))


# ---- local_corr_softmax ----------------------------------------------------------------------------------------------
LCS_EDGE = [
    # name, B, h, w, ry, rx, stereo, feature scale
    ("stencil_120x208_b2", 2, 120, 208, 4, 4, False, 1.5),     # the 1/4-scale map: 6.5 tiles wide, 15 tiles high
    ("stencil_8x32_one_tile", 1, 8, 32, 4, 4, False, 1.5),
    ("stencil_9x33", 2, 9, 33, 4, 4, False, 1.5),               # one pixel into the second tile both ways
    ("stencil_7x31", 2, 7, 31, 4, 4, False, 1.5),               # one ragged tile
    ("stencil_5x5", 2, 5, 5, 4, 4, False, 1.5),                 # map smaller than the window
    ("stencil_64x96_b3", 3, 64, 96, 4, 4, False, 1.5),          # many tiles per image, batch 3
    ("stencil_peaked_60x104", 2, 60, 104, 4, 4, False, 8.0),    # logits about +-200
    ("gather_stereo_136x240_b2", 2, 136, 240, 0, 4, True, 1.5),
    ("gather_stereo_narrow_6x7", 2, 6, 7, 0, 4, True, 1.5),      # row narrower than the window
    ("gather_flow_r3_30x50", 2, 30, 50, 3, 3, False, 1.5),
]


@pytest.mark.parametrize("name,B,h,w,ry,rx,stereo,scale", LCS_EDGE)
def test_local_corr_softmax_edges(name, B, h, w, ry, rx, stereo, scale):
    gen = g(name)
    f0, f1 = _feat(B, h, w, gen, scale)
    stencil = lcs_key(ry, rx, stereo)[1] == "stencil"
    pix = ref64.pixel_subset(B, h, w, gen, (32,) if stencil else (), (8,) if stencil else ())
    ref, bnd = ref64.local_corr_softmax64(f0, f1, ry, rx, stereo, pix, stencil)
    out = OPS.local_corr_softmax(f0.cuda(), f1.cuda(), h, w, ry, rx, stereo).cpu()
    ref64.check("lcs " + name, out[pix], ref, bnd)


@pytest.mark.parametrize("dx,dy", [(3, -2), (-4, 4), (0, 1)])
def test_local_corr_softmax_stencil_recovers_translation(dx, dy):
    """f1 = f0 moved by (dx, dy) with peaked features: away from the border every pixel's flow is exactly (dx, dy)."""
    B, h, w = 2, 64, 96
    f0 = torch.randn((B, h, w, C), generator=g("translation %d %d" % (dx, dy))) * 4.0
    f1 = torch.roll(f0, (dy, dx), (1, 2))
    out = OPS.local_corr_softmax(f0.cuda(), f1.cuda(), h, w, 4, 4, False).cpu()[:, 8:h - 8, 8:w - 8]
    assert torch.equal(out, torch.tensor([float(dx), float(dy)]).expand_as(out)), (out - torch.tensor([dx, dy])).abs().max()


# ---- local_corr_volume and flow_warp ---------------------------------------------------------------------------------
def make_flow(kind, B, h, w, fd, gen):
    shp = (B, h, w, fd)
    if kind == "zero":
        return torch.zeros(shp)
    if kind == "integer":
        return torch.randint(-6, 7, shp, generator=gen).float()
    if kind == "half":
        return torch.randint(-4, 5, shp, generator=gen).float() + torch.where(torch.rand(shp, generator=gen) < 0.5, 0.5, -0.5)
    if kind == "near_int":
        return torch.randint(-4, 5, shp, generator=gen).float() + (torch.rand(shp, generator=gen) - 0.5) * 2e-6
    if kind == "sigma12":
        return torch.randn(shp, generator=gen) * 12
    if kind == "outside":                                    # the whole window right of the image
        return w + 5 + torch.rand(shp, generator=gen) * 5
    if kind == "edge":                                       # positions in (-1, 0): the tap x0 = -1 (y0 = -1) is read
        ys, xs = torch.meshgrid(torch.arange(h).float(), torch.arange(w).float(), indexing="ij")
        own = torch.stack((xs, ys), -1)[None, ..., :fd]
        if fd == 1:                                          # a disparity d moves x to x - d
            return own + torch.rand(shp, generator=gen)
        return -own - torch.rand(shp, generator=gen)
    raise ValueError(kind)


CV_EDGE = [
    # flow kind, fd, (B, h, w)
    ("zero", 2, (2, 120, 208)), ("integer", 2, (2, 120, 208)), ("half", 2, (2, 120, 208)), ("near_int", 2, (2, 120, 208)),
    ("sigma12", 2, (2, 120, 208)), ("outside", 2, (2, 120, 208)), ("edge", 2, (2, 120, 208)),
    ("sigma12", 1, (2, 120, 208)), ("half", 1, (2, 120, 208)), ("edge", 1, (2, 120, 208)), ("outside", 1, (2, 60, 104)),
    ("sigma12", 2, (2, 60, 104)), ("near_int", 1, (2, 60, 104)), ("integer", 1, (2, 60, 104)),
]


@pytest.mark.parametrize("kind,fd,shape", CV_EDGE)
def test_corr_volume_and_flow_warp_edges(kind, fd, shape):
    B, h, w = shape
    name = "%s fd %d %dx%d" % (kind, fd, h, w)
    gen = g(name)
    f0, f1 = _feat(B, h, w, gen, 1.5)
    fl = make_flow(kind, B, h, w, fd, gen)
    pix = ref64.pixel_subset(B, h, w, gen, (), (), n_seam=0, n_rand=600)
    ref, bnd = ref64.local_corr_volume64(f0, f1, fl, 4, pix)
    corr = OPS.local_corr_volume(f0.cuda(), f1.cuda(), fl.cuda(), h, w, 4).cpu()
    ref64.check("corr volume " + name, corr[pix], ref, bnd)
    ref, bnd = ref64.flow_warp64(f1, fl, pix)
    warped = OPS.flow_warp(f1.cuda(), fl.cuda(), h, w).cpu()
    ref64.check("flow warp " + name, warped[pix], ref, bnd)
    if kind == "outside":
        assert corr.abs().max() == 0 and warped.abs().max() == 0


# ---- propagate_local ---------------------------------------------------------------------------------------------------
PROP_EDGE = [
    # fd, (B, h, w), q/k scale
    (2, (2, 120, 208), 1.5), (1, (2, 136, 240), 1.5), (2, (2, 60, 104), 8.0), (1, (2, 120, 208), 8.0),
]


@pytest.mark.parametrize("fd,shape,scale", PROP_EDGE)
def test_propagate_local_strided_rows(fd, shape, scale):
    """q / k as the [..., :128] / [..., 128:] views of one [nb, L, 256] projection (row stride 256), as the module passes
    them."""
    B, h, w = shape
    gen = g("prop %d %s %g" % (fd, shape, scale))
    qk = torch.randn((B, h * w, 256), generator=gen) * scale
    fl = torch.randn((B, h, w, fd), generator=gen) * 6
    pix = ref64.pixel_subset(B, h, w, gen)
    ref, bnd = ref64.propagate_local64(qk[..., :128].reshape(B, h, w, C), qk[..., 128:].reshape(B, h, w, C), fl, 1, pix)
    qkd = qk.cuda()
    q, k = qkd[:, :, :128], qkd[:, :, 128:]
    assert q.stride(-2) == 256 and k.stride(-2) == 256
    out = OPS.propagate_local(q, k, fl.cuda(), h, w, 1).cpu()
    ref64.check("propagate fd %d %dx%d scale %g" % (fd, h, w, scale), out[pix], ref, bnd)


# ---- depth_corr_softmax ----------------------------------------------------------------------------------------------
DEPTH_EDGE = [
    # camera motion, negative in-image correlations (argmax ties at logit 0)
    ("bidir", False), ("rotated", False), ("forward", False), ("forward", True),
]


@pytest.mark.parametrize("kind,neg", DEPTH_EDGE)
def test_depth_corr_softmax_edges(kind, neg):
    """64 candidates over the workloads' depth range at 48 x 64, bidirectional poses (pose and its inverse, batch 2) built
    by UniMatch.depth_cameras; "forward" moves 2 units forward so near candidates project behind the camera."""
    B, h, w = 2, 48, 64
    name = "depth %s%s" % (kind, " neg" if neg else "")
    f0, f1, cams = depth_setup(B, h, w, zlib.crc32(name.encode()) % 1000, kind, neg)
    pix = ref64.pixel_subset(B, h, w, g(name), (), (), n_seam=0, n_rand=400)
    ref, bnd, s, ds = ref64.depth_corr64(f0, f1, cams["K"], cams["K_inv"], cams["pose"], cams["cand"], pix)
    dev = [t.contiguous().cuda() for t in (f0, f1, cams["K"], cams["K_inv"], cams["pose"], cams["cand"])]
    soft = OPS.depth_corr_softmax(*dev, h, w, False).cpu()[..., 0]
    ref64.check(name + " softmax", soft[pix], ref, bnd)
    arg = OPS.depth_corr_softmax(*dev, h, w, True).cpu()[..., 0]
    ref64.check_argmax(name, arg[pix], cams["cand"], s, ds)


# ---- convex_upsample / upsample2x / add_position ---------------------------------------------------------------------
CONVEX_EDGE = [
    # factor, fd, mult, (B, h, w), mask logit scale
    (4, 2, 4, (2, 120, 208), 3.0), (4, 1, 4, (2, 136, 240), 3.0), (8, 2, 8, (2, 60, 104), 3.0), (8, 2, 1, (2, 48, 64), 3.0),
    (8, 1, 1, (2, 48, 64), 3.0), (4, 2, 4, (2, 60, 104), 60.0), (8, 1, 1, (2, 48, 64), 60.0), (8, 2, 8, (1, 60, 104), 60.0),
]


@pytest.mark.parametrize("factor,fd,mult,shape,scale", CONVEX_EDGE)
def test_convex_upsample_edges(factor, fd, mult, shape, scale):
    B, h, w = shape
    name = "convex F %d fd %d mult %d %dx%d scale %g" % (factor, fd, mult, h, w, scale)
    gen = g(name)
    fl = torch.randn((B, h, w, fd), generator=gen) * 6
    mask = torch.randn((B, h, w, 9 * factor * factor), generator=gen) * scale
    rows = torch.cat((torch.tensor([0, 1, h - 2, h - 1]), torch.randperm(h, generator=gen)[:6])).unique()
    ref, bnd = ref64.convex_upsample64(fl, mask, factor, mult, rows)
    out = OPS.convex_upsample(fl.cuda(), mask.cuda(), factor, float(mult)).cpu()
    sel = (rows[:, None] * factor + torch.arange(factor)).reshape(-1)
    ref64.check(name, out[:, :, sel], ref, bnd)


@pytest.mark.parametrize("fd,shape", [(2, (2, 60, 104)), (1, (2, 60, 104)), (2, (2, 68, 120)), (1, (2, 68, 120)),
                                      (2, (2, 1, 50)), (1, (3, 1, 33))])
def test_upsample2x_edges(fd, shape):
    B, h, w = shape
    fl = torch.randn((B, h, w, fd), generator=g("up2 %d %s" % (fd, shape))) * 8
    ref, bnd = ref64.upsample2x64(fl, 2.0)
    ref64.check("upsample2x fd %d %dx%d" % (fd, h, w), OPS.upsample2x(fl.cuda(), 2.0).cpu(), ref, bnd)


@pytest.mark.parametrize("n,h,w,wh,ww", [(4, 120, 208, 15, 26), (2, 60, 104, 30, 52)])
def test_add_position_bit_exact(n, h, w, wh, ww):
    """4 x 120 x 208 x 128 floats take the kernel's grid-stride loop."""
    gen = g("addpos %d %d" % (n, h))
    x = torch.randn((n, h, w, C), generator=gen)
    table = torch.randn((wh, ww, C), generator=gen)
    out = OPS.add_position(x.cuda(), table.cuda(), h, w).cpu()
    assert torch.equal(out, ref64.add_position_ref(x, table, h, w))
    print("%-60s bit-exact" % ("add_position %dx%dx%d table %dx%d" % (n, h, w, wh, ww)))


# ---- conv7x7_small ---------------------------------------------------------------------------------------------------
STEM_EDGE = [
    # (N, H, W), normalisation folded in
    ((2, 480, 832), True), ((2, 375, 1242), True), ((2, 375, 1242), False),
]


@pytest.mark.parametrize("shape,norm", STEM_EDGE)
def test_conv7x7_stem_edges(shape, norm):
    """The image stem: 3 -> 64, stride 2, two planar sources (first and second image of the pair), raw pixels with saturated
    0 / 255 blocks; 375 x 1242 leaves ragged 32 x 8 output tiles and runs more tiles than persistent CTAs."""
    N, H, W = shape
    x = stem_images(N, H, W, zlib.crc32(str(shape).encode()) % 1000)
    if not norm:
        x = (x / 127.5 - 1.0).float()
    wt = torch.randn((64, 3, 7, 7), generator=g("stem %s" % (shape,))) * (2.0 / 147) ** 0.5
    sc, sh = (STEM_SCALE, STEM_SHIFT) if norm else (None, None)
    ref, bnd = ref64.conv7x7_64(x, wt, None, 2, False, sc, sh)
    out = torch.zeros(ref.shape, device="cuda")
    OPS.conv7x7_small(x[:N // 2].cuda(), x[N // 2:].cuda(), True, wt.cuda(), None, 2, False, sc, sh, out, None)
    ref64.check("stem %dx%d norm %s" % (H, W, norm), out.cpu(), ref, bnd, ref64.conv_locator(16))


FLOWENC_EDGE = [(1, "split"), (2, "split"), (1, "f32"), (2, "f32")]


@pytest.mark.parametrize("cin,output", FLOWENC_EDGE)
def test_conv7x7_flow_encoder_edges(cin, output):
    """The flow encoder's first layer: 1-2 -> 128, stride 1, bias + ReLU, flows up to 50 px at 120 x 208; split planes only,
    as the module writes it, or fp32 only."""
    B, h, w = 2, 120, 208
    gen = g("flow encoder %d %s" % (cin, output))
    fl = (torch.randn((B, h, w, cin), generator=gen) * 20).clamp(-50, 50)
    wt = torch.randn((128, cin, 7, 7), generator=gen) * (2.0 / (49 * cin)) ** 0.5
    bias = torch.randn(128, generator=gen) * 0.1
    ref, bnd = ref64.conv7x7_64(fl.permute(0, 3, 1, 2), wt, bias, 1, True)
    out_f = torch.zeros((B, h, w, C), device="cuda") if output == "f32" else None
    out_s = torch.zeros((2, B, h, w, C), dtype=torch.float16, device="cuda") if output == "split" else None
    OPS.conv7x7_small(fl.cuda(), None, False, wt.cuda(), bias.cuda(), 1, True, None, None, out_f, out_s)
    name = "flow encoder cin %d %s" % (cin, output)
    if output == "f32":
        ref64.check(name, out_f.cpu(), ref, bnd, ref64.conv_locator(16))
    else:
        ref64.check(name, (out_s[0].double() + out_s[1].double()).cpu(), ref, ref64.split_out_bound(ref, bnd),
                    ref64.conv_locator(16))


# ---- the keys the tables above cover ---------------------------------------------------------------------------------
def covered_keys():
    keys = set()
    for name, B, h, w, ry, rx, stereo, _ in LCS_EDGE:
        keys.add(lcs_key(ry, rx, stereo))
    for kind, fd, _ in CV_EDGE:
        keys.add(corr_volume_key(fd))
        keys.add(flow_warp_key(fd))
    for fd, *_ in PROP_EDGE:
        keys.add(propagate_key(1, 256, 256, fd))
    for _ in DEPTH_EDGE:
        keys.add(depth_key(64, False))
        keys.add(depth_key(64, True))
    for factor, fd, mult, *_ in CONVEX_EDGE:
        keys.add(convex_key(factor, fd, mult))
    keys |= {upsample2x_key(1), upsample2x_key(2), add_position_key()}
    for _, norm in STEM_EDGE:
        keys.add(conv7x7_key(3, 2, True, True, norm, True, False))
    for cin, output in FLOWENC_EDGE:
        keys.add(conv7x7_key(cin, 1, False, False, False, output == "f32", output == "split"))
    return keys
