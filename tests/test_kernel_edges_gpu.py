"""Tensor-core convolution / Linear, window attention, softmax expectation, fused FFN and instance norm at their tile,
window and magnitude edges, each against the float64 reference and per-element error bound of tests/ref64.py (the printed
`max err/bound` is the headroom).  The last test takes a census of the dispatch keys the bench workloads launch and
requires every one of them to appear in the case tables here."""
import inspect
import math
import zlib

import pytest
import torch

import ref64
import test_matching_edges_gpu as M
from unimatch_b200 import ops

pytestmark = pytest.mark.gpu
OPS = torch.ops.unimatch_sm100
C = 128
LAZY_THRESH = 8.0 * math.sqrt(C) / 1.4426950408889634


def g(seed):
    return torch.Generator().manual_seed(seed)


# ---- attention -------------------------------------------------------------------------------------------------------
ATTN_EDGE = [
    # name, n, h, w, kh, kw, shift, kv_shift, q/k scale          dispatch
    ("lw127_full", 2, 1, 127, 1, 1, False, 1, 1.5),             # CUDA cores: below one query tile
    ("lw128_full", 2, 8, 16, 1, 1, False, 1, 1.5),              # exactly one query tile
    ("lw129_full", 2, 3, 43, 1, 1, False, 1, 1.5),              # one-row last query tile, one-key last key tile
    ("lw192_full", 2, 12, 16, 1, 1, False, 0, 1.5),             # second consumer warpgroup holds only padding
    ("lw2048_full", 1, 32, 64, 1, 1, False, 0, 1.5),            # = MAX_LP
    ("lw2100_full", 1, 30, 70, 1, 1, False, 0, 1.5),            # dense window > MAX_LP: CUDA cores
    ("full1d_48x156", 2, 48, 156, 48, 1, False, 1, 1.5),        # KITTI stereo at 1/8: 1-D rows on the tensor cores
    ("full1d_136x240", 2, 136, 240, 136, 1, False, 1, 1.5),
    ("swin1d_shifted_lw256", 2, 4, 512, 4, 2, True, 1, 1.5),    # 1-D region mask on the tensor cores
    ("swin2d_lw390", 2, 30, 52, 2, 2, False, 1, 1.5),
    ("swin2d_first_tile_masked", 2, 32, 16, 2, 2, True, 1, 1.5),
    ("swin2d_lw2304_cuda_cores", 1, 96, 96, 2, 2, False, 0, 1.5),  # windows > MAX_LP (Middlebury stereo at 1/8: 6144)
    ("swin1d_lw60_cuda_cores", 2, 4, 240, 4, 4, False, 1, 1.5),  # gmstereo-scale2's 1-D windows
    ("swin1d_lw60_shifted_cuda_cores", 2, 4, 240, 4, 4, True, 1, 1.5),
    ("three_streams_kvshift2", 3, 16, 24, 2, 2, True, 2, 1.5),
    ("peaked_pm200", 2, 12, 16, 1, 1, False, 1, 8.0),          # scaled logits up to about +-200
]


def _geom(h, w, kh, kw, shift):
    wh, ww = h // kh, w // kw
    sh = (wh // 2 if kh != h else 0) if shift else 0
    sw = ww // 2 if shift else 0
    return sh, sw, ops.MASK_SWIN if shift else ops.MASK_NONE


def _planes(x, tok, lp):
    """[n, L, 128] fp32 -> window-major fp16 (hi, lo) planes [2, n, nwin, lp, 128], padding rows zero."""
    n = x.shape[0]
    nwin, lw = tok.shape
    pl = torch.zeros((2, n, nwin, lp, C), dtype=torch.float16)
    xs = x[:, tok.reshape(-1)].view(n, nwin, lw, C)
    hi = xs.half()
    pl[0, :, :, :lw] = hi
    pl[1, :, :, :lw] = (xs - hi.float()).half()
    return pl


def _run_attention(name, q, k, v, kvs, h, w, kh, kw, shift):
    n = q.shape[0]
    sh, sw, mask = _geom(h, w, kh, kw, shift)
    ref, bnd, loc = ref64.attention64(q, k, v, kvs, h, w, kh, kw, sh, sw, mask)
    lp = ops.attention_planes_lp(h, w, kh, kw, sh, sw, mask)
    out = OPS.window_attention(q.cuda(), k.cuda(), v.cuda(), kvs, h, w, kh, kw, sh, sw, mask)
    ref64.check("%s rows (%s)" % (name, "tc" if lp else "cuda cores"), out, ref, bnd, loc)
    if lp:
        tok, _ = ref64.window_layout(h, w, kh, kw, sh, sw)
        out_f = torch.full((n, h * w, C), 3.0).cuda()
        out_s = torch.full((2, n * h * w + 16, C), 7.0, dtype=torch.float16).cuda()
        OPS.window_attention_planes(_planes(q, tok, lp).cuda(), _planes(k, tok, lp).cuda(), _planes(v, tok, lp).cuda(), n, kvs,
                                    h, w, kh, kw, sh, sw, mask, out_f, out_s)
        ref64.check(name + " planes out_f32", out_f, ref, bnd, loc)
        ref64.check(name + " planes out_split", (out_s[0].double() + out_s[1].double())[:n * h * w].view(n, h * w, C).cpu(),
                    ref, ref64.split_out_bound(ref, bnd), loc)
        assert (out_s[:, n * h * w:] == 7.0).all(), "rows past the tokens were written"
        _, bnd_cc, _ = ref64.attention64(q, k, v, kvs, h, w, kh, kw, sh, sw, mask, tc=False)
        ops.set_force_cuda_cores(True)
        try:
            out_cc = OPS.window_attention(q.cuda(), k.cuda(), v.cuda(), kvs, h, w, kh, kw, sh, sw, mask)
        finally:
            ops.set_force_cuda_cores(False)
        ref64.check(name + " forced cuda cores", out_cc, ref, bnd_cc, loc)
    return lp


@pytest.mark.parametrize("name,n,h,w,kh,kw,shift,kvs,scale", ATTN_EDGE)
def test_attention_edges(name, n, h, w, kh, kw, shift, kvs, scale):
    gen = g(zlib.crc32(name.encode()) % 10000)
    L = h * w
    q, k = (torch.randn((n, L, C), generator=gen) * scale for _ in range(2))
    v = torch.randn((n, L, C), generator=gen)
    lp = _run_attention(name, q, k, v, kvs, h, w, kh, kw, shift)
    lw = (h // kh) * (w // kw)
    assert (lp > 0) == (128 <= lw <= 2048), (name, lp)


@pytest.mark.parametrize("grow,tile", [(LAZY_THRESH - 0.25, 1), (LAZY_THRESH + 0.25, 1), (60.0 * math.sqrt(C), 2)])
def test_attention_lazy_rescale(grow, tile):
    """The running max grows in a later key tile by LAZY_THRESH -/+ eps, or by ~60 scaled-logit units in the last tile."""
    gen = g(int(grow))
    n, h, w = 2, 12, 16
    q = torch.randn((n, h * w, C), generator=gen) * 0.3
    k = torch.randn((n, h * w, C), generator=gen) * 0.3
    v = torch.randn((n, h * w, C), generator=gen)
    q[..., 0] = 16.0
    k[..., 0] = 0.0
    k[:, 64 * tile + 5, 0] = grow / 16.0
    _run_attention("lazy grow %.2f tile %d" % (grow, tile), q, k, v, 1, h, w, 1, 1, False)


# ---- softmax expectation ---------------------------------------------------------------------------------------------
EXP_EDGE = [
    # name, n_total, n_streams, kv_shift, h, w, vdim, value_mode, post, kh, kw, mask, q/k scale
    ("corr_bidir_L6240", 2, 2, 1, 60, 104, 2, ops.VALUE_COORDS, ops.POST_MINUS_OWN, 1, 1, ops.MASK_NONE, 1.5),
    ("prop_vdim2_L6240", 2, 2, 0, 60, 104, 2, ops.VALUE_TENSOR, ops.POST_NONE, 1, 1, ops.MASK_NONE, 1.5),
    ("prop_vdim1_L8160", 2, 2, 0, 68, 120, 1, ops.VALUE_TENSOR, ops.POST_NONE, 1, 1, ops.MASK_NONE, 1.5),
    ("stereo_causal_w120", 2, 2, 1, 8, 120, 1, ops.VALUE_XCOORD, ops.POST_OWN_MINUS, 8, 1, ops.MASK_CAUSAL, 1.5),
    ("stereo_causal_w240", 2, 2, 1, 6, 240, 1, ops.VALUE_XCOORD, ops.POST_OWN_MINUS, 6, 1, ops.MASK_CAUSAL, 1.5),
    ("corr_peaked_L6240", 2, 2, 1, 60, 104, 2, ops.VALUE_COORDS, ops.POST_MINUS_OWN, 1, 1, ops.MASK_NONE, 8.0),
]


@pytest.mark.parametrize("name,nt,ns,kvs,h,w,vdim,vm,post,kh,kw,mask,scale", EXP_EDGE)
def test_softmax_expectation_edges(name, nt, ns, kvs, h, w, vdim, vm, post, kh, kw, mask, scale):
    gen = g(zlib.crc32(name.encode()) % 10000)
    L = h * w
    q = torch.randn((nt, L, C), generator=gen) * scale
    k = torch.randn((nt, L, C), generator=gen) * scale
    vals = torch.randn((nt, L, vdim), generator=gen) * 3 if vm == ops.VALUE_TENSOR else None
    # query rows checked: the first and last 160 (ragged tiles, image borders) and 320 random ones
    rows = torch.cat((torch.arange(160), torch.arange(L - 160, L), torch.randperm(L, generator=gen)[:320])).unique()
    ref, bnd = ref64.expectation64(q, k, vals, ns, kvs, vdim, vm, post, h, w, kh, kw, mask, rows)
    tc = _expect_tc(h, w, kh, kw, mask, nt, vm)
    for force in ((False, True) if tc else (False,)):
        ops.set_force_cuda_cores(force)
        try:
            out = OPS.softmax_expectation(q.cuda(), k.cuda(), None if vals is None else vals.cuda(), ns, kvs, vdim, vm, post,
                                          h, w, kh, kw, mask)
        finally:
            ops.set_force_cuda_cores(False)
        ref64.check("%s (%s)" % (name, "cuda cores" if force or not tc else "tc"), out[:, rows].cpu(), ref, bnd)


# ---- convolution / Linear --------------------------------------------------------------------------------------------
# The C dispatch rule of um_conv2d_tc (unimatch_b200/csrc/um_conv_tc.cu, the UM_CONV_CASE table after the window-plane
# branch): the requested tile width 256 / 192 runs as 128 / 96; K >= 512 (8 stages of 64) selects the multi-stage
# accumulators (G = 2 for 128 / 96, 4 for 64 / 16); the listed (bn, G, mode, act) have their own epilogue, the rest run
# the run-time-mode one.
FIXED = {(128, 1, 0, 0), (128, 1, 0, 1), (128, 1, 0, 4), (128, 1, 3, 0), (128, 2, 3, 0), (128, 2, 0, 0), (128, 2, 0, 1),
         (128, 2, 1, 0), (128, 2, 2, 0), (96, 2, 0, 1), (64, 4, 0, 0), (64, 4, 0, 1)}


def conv_dispatch(bn, ktot, mode, act, win):
    """(bn, G, MODE, ACT, WIN) of the conv_tc_kernel instantiation a launch runs."""
    if win:
        return (128, 1, 0, 0, True)
    b = {256: 128, 192: 96}.get(bn, bn)
    gg = ({128: 2, 96: 2}.get(b, 4)) if ktot // 64 >= 8 else 1
    key = (b, gg, mode, act if mode == ops.CONV_LINEAR else 0)
    return key + (False,) if key in FIXED else (b, gg, -1, -1, False)


def conv_key(bn, ktot, mode, act, win, stride, pre):
    b = {256: 128, 192: 96}.get(bn, bn)
    return ("conv", b, ktot // 64 >= 8, mode, act if mode == ops.CONV_LINEAR else 0, win, stride, pre)


L_, ZR, Q, LN = ops.CONV_LINEAR, ops.CONV_GRU_ZR, ops.CONV_GRU_Q, ops.CONV_LN
A0, RELU, TANH, SIG, GELU = ops.ACT_NONE, ops.ACT_RELU, ops.ACT_TANH, ops.ACT_SIGMOID, ops.ACT_GELU
CONV_EDGE = [
    # name, cins, cout, k (kh, kw), bn, mode, act, (h, w), stride, pre, batch, act scale, repeats
    ("lin128_g1_none", [128], 128, (1, 1), 128, L_, A0, (20, 33), 1, False, 2, 1.0, 1),
    ("lin128_g1_relu", [128], 256, (1, 1), 256, L_, RELU, (20, 33), 1, False, 2, 1.0, 1),
    ("lin128_g1_gelu", [128, 128], 512, (1, 1), 128, L_, GELU, (24, 16), 1, False, 1, 1.0, 1),
    ("ln128_g1", [128], 128, (1, 1), 128, LN, 0, (40, 16), 1, False, 1, 1.0, 1),
    ("ln128_g2", [1024], 128, (1, 1), 128, LN, 0, (24, 16), 1, False, 1, 1.0, 1),
    ("lin128_g2_none", [256], 128, (3, 3), 128, L_, A0, (20, 33), 1, False, 2, 1.0, 1),
    ("lin128_g2_relu", [256], 256, (3, 3), 256, L_, RELU, (20, 33), 1, False, 1, 1.0, 1),
    ("zr128_g2", [128, 256], 256, (1, 5), 128, ZR, 0, (12, 40), 1, False, 2, 1.0, 1),
    ("q128_g2", [128, 256], 128, (5, 1), 128, Q, 0, (24, 16), 1, False, 2, 1.0, 1),
    ("zr128_g2_pre", [128], 256, (1, 5), 256, ZR, 0, (12, 40), 1, True, 2, 1.0, 1),
    ("q128_g2_pre", [128], 128, (5, 1), 128, Q, 0, (24, 16), 1, True, 2, 1.0, 1),
    ("lin96_g2_relu", [256], 192, (3, 3), 96, L_, RELU, (20, 33), 1, False, 1, 1.0, 1),
    ("lin64_g4_none", [128], 64, (3, 3), 64, L_, A0, (20, 33), 1, False, 2, 1.0, 1),
    ("lin64_g4_relu", [128], 64, (3, 3), 64, L_, RELU, (20, 33), 1, False, 2, 1.0, 1),
    # run-time-mode instantiations
    ("rt128_g1_tanh", [128], 128, (1, 1), 128, L_, TANH, (20, 33), 1, False, 2, 1.0, 1),
    ("rt128_g1_sigmoid", [128], 128, (1, 1), 128, L_, SIG, (20, 33), 1, False, 2, 1.0, 1),
    ("rt128_g1_zr", [128], 256, (1, 1), 128, ZR, 0, (20, 33), 1, False, 2, 1.0, 1),
    ("rt128_g2_sigmoid", [512], 128, (1, 1), 128, L_, SIG, (20, 33), 1, False, 2, 1.0, 1),
    ("rt128_g2_gelu", [512], 256, (1, 1), 256, L_, GELU, (20, 33), 1, False, 1, 1.0, 1),
    ("rt128_g2_tanh", [128], 128, (3, 3), 128, L_, TANH, (20, 33), 1, False, 1, 1.0, 1),
    ("rt96_g1_relu", [128], 96, (1, 1), 96, L_, RELU, (20, 33), 1, False, 2, 1.0, 1),
    ("rt96_g2_tanh", [256], 96, (3, 3), 96, L_, TANH, (20, 33), 1, False, 1, 1.0, 1),
    ("rt96_g2_none", [256], 192, (3, 3), 192, L_, A0, (20, 33), 1, False, 1, 1.0, 1),
    ("rt64_g1_relu", [128], 64, (1, 1), 64, L_, RELU, (20, 33), 1, False, 2, 1.0, 1),
    ("rt64_g1_none", [64], 64, (1, 1), 64, L_, A0, (20, 33), 1, False, 2, 1.0, 1),
    ("rt96_g1_none", [64], 96, (1, 1), 96, L_, A0, (20, 33), 1, False, 2, 1.0, 1),
    ("rt64_g4_sigmoid", [128], 64, (3, 3), 64, L_, SIG, (20, 33), 1, False, 2, 1.0, 1),
    ("rt16_g1_none", [128], 2, (3, 1), 16, L_, A0, (20, 33), 1, False, 2, 1.0, 1),
    ("rt16_g4_flow_head", [256], 2, (3, 3), 16, L_, A0, (20, 33), 1, False, 2, 1.0, 1),
    # strides
    ("stride2_3x3", [64], 96, (3, 3), 128, L_, A0, (32, 48), 2, False, 2, 1.0, 1),
    ("stride2_1x1", [64], 96, (1, 1), 128, L_, A0, (32, 48), 2, False, 2, 1.0, 1),
    ("stride4_3x3", [64], 64, (3, 3), 64, L_, RELU, (64, 96), 4, False, 2, 1.0, 1),
    ("stride8_1x1", [64], 128, (1, 1), 128, L_, A0, (128, 136), 8, False, 1, 1.0, 1),
    # persistent CTAs over many tiles, repeated (staging-buffer ring / barrier phases)
    ("persistent_g1", [128], 640, (1, 1), 128, L_, A0, (400, 16), 1, False, 1, 1.0, 3),
    ("persistent_g2", [256], 128, (3, 3), 128, L_, RELU, (160, 128), 1, False, 1, 1.0, 3),
    ("persistent_g4", [128], 64, (3, 3), 64, L_, A0, (152, 64), 1, False, 2, 1.0, 3),
    # operand magnitudes: activations x 2^-8 ... 2^8 with fan-in weights
    ("mag_2^-8", [128], 128, (3, 3), 128, L_, A0, (20, 33), 1, False, 1, 2.0 ** -8, 1),
    ("mag_2^-4", [128], 128, (1, 1), 128, L_, A0, (20, 33), 1, False, 1, 2.0 ** -4, 1),
    ("mag_2^4", [128], 128, (1, 1), 128, L_, A0, (20, 33), 1, False, 1, 2.0 ** 4, 1),
    ("mag_2^8", [128], 128, (3, 3), 128, L_, A0, (20, 33), 1, False, 1, 2.0 ** 8, 1),
]


@pytest.mark.parametrize("name,cins,cout,ks,bn,mode,act,hw,stride,pre,b,scale,reps", CONV_EDGE)
def test_conv2d_tc_edges(name, cins, cout, ks, bn, mode, act, hw, stride, pre, b, scale, reps):
    """Ragged pixel tiles (20 x 33 is 2 x 3 tiles of 8 x 16, both partial), outputs at channel offsets 4 (fp32) and 64
    (split planes), against ref64.conv64."""
    h, w = hw
    kh, kw = ks
    gen = g(zlib.crc32(name.encode()) % 10000)
    cin = sum(cins) + (128 if pre else 0)
    wt = torch.randn((cout, cin, kh, kw), generator=gen) * (2.0 / (cin * kh * kw)) ** 0.5
    bias = torch.randn(cout, generator=gen) * 0.1 * scale
    xs = [torch.randn((b, h, w, c), generator=gen) * scale for c in ([128] + cins if pre else cins)]
    hh = torch.tanh(torch.randn((b, h, w, 128), generator=gen))
    zz = torch.sigmoid(torch.randn((b, h, w, 128), generator=gen))
    gamma, beta = torch.randn(128, generator=gen), torch.randn(128, generator=gen)
    pad = (kh // 2, kw // 2)
    bb = None if mode == LN else bias
    res = torch.randn((b, h, w, 128), generator=gen) if mode == LN else None
    aux0 = hh if mode in (ZR, Q) else res
    ref, bnd = ref64.conv64(xs, wt, bb, pad, stride, mode, act, aux0=aux0, aux1=zz if mode == Q else None, gamma=gamma,
                            beta=beta)
    dev = "cuda"
    pre_t = None
    if pre:                                                  # the first 128 input channels (+ bias) as a pre-accumulated input
        wfix = ops.prep_conv_weight(wt[:, :128].contiguous(), [128], cout)
        s_fix = torch.zeros((2, b, h, w, 128), dtype=torch.float16, device=dev)
        OPS.split_planes(xs[0].to(dev), s_fix, 0)
        pre_t = torch.zeros((b, h, w, cout), device=dev)
        OPS.conv2d_tc(s_fix, None, wfix.to(dev), bias.to(dev), kh, kw, pad[0], pad[1], cout, cout, L_, A0, pre_t, 0, None, 0,
                      None, None)
        xs_k, wt_k, bias_k = xs[1:], wt[:, 128:].contiguous(), None
    else:
        xs_k, wt_k, bias_k = xs, wt, bb
    cout_p = (cout + bn - 1) // bn * bn
    wp = ops.prep_conv_weight(wt_k, [x.shape[-1] for x in xs_k], cout_p).to(dev)
    srcs = []
    for x in xs_k:
        buf = torch.zeros((2, b, h, w, (x.shape[-1] + 63) // 64 * 64), dtype=torch.float16, device=dev)
        OPS.split_planes(x.to(dev), buf, 0)
        srcs.append(buf)
    ho, wo = ref.shape[1], ref.shape[2]
    zr = mode == ZR
    co_f = 128 if zr else cout
    off_f, off_s = (0, 0) if zr else (4, 64)
    loc = ref64.conv_locator({256: 128, 192: 96}.get(bn, bn))
    for rep in range(reps):
        out_f = torch.zeros((b, ho, wo, co_f + off_f + (4 if not zr else 0)), device=dev)
        out_s = torch.zeros((2, b, ho, wo, (co_f + off_s + 63) // 64 * 64 + 64), dtype=torch.float16, device=dev)
        OPS.conv2d_tc(srcs[0], srcs[1] if len(srcs) > 1 else None, wp, None if bias_k is None else bias_k.to(dev), kh, kw,
                      pad[0], pad[1], cout, bn, mode, act, out_f, off_f, out_s, off_s, None if aux0 is None else aux0.to(dev),
                      zz.to(dev) if mode == Q else None, gamma.to(dev) if mode == LN else None,
                      beta.to(dev) if mode == LN else None, stride, 0, None, None, 0, 0, 0, pre_t)
        got_f = out_f.cpu()
        got_s = (out_s[0].double() + out_s[1].double()).cpu()
        tag = "%s%s" % (name, " rep %d" % rep if reps > 1 else "")
        if zr:
            ref64.check(tag + " z", got_f, ref[..., :128], bnd[..., :128], loc)
            ref64.check(tag + " r*h split", got_s[..., :128], ref[..., 128:],
                        ref64.split_out_bound(ref[..., 128:], bnd[..., 128:]), loc)
        else:
            ref64.check(tag + " f32", got_f[..., off_f:off_f + cout], ref, bnd, loc)
            ref64.check(tag + " split", got_s[..., off_s:off_s + cout], ref, ref64.split_out_bound(ref, bnd), loc)
            assert got_f[..., :off_f].abs().max() == 0 and got_f[..., off_f + cout:].abs().max() == 0
            assert got_s[..., :off_s].abs().max() == 0 and got_s[..., off_s + cout:].abs().max() == 0


def test_conv2d_tc_window_plane_output_edge():
    """The window-plane instantiation: a 128 -> 384 projection writing q / k / v straight into the attention's planes."""
    gen = g(8100)
    n, h, w, K = 2, 30, 52, 2
    rows = n * h * w
    x = torch.randn((rows, C), generator=gen)
    wt = torch.randn((384, C, 1, 1), generator=gen) * (2.0 / C) ** 0.5
    wh_, ww_ = h // K, w // K
    sh, sw = wh_ // 2, ww_ // 2
    geom = (h, w, K, K, sh, sw, ops.MASK_SWIN)
    lp = ops.attention_planes_lp(*geom)
    src = torch.zeros((2, rows, C), dtype=torch.float16).cuda()
    OPS.split_planes(x.cuda(), src, 0)
    wd = torch.zeros((3, 2, n, K * K, lp, C), dtype=torch.float16).cuda()
    OPS.conv2d_tc(src, None, ops.prep_conv_weight(wt, [C], 384).cuda(), None, 1, 1, 0, 0, 384, 128, L_, A0, None, 0, None, 0,
                  None, None, None, None, 1, rows, wd, geom, 0, 384, n)
    ref, bnd = ref64.conv64([x.view(1, rows // 16, 16, C)], wt)
    ref, bnd = ref.view(n, h * w, 384), bnd.view(n, h * w, 384)
    tok, _ = ref64.window_layout(h, w, K, K, sh, sw)
    got = (wd[:, 0].double() + wd[:, 1].double()).cpu()                     # [3, n, nwin, lp, 128]
    lw = tok.shape[1]
    for o in range(3):
        r = ref[..., 128 * o:128 * (o + 1)][:, tok.reshape(-1)].view(n, K * K, lw, C)
        e = bnd[..., 128 * o:128 * (o + 1)][:, tok.reshape(-1)].view(n, K * K, lw, C)
        ref64.check("window planes op %d" % o, got[o, :, :, :lw], r, ref64.split_out_bound(r, e))
    assert got[:, :, :, lw:].abs().max() == 0                               # window padding rows untouched


# ---- fused FFN -------------------------------------------------------------------------------------------------------
FFN_F64 = [(256, 128), (512, 1024), (256 * 77, 1024), (256 * 150, 256), (1024, 1024)]     # (rows, hidden)


@pytest.mark.parametrize("rows,hidden", FFN_F64)
def test_ffn_tc_vs_float64(rows, hidden):
    gen = g(9000 + rows % 997 + hidden)
    w1 = torch.randn((hidden, 256, 1, 1), generator=gen) * (2.0 / 256) ** 0.5
    w2 = torch.randn((128, hidden, 1, 1), generator=gen) * (1.0 / hidden) ** 0.5
    xs = [torch.randn((rows, 128), generator=gen) for _ in range(2)]
    res = torch.randn((rows, 128), generator=gen)
    gamma, beta = torch.randn(128, generator=gen), torch.randn(128, generator=gen)
    srcs = []
    for x in xs:
        buf = torch.zeros((2, rows, 128), dtype=torch.float16).cuda()
        OPS.split_planes(x.cuda(), buf, 0)
        srcs.append(buf)
    out_f = torch.zeros((rows, 128)).cuda()
    out_s = torch.zeros((2, rows, 128), dtype=torch.float16).cuda()
    OPS.ffn_tc(srcs[0], srcs[1], ops.prep_conv_weight(w1, [128, 128], hidden).cuda(),
               ops.prep_conv_weight(w2, [hidden], 128).cuda(), res.cuda(), gamma.cuda(), beta.cuda(), out_f, out_s, rows)
    sel = torch.arange(rows) if rows <= 1024 else torch.cat((torch.arange(256), torch.arange(rows - 256, rows),
                                                             torch.randperm(rows, generator=gen)[:512])).unique()
    ref, bnd = ref64.ffn64(xs[0][sel], xs[1][sel], w1, w2, res[sel], gamma, beta)
    ref64.check("ffn %d x %d f32" % (rows, hidden), out_f.cpu()[sel], ref, bnd)
    ref64.check("ffn %d x %d split" % (rows, hidden), (out_s[0].double() + out_s[1].double()).cpu()[sel], ref,
                ref64.split_out_bound(ref, bnd))


# ---- instance norm ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ratio", [0.0, 10.0, 100.0])
@pytest.mark.parametrize("c", [64, 96, 128])
def test_instance_norm_stats_large_maps(c, ratio):
    """The backbone's first-stage maps (240 x 416 pixels) with |mean| / std up to 100: rstd to 1e-6 relative, the mean
    within fp32 rounding."""
    gen = g(9500 + c + int(ratio))
    n, h, w = 2, 240, 416
    std = torch.rand((n, 1, 1, c), generator=gen) * 2 + 0.25
    sign = torch.where(torch.rand((n, 1, 1, c), generator=gen) < 0.5, -1.0, 1.0)
    x = sign * ratio * std + std * torch.randn((n, h, w, c), generator=gen)
    mean, rstd, sd = ref64.instance_norm_stats64(x)
    st = OPS.instance_norm_stats(x.cuda()).double().cpu()
    ref64.check("instance norm rstd c %d ratio %g" % (c, ratio), st[:, 1], rstd, 1e-6 * rstd)
    ref64.check("instance norm mean c %d ratio %g" % (c, ratio), st[:, 0], mean, 2.0 ** -24 * mean.abs() + 2.0 ** -22 * sd)


# ---- launch census ---------------------------------------------------------------------------------------------------
def _expect_tc(h, w, kh, kw, mask, n_total, value_mode):
    g_ = ops.AttnGeom(h, w, kh, kw, 0, 0, mask)
    import ctypes
    return ops.LIB.um_softmax_expectation_workspace(ctypes.byref(g_), n_total, value_mode) > 0


def _attn_class(h, w, kh, kw, sh, sw):
    shape = "full2d" if kh == 1 and kw == 1 else "full1d" if (kh == h and kw == 1) else "swin1d" if kh == h else "swin2d"
    return shape + ("_shifted" if sh or sw else "")


def attn_key(h, w, kh, kw, sh, sw, mask):
    return ("attn", ops.attention_planes_lp(h, w, kh, kw, sh, sw, mask) > 0, _attn_class(h, w, kh, kw, sh, sw))


def expect_key(h, w, kh, kw, mask, n_total, value_mode):
    return ("expect", _expect_tc(h, w, kh, kw, mask, n_total, value_mode), value_mode, mask)


def covered_keys():
    keys = set()
    for name, cins, cout, ks, bn, mode, act, hw, stride, pre, *_ in CONV_EDGE:
        ktot = sum((c + 63) // 64 * 64 for c in cins) * ks[0] * ks[1]
        keys.add(conv_key(bn, ktot, mode, act, False, stride, pre))
    keys.add(conv_key(128, 128, L_, A0, True, 1, False))                    # test_conv2d_tc_window_plane_output_edge
    for name, n, h, w, kh, kw, shift, *_ in ATTN_EDGE:
        sh, sw, mask = _geom(h, w, kh, kw, shift)
        keys.add(attn_key(h, w, kh, kw, sh, sw, mask))
    for name, nt, ns, kvs, h, w, vdim, vm, post, kh, kw, mask, _ in EXP_EDGE:
        keys.add(expect_key(h, w, kh, kw, mask, nt, vm))
    return keys | M.covered_keys()                                          # tests/test_matching_edges_gpu.py


def test_case_tables_reach_every_conv_instantiation():
    inst = set()
    for name, cins, cout, ks, bn, mode, act, *_ in CONV_EDGE:
        inst.add(conv_dispatch(bn, sum((c + 63) // 64 * 64 for c in cins) * ks[0] * ks[1], mode, act, False))
    inst.add(conv_dispatch(128, 128, L_, A0, True))
    table = {k + (False,) for k in FIXED} | {(b, gg, -1, -1, False) for b in (128, 96, 64, 16) for gg in (1, {128: 2, 96: 2}.get(b, 4))}
    table.add((128, 1, 0, 0, True))
    assert table <= inst, sorted(table - inst)


class _Census:
    """Stands in for torch.ops.unimatch_sm100 in unimatch_b200.unimatch: records the dispatch key of every launch and
    delegates to the real op."""

    def __init__(self, real):
        self.real, self.keys = real, set()
        self.conv_sig = inspect.signature(ops._conv2d_tc)

    def __getattr__(self, name):
        fn = getattr(self.real, name)
        rec = getattr(self, "_key_" + name, None)
        if rec is None:
            return fn

        def wrapped(*a, **kw):
            self.keys.add(rec(*a, **kw))
            return fn(*a, **kw)
        return wrapped

    def _key_conv2d_tc(self, *a, **kw):
        b = self.conv_sig.bind(*a, **kw)
        b.apply_defaults()
        p = b.arguments
        ktot = sum(s.shape[-1] for s in (p["src0"], p["src1"]) if s is not None) * p["kh"] * p["kw"]
        return conv_key(p["bn"], ktot, p["mode"], p["act"], p["win_dst"] is not None, p["stride"], p["pre"] is not None)

    def _key_window_attention(self, q, k, v, kvs, h, w, kh, kw, sh, sw, mask):
        return attn_key(h, w, kh, kw, sh, sw, mask)

    def _key_window_attention_planes(self, qp, kp, vp, n, kvs, h, w, kh, kw, sh, sw, mask, *rest):
        return attn_key(h, w, kh, kw, sh, sw, mask)

    def _key_softmax_expectation(self, q, k, values, ns, kvs, vdim, vm, post, h, w, kh, kw, mask):
        return expect_key(h, w, kh, kw, mask, q.shape[0], vm)

    def _key_local_corr_softmax(self, f0, f1, h, w, ry, rx, stereo):
        return M.lcs_key(ry, rx, stereo)

    def _key_local_corr_volume(self, f0, f1, flow, h, w, radius):
        return M.corr_volume_key(flow.shape[-1])

    def _key_flow_warp(self, f, flow, h, w):
        return M.flow_warp_key(flow.shape[-1])

    def _key_propagate_local(self, q, k, flow, h, w, radius):
        return M.propagate_key(radius, q.stride(-2), k.stride(-2), flow.shape[-1])

    def _key_depth_corr_softmax(self, f0, f1, K, Kinv, pose, cand, h, w, from_argmax):
        return M.depth_key(cand.numel(), from_argmax)

    def _key_convex_upsample(self, flow, mask, factor, mult):
        return M.convex_key(factor, flow.shape[-1], mult)

    def _key_upsample2x(self, flow, mult):
        return M.upsample2x_key(flow.shape[-1])

    def _key_add_position(self, x, table, h, w):
        return M.add_position_key()

    def _key_conv7x7_small(self, in0, in1, nchw, weight, bias, stride, relu, scale, shift, out_f32, out_split):
        return M.conv7x7_key(weight.shape[1], stride, nchw, in1 is not None, scale is not None, out_f32 is not None,
                             out_split is not None)


CENSUS_RES = {"flow": (480, 832), "stereo": (544, 960), "depth": (384, 512)}


def test_launch_census_of_bench_workloads(monkeypatch):
    """One pair of every workload in spec.WORKLOADS at its real resolution; every conv / attention / expectation /
    matching-path dispatch key it launches must be one the case tables here or in tests/test_matching_edges_gpu.py test."""
    import unimatch_b200.unimatch as um
    from unimatch_b200.spec import WORKLOADS
    from unimatch_b200.synthetic import synthetic_batch, synthetic_model
    census = _Census(um._OPS)
    monkeypatch.setattr(um, "_OPS", census)
    for wl, cfg in WORKLOADS.items():
        H, W = CENSUS_RES[cfg["model"]["task"]]
        model = synthetic_model(wl)
        inp = {k: v.cuda() for k, v in synthetic_batch(cfg["model"]["task"], 1, H, W).items()}
        with torch.no_grad():
            model(inp["img0"], inp["img1"], intrinsics=inp.get("intrinsics"), pose=inp.get("pose"), **cfg["call"])
        torch.cuda.synchronize()
        print("census: ran", wl, H, W)
    for key in sorted(census.keys, key=str):
        print("census:", key)
    missing = census.keys - covered_keys()
    assert not missing, "launch configurations without an edge case: %s" % sorted(missing, key=str)
