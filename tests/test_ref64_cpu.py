"""The float64 references of tests/ref64.py and their error bounds, checked on the CPU:
  * they agree with the fp32 oracle statements of tests/refops.py (within the bound);
  * an emulation of the kernels' arithmetic (fp16 (hi, lo) split, hi*hi + hi*lo + lo*hi, fp32 accumulation, online softmax
    over 64-key tiles with the lazy rescale, P split into (hi, lo)) passes the bounds;
  * the same emulation with one defect injected fails them.  This is what makes the GPU edge suite able to catch a subtly
    wrong kernel."""
import math

import numpy as np
import pytest
import torch

import ref64
import refops
from unimatch_b200 import ops

C = 128
EXP_SCALE = 1.4426950408889634 / math.sqrt(C)
LAZY_THRESH = 8.0 / EXP_SCALE                      # raw-logit units, as in um_attention_tc.cu


def g(seed):
    return torch.Generator().manual_seed(seed)


def hl(x):
    x = x.float()
    hi = x.half().float()
    return hi, (x - hi).half().float()


def rejects(name, got, ref, bound, locate=None):
    with pytest.raises(AssertionError):
        ref64.check(name, got, ref, bound, locate)


# ---- convolution ----------------------------------------------------------------------------------------------------
def emu_conv(x, wt, bias, pad, stride, defect=None):
    """fp32 emulation of um_conv2d_tc's products on channel-last x: lo*hi + hi*lo + hi*hi."""
    xh, xl = hl(x.permute(0, 3, 1, 2))
    wh, wl = hl(wt)
    F = torch.nn.functional
    c = lambda a, b: F.conv2d(a, b, None, stride=stride, padding=pad)
    if defect == "hi_only":
        y = c(xh, wh)
    elif defect == "drop_hi_lo":
        y = c(xl, wh) + c(xh, wh)
    else:
        y = c(xl, wh) + c(xh, wl) + c(xh, wh)
    y = y.permute(0, 2, 3, 1)
    return y + bias if bias is not None else y


CONV_CPU_CASES = [
    # cins, cout, k, stride, scale
    ([128], 128, 1, 1, 1.0),
    ([256], 64, 3, 1, 1.0),
    ([64], 96, 3, 2, 1.0),
    ([128], 64, 3, 1, 2.0 ** -8),          # small activations: fp16 subnormal lo parts
    ([128], 64, 1, 1, 2.0 ** 8),
]


def _conv_inputs(cins, cout, k, scale, seed):
    gen = g(seed)
    cin = sum(cins)
    xs = [torch.randn((2, 12, 20, c), generator=gen) * scale for c in cins]
    wt = torch.randn((cout, cin, k, k), generator=gen) * (2.0 / (cin * k * k)) ** 0.5
    bias = torch.randn(cout, generator=gen) * 0.1 * scale
    return xs, wt, bias


@pytest.mark.parametrize("cins,cout,k,stride,scale", CONV_CPU_CASES)
def test_conv64_matches_oracle_and_emulation(cins, cout, k, stride, scale):
    xs, wt, bias = _conv_inputs(cins, cout, k, scale, 10 + cout + k)
    ref, bnd = ref64.conv64(xs, wt, bias, (k // 2, k // 2), stride)
    x = torch.cat(xs, -1)
    oracle = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2), wt, bias, stride=stride, padding=k // 2).permute(0, 2, 3, 1)
    ref64.check("conv oracle %s" % ((cins, cout, k, stride, scale),), oracle, ref, bnd)
    ref64.check("conv emulation %s" % ((cins, cout, k, stride, scale),), emu_conv(x, wt, bias, k // 2, stride), ref, bnd)


@pytest.mark.parametrize("defect", ["hi_only", "drop_hi_lo"])
@pytest.mark.parametrize("cins,cout,k", [([128], 128, 1), ([256], 64, 3)])
def test_conv64_rejects_split_defects(defect, cins, cout, k):
    xs, wt, bias = _conv_inputs(cins, cout, k, 1.0, 20 + cout)
    ref, bnd = ref64.conv64(xs, wt, bias, (k // 2, k // 2), 1)
    rejects("conv %s" % defect, emu_conv(torch.cat(xs, -1), wt, bias, k // 2, 1, defect), ref, bnd, ref64.conv_locator(128))


@pytest.mark.parametrize("mode", ["zr", "q", "ln", "lin_pre"])
def test_conv64_epilogues_match_refops(mode):
    """GRU_ZR / GRU_Q / LayerNorm(+residual) epilogues and the pre-accumulated input against tests/refops.py."""
    gen = g(40 + len(mode))
    b, h, w = 1, 6, 20
    cout = 256 if mode == "zr" else 128
    wt = torch.randn((cout, 128, 1, 3), generator=gen) * (2.0 / 384) ** 0.5
    bias = torch.randn(cout, generator=gen) * 0.1
    x = torch.randn((b, h, w, 128), generator=gen)
    hh = torch.tanh(torch.randn((b, h, w, 128), generator=gen))
    zz = torch.sigmoid(torch.randn((b, h, w, 128), generator=gen))
    gamma, beta = torch.randn(128, generator=gen), torch.randn(128, generator=gen)
    pre = torch.randn((b, h, w, cout), generator=gen) if mode == "lin_pre" else None
    m = {"zr": ops.CONV_GRU_ZR, "q": ops.CONV_GRU_Q, "ln": ops.CONV_LN, "lin_pre": ops.CONV_LINEAR}[mode]
    act = ops.ACT_GELU if mode == "lin_pre" else 0
    bb = None if mode == "ln" else bias
    ref, bnd = ref64.conv64([x], wt, bb, (0, 1), 1, m, act, aux0=hh if mode in ("zr", "q", "ln") else None,
                            aux1=zz if mode == "q" else None, gamma=gamma, beta=beta, pre=pre)
    wp = ops.prep_conv_weight(wt, [128], cout)
    src = torch.zeros((2, b, h, w, 128), dtype=torch.float16)
    refops.split_planes(x, src, 0)
    out_f = torch.zeros((b, h, w, 128 if mode == "zr" else cout))
    out_s = torch.zeros((2, b, h, w, 128 if mode == "zr" else cout), dtype=torch.float16)
    refops.conv2d_tc(src, None, wp, bb, 1, 3, 0, 1, cout, 128, m, act, out_f, 0, out_s, 0,
                     hh if mode in ("zr", "q", "ln") else None, zz if mode == "q" else None, gamma, beta, pre=pre)
    got_s = out_s[0].double() + out_s[1].double()
    if mode == "zr":
        ref64.check("zr z", out_f, ref[..., :128], bnd[..., :128])
        ref64.check("zr r*h", got_s, ref[..., 128:], ref64.split_out_bound(ref[..., 128:], bnd[..., 128:]))
    else:
        ref64.check(mode, out_f, ref, bnd)
        ref64.check(mode + " split", got_s, ref, ref64.split_out_bound(ref, bnd))


def test_ffn64_matches_refops():
    gen = g(50)
    rows, hidden = 256, 512
    w1 = torch.randn((hidden, 256, 1, 1), generator=gen) * (2.0 / 256) ** 0.5
    w2 = torch.randn((128, hidden, 1, 1), generator=gen) * (1.0 / hidden) ** 0.5
    xs = [torch.randn((rows, 128), generator=gen) for _ in range(2)]
    res = torch.randn((rows, 128), generator=gen)
    gamma, beta = torch.randn(128, generator=gen), torch.randn(128, generator=gen)
    ref, bnd = ref64.ffn64(xs[0], xs[1], w1, w2, res, gamma, beta)
    srcs = []
    for x in xs:
        buf = torch.zeros((2, rows, 128), dtype=torch.float16)
        refops.split_planes(x, buf, 0)
        srcs.append(buf)
    out = torch.zeros((rows, 128))
    refops.ffn_tc(srcs[0], srcs[1], ops.prep_conv_weight(w1, [128, 128], hidden), ops.prep_conv_weight(w2, [hidden], 128),
                  res, gamma, beta, out, None, rows)
    ref64.check("ffn vs refops", out, ref, bnd)


# ---- window attention -----------------------------------------------------------------------------------------------
def emu_attention(q, k, v, kv_shift, h, w, kh, kw, sh, sw, mask_mode, defect=None):
    """fp32 emulation of attn_tc_kernel: split logits, -100*sqrt(C) Swin mask, 64-key tiles with the lazy rescale,
    P split into (hi, lo) for P V, O / l at the end."""
    n = q.shape[0]
    tok, reg = ref64.window_layout(h, w, kh, kw, sh, sw)
    if defect == "mask_band":
        _, reg = ref64.window_layout(h, w, kh, kw, sh, max(sw - 1, 1) if sw else 0)
        if sh:
            _, reg = ref64.window_layout(h, w, kh, kw, max(sh - 1, 1), sw)
    nwin, lw = tok.shape
    out = torch.zeros((n, h * w, C))
    T = (lw + 63) // 64
    for s_ in range(n):
        ks = (s_ + kv_shift) % n
        for wi in range(nwin):
            t = tok[wi]
            qh, ql = hl(q[s_, t])
            kh_, kl = hl(k[ks, t])
            vh, vl = hl(v[ks, t])
            if defect == "hi_only":
                s = qh @ kh_.T
            elif defect == "drop_hi_lo":
                s = ql @ kh_.T + qh @ kh_.T
            else:
                s = ql @ kh_.T + qh @ kl.T + qh @ kh_.T
            if mask_mode == ops.MASK_SWIN:
                s = torch.where(reg[wi][:, None] != reg[wi][None, :], s - np.float32(100.0 * math.sqrt(C)), s)
            m = torch.full((lw, 1), -math.inf)
            l = torch.zeros((lw, 1))
            o = torch.zeros((lw, C))
            for j in range(T):
                if defect == "skip_last_tile" and j == T - 1 and lw % 64:
                    break
                sj = s[:, 64 * j:64 * (j + 1)]
                mx = sj.max(-1, keepdim=True).values
                grow = mx > m + LAZY_THRESH
                alpha = torch.where(grow, torch.exp2((m - mx) * np.float32(EXP_SCALE)), torch.ones_like(m))
                m = torch.where(grow, mx, m)
                if defect != "no_alpha":
                    o = o * alpha
                p = torch.exp2(sj * np.float32(EXP_SCALE) - m * np.float32(EXP_SCALE))
                l = l * alpha + p.sum(-1, keepdim=True)
                ph, pl = hl(p)
                vj_h, vj_l = vh[64 * j:64 * (j + 1)], vl[64 * j:64 * (j + 1)]
                if defect == "hi_only":
                    o = o + ph @ vj_h
                else:
                    o = o + pl @ vj_h + ph @ vj_l + ph @ vj_h
            dst = t if defect != "token_off_by_one" else torch.roll(t, 1)
            out[s_, dst] = o / l
    return out


ATTN_CPU_CASES = [
    # name, n, h, w, kh, kw, shift, kv_shift
    ("lw128_full", 2, 8, 16, 1, 1, False, 1),
    ("lw129_full", 1, 3, 43, 1, 1, False, 0),
    ("lw192_full", 2, 12, 16, 1, 1, False, 1),
    ("swin2d_lw128_first_tile_masked", 1, 32, 16, 2, 2, True, 0),
    ("swin1d_lw160_shifted", 2, 2, 320, 2, 2, True, 1),
    ("full1d_rows_lw156", 2, 3, 156, 3, 1, False, 1),
    ("three_streams", 3, 8, 24, 1, 1, False, 2),
]


def _geom(h, w, kh, kw, shift):
    wh, ww = h // kh, w // kw
    sh = (wh // 2 if kh != h else 0) if shift else 0
    sw = ww // 2 if shift else 0
    return sh, sw, ops.MASK_SWIN if shift else ops.MASK_NONE


def _qkv(n, L, seed, scale=1.5):
    gen = g(seed)
    return [torch.randn((n, L, C), generator=gen) * sc for sc in (scale, scale, 1.0)]


@pytest.mark.parametrize("name,n,h,w,kh,kw,shift,kvs", ATTN_CPU_CASES)
def test_attention64_matches_oracle_and_emulation(name, n, h, w, kh, kw, shift, kvs):
    sh, sw, mask = _geom(h, w, kh, kw, shift)
    q, k, v = _qkv(n, h * w, 60 + h * w)
    ref, bnd, loc = ref64.attention64(q, k, v, kvs, h, w, kh, kw, sh, sw, mask)
    if not (kh == h and kw > 1 and shift and h > 1):      # (the oracle's 1-D shifted form needs kh == h)
        ref64.check(name + " oracle", refops.window_attention(q, k, v, kvs, h, w, kh, kw, sh, sw, mask), ref, bnd, loc)
    r = ref64.check(name + " emulation", emu_attention(q, k, v, kvs, h, w, kh, kw, sh, sw, mask), ref, bnd, loc)
    assert r < 0.5                                        # headroom for the GPU's truncating accumulation


@pytest.mark.parametrize("defect,case", [
    ("hi_only", "lw192_full"), ("drop_hi_lo", "lw192_full"), ("skip_last_tile", "lw129_full"),
    ("token_off_by_one", "lw128_full"), ("mask_band", "swin2d_lw128_first_tile_masked"),
    ("mask_band", "swin1d_lw160_shifted")])
def test_attention64_rejects_defects(defect, case):
    name, n, h, w, kh, kw, shift, kvs = next(c for c in ATTN_CPU_CASES if c[0] == case)
    sh, sw, mask = _geom(h, w, kh, kw, shift)
    q, k, v = _qkv(n, h * w, 60 + h * w)
    ref, bnd, loc = ref64.attention64(q, k, v, kvs, h, w, kh, kw, sh, sw, mask)
    rejects(name + " " + defect, emu_attention(q, k, v, kvs, h, w, kh, kw, sh, sw, mask, defect), ref, bnd, loc)


def lazy_logits(n, h, w, grow, tile, seed):
    """q, k, v of full attention (window = whole map) whose scaled logits are small in the first key tile and jump by
    `grow` raw-logit units at one key of key tile `tile` for every query."""
    gen = g(seed)
    L = h * w
    q = torch.randn((n, L, C), generator=gen) * 0.3
    k = torch.randn((n, L, C), generator=gen) * 0.3
    v = torch.randn((n, L, C), generator=gen)
    q[..., 0] = 16.0
    k[..., 0] = 0.0
    k[:, 64 * tile + 5, 0] = grow / 16.0
    return q, k, v


def test_lazy_rescale_threshold_and_missing_alpha():
    """The running max grows in a later key tile just under / just over LAZY_THRESH, and by ~60 scaled units in the last
    tile: the emulation passes; the one that forgets alpha on the P V accumulator fails."""
    for grow, tile in ((LAZY_THRESH - 0.5, 1), (LAZY_THRESH + 0.5, 1), (60.0 * math.sqrt(C), 2)):
        q, k, v = lazy_logits(1, 12, 16, grow, tile, 70 + tile)
        ref, bnd, loc = ref64.attention64(q, k, v, 0, 12, 16, 1, 1, 0, 0, ops.MASK_NONE)
        ref64.check("lazy grow %.1f tile %d" % (grow, tile), emu_attention(q, k, v, 0, 12, 16, 1, 1, 0, 0, 0), ref, bnd, loc)
        if grow > LAZY_THRESH:
            rejects("lazy no alpha", emu_attention(q, k, v, 0, 12, 16, 1, 1, 0, 0, 0, "no_alpha"), ref, bnd, loc)


def test_peaked_logits_emulation_passes():
    q, k, v = _qkv(1, 192, 80, scale=8.0)                 # scaled logits up to about +-200
    ref, bnd, loc = ref64.attention64(q, k, v, 0, 12, 16, 1, 1, 0, 0, ops.MASK_NONE)
    ref64.check("peaked", emu_attention(q, k, v, 0, 12, 16, 1, 1, 0, 0, 0), ref, bnd, loc)


EXP_CPU_CASES = [
    (4, 2, 2, 7, 9, 2, ops.VALUE_COORDS, ops.POST_MINUS_OWN, 1, 1, ops.MASK_NONE),
    (2, 1, 1, 3, 100, 1, ops.VALUE_XCOORD, ops.POST_OWN_MINUS, 3, 1, ops.MASK_CAUSAL),
    (2, 2, 0, 12, 30, 2, ops.VALUE_TENSOR, ops.POST_NONE, 1, 1, ops.MASK_NONE),
]


@pytest.mark.parametrize("nt,ns,kvs,h,w,vdim,vm,post,kh,kw,mask", EXP_CPU_CASES)
def test_expectation64_matches_oracle(nt, ns, kvs, h, w, vdim, vm, post, kh, kw, mask):
    gen = g(90 + h * w)
    L = h * w
    q = torch.randn((nt, L, C), generator=gen) * 1.5
    k = torch.randn((nt, L, C), generator=gen) * 1.5
    vals = torch.randn((nt, L, vdim), generator=gen) * 3 if vm == ops.VALUE_TENSOR else None
    ref, bnd = ref64.expectation64(q, k, vals, ns, kvs, vdim, vm, post, h, w, kh, kw, mask)
    ref64.check("expectation oracle", refops.softmax_expectation(q, k, vals, ns, kvs, vdim, vm, post, h, w, kh, kw, mask),
                ref, bnd)


# ---- instance norm --------------------------------------------------------------------------------------------------
def emu_in_stats(x, shifted):
    """fp32 per-lane sums in the order of in_partial_kernel (64 chunks x 16 row lanes, sequential per lane), combined in
    float64.  shifted: sums of x - pivot (pivot = fp32 mean of the first 16 pixels); otherwise E[x^2] - mean^2."""
    hw = x.shape[0]
    xs = x.astype(np.float32)
    piv = np.float32(0.0)
    if shifted:
        piv = np.float32(0.0)
        for i in range(min(16, hw)):
            piv = np.float32(piv + xs[i])
        piv = np.float32(piv / np.float32(min(16, hw)))
        xs = (xs - piv).astype(np.float32)
    rpc = (hw + 63) // 64
    s = q = 0.0
    for c0 in range(0, hw, rpc):
        chunk = xs[c0:c0 + rpc]
        for lane in range(16):
            v = chunk[lane::16]
            s += float(np.cumsum(v, dtype=np.float32)[-1]) if v.size else 0.0
            q += float(np.cumsum(v * v, dtype=np.float32)[-1]) if v.size else 0.0
    mean = s / hw
    var = max(q / hw - mean * mean, 0.0)
    return float(piv) + mean, 1.0 / math.sqrt(var + 1e-5)


@pytest.mark.parametrize("ratio", [0.0, 10.0, 100.0])
def test_instance_norm_stats_need_shifted_sums(ratio):
    """At hw = 240 x 416 and |mean| / std = 100, E[x^2] - mean^2 from fp32 sums loses the 1e-6 rstd target; sums of x minus a
    pivot keep it."""
    rng = np.random.default_rng(100 + int(ratio))
    std = 0.7
    x = (ratio * std + std * rng.standard_normal(240 * 416)).astype(np.float32)
    mean, rstd, _ = ref64.instance_norm_stats64(torch.from_numpy(x).view(1, -1, 1, 1))
    m_ok, r_ok = emu_in_stats(x, True)
    assert abs(r_ok / rstd.item() - 1) <= 1e-6 and abs(m_ok - mean.item()) <= 2.0 ** -23 * abs(mean.item()) + 1e-6 * std
    if ratio >= 100:
        _, r_bad = emu_in_stats(x, False)
        assert abs(r_bad / rstd.item() - 1) > 1e-6


# ---- matching-path kernels: fp32 emulations of um_local.cu / um_local_stencil.cu / um_misc.cu / um_stem.cu ---------
F32 = torch.float32
SQRT_C32 = torch.tensor(math.sqrt(C), dtype=F32)


def fma(a, b, c):
    """fmaf: the exact product plus c, rounded once to fp32."""
    return (a.double() * b.double() + c.double()).float()


def norm_window(p, size):
    c = torch.tensor(float(size - 1), dtype=F32) / 2.0
    return (p - c) / c


def norm_sample(p, size):
    return 2.0 * p / torch.tensor(float(size - 1), dtype=F32) - 1.0


def unnorm(g, size):
    return ((g + 1.0) / 2.0) * torch.tensor(float(size - 1), dtype=F32)


def emu_taps(img, b, ix, iy, defect=None):
    """sample() of um_local.cu on fp32 img [B, h, w, C] at fp32 positions [P, K]: make_tap weights, the four taps in ATen
    order as FMAs, zeros outside (defect "replicate": border taps clamped)."""
    h, w = img.shape[1], img.shape[2]
    fx, fy = torch.floor(ix), torch.floor(iy)
    x0, y0 = fx.long(), fy.long()
    xe, ye = fx + 1.0, fy + 1.0
    wts = ((xe - ix) * (ye - iy), (ix - fx) * (ye - iy), (xe - ix) * (iy - fy), (ix - fx) * (iy - fy))
    acc = torch.zeros(ix.shape + (img.shape[-1],), dtype=F32)
    bb = b.view(-1, *([1] * (ix.dim() - 1))).expand_as(x0)
    for wt, (dy, dx) in zip(wts, ((0, 0), (0, 1), (1, 0), (1, 1))):
        yy, xx = y0 + dy, x0 + dx
        ok = (yy >= 0) & (yy < h) & (xx >= 0) & (xx < w)
        if defect == "replicate":
            ok = torch.ones_like(ok)
        v = img[bb, yy.clamp(0, h - 1), xx.clamp(0, w - 1)]
        acc = torch.where(ok[..., None], fma(wt[..., None], v, acc), acc)
    return acc


def emu_dot8(a, v):
    """dot_partial + reduce8: lane `sub` chains 16 FMAs over channels sub*4 + 32 i + j, then three xor-shuffle adds.
    a [P, C], v [P, K, C] fp32 -> [P, K]."""
    va = v.view(*v.shape[:-1], 4, 8, 4)                                  # [.., i, sub, j]
    aa = a.view(a.shape[0], 1, 4, 8, 4).expand_as(va)
    s = torch.zeros(va.shape[:-3] + (8,), dtype=F32)
    for i in range(4):
        for j in range(4):
            s = fma(aa[..., i, :, j], va[..., i, :, j], s)
    for m in (4, 2, 1):
        s = s + s[..., torch.arange(8) ^ m]
    return s[..., 0]


def emu_online(logits, vals):
    """The kernels' online softmax over the taps in order: m, l and the value sums in fp32 with FMA rescales.
    logits [P, K], vals [P, K, d] -> (l, sums [P, d], m)."""
    P, K = logits.shape
    m = torch.full((P,), -math.inf)
    l = torch.zeros(P)
    acc = torch.zeros((P, vals.shape[-1]))
    for k in range(K):
        s = logits[:, k]
        mn = torch.maximum(m, s)
        al, p = torch.exp(m - mn), torch.exp(s - mn)
        l = fma(l, al, p)
        acc = fma(acc, al[:, None], (p[:, None] * vals[:, k]))
        m = mn
    return l, acc, m


def emu_merge(parts):
    l, acc, m = parts[0]
    for l2, a2, m2 in parts[1:]:
        mn = torch.maximum(m, m2)
        a0, a1 = torch.exp(m - mn), torch.exp(m2 - mn)
        l, acc, m = fma(l, a0, l2 * a1), fma(acc, a0[:, None], a2 * a1[:, None]), mn
    return l, acc, m


def emu_local_corr_softmax(f0, f1, ry, rx, stereo, pix, stencil, defect=None):
    B, h, w, _ = f0.shape
    b, y, x = pix
    dy, dx = ref64.window_offsets(ry, rx)
    sy, sx = y[:, None] + dy, x[:, None] + dx
    valid = (sx >= 0) & (sx < w) & (sy >= 0) & (sy < h)
    a = f0[b, y, x]
    if stencil:                                          # integer taps, one FMA chain over the 128 channels
        v = f1[b[:, None].expand_as(sx), sy.clamp(0, h - 1), sx.clamp(0, w - 1)] * valid[..., None]
        if defect == "drop_halo_col":                   # the last halo column of the 32-wide tile is never staged
            v = v * (sx != (x // 32 * 32 + 35)[:, None])[..., None]
        s = torch.zeros(sx.shape, dtype=F32)
        for c in range(C):
            s = fma(a[:, None, c], v[..., c], s)
    else:
        ix = unnorm(norm_window(sx.float(), w), w)
        iy = unnorm(norm_window(sy.float(), h), h)
        s = emu_dot8(a, emu_taps(f1, b, ix, iy))
    s = s / SQRT_C32
    if defect != "oob_logit0":
        s = torch.where(valid, s, torch.full_like(s, -1e9))
    vals = torch.stack((sx, sy), -1).float()
    if stencil:
        nrow = 2 * rx + 1
        rows = [(0, 1), (2, 3), (4, 5), (6, 7), (8,)]
        if defect == "drop_last_row":
            rows = rows[:-1]
        parts = [emu_online(s[:, r[0] * nrow:(r[-1] + 1) * nrow], vals[:, r[0] * nrow:(r[-1] + 1) * nrow]) for r in rows]
        l, acc, _ = emu_merge(parts)
    else:
        l, acc, _ = emu_online(s, vals)
    o = acc / l[:, None] - torch.stack((x, y), -1).float()
    return -o[:, :1] if stereo else o


def _feat(B, h, w, seed, scale=1.5):
    gen = g(seed)
    return torch.randn((B, h, w, C), generator=gen) * scale, torch.randn((B, h, w, C), generator=gen) * scale


def _sub(B, h, w, seed, tx=(), ty=()):
    return ref64.pixel_subset(B, h, w, g(seed), tx, ty, n_seam=400, n_rand=200)


LCS_CPU = [
    # name, B, h, w, ry, rx, stereo, stencil
    ("stencil_18x70", 2, 18, 70, 4, 4, False, True),
    ("gather_flow_r3", 1, 14, 23, 3, 3, False, False),
    ("gather_stereo", 2, 10, 40, 0, 4, True, False),
]


@pytest.mark.parametrize("name,B,h,w,ry,rx,stereo,stencil", LCS_CPU)
def test_local_corr_softmax64_matches_oracle_and_emulation(name, B, h, w, ry, rx, stereo, stencil):
    f0, f1 = _feat(B, h, w, 200 + w)
    pix = _sub(B, h, w, 201, (32,), (8,))
    ref, bnd = ref64.local_corr_softmax64(f0, f1, ry, rx, stereo, pix, stencil)
    oracle = refops.local_corr_softmax(f0, f1, h, w, ry, rx, stereo)[pix]
    _, bnd_g = ref64.local_corr_softmax64(f0, f1, ry, rx, stereo, pix, False)
    ref64.check(name + " oracle", oracle, ref, bnd_g)                    # the oracle's taps go through grid_sample
    r = ref64.check(name + " emulation", emu_local_corr_softmax(f0, f1, ry, rx, stereo, pix, stencil), ref, bnd)
    assert r < 0.5


@pytest.mark.parametrize("defect,case", [("drop_last_row", "stencil_18x70"), ("drop_halo_col", "stencil_18x70"),
                                         ("oob_logit0", "stencil_18x70"), ("oob_logit0", "gather_stereo")])
def test_local_corr_softmax64_rejects_defects(defect, case):
    name, B, h, w, ry, rx, stereo, stencil = next(c for c in LCS_CPU if c[0] == case)
    f0, f1 = _feat(B, h, w, 200 + w)
    pix = _sub(B, h, w, 201, (32,), (8,))
    ref, bnd = ref64.local_corr_softmax64(f0, f1, ry, rx, stereo, pix, stencil)
    rejects(name + " " + defect, emu_local_corr_softmax(f0, f1, ry, rx, stereo, pix, stencil, defect), ref, bnd)


def test_local_corr_softmax64_translation_property():
    """f1 = f0 shifted by (dx, dy): away from the border the window's peak is the shift (peaked features)."""
    B, h, w = 1, 24, 40
    f0, _ = _feat(B, h, w, 210, 4.0)
    f1 = torch.roll(f0, (2, -3), (1, 2))                  # f1[y + 2, x - 3] = f0[y, x]
    ys, xs = torch.meshgrid(torch.arange(6, h - 6), torch.arange(6, w - 6), indexing="ij")
    pix = (torch.zeros(ys.numel(), dtype=torch.long), ys.reshape(-1), xs.reshape(-1))
    ref, bnd = ref64.local_corr_softmax64(f0, f1, 4, 4, False, pix, True)
    assert torch.allclose(ref, torch.tensor([-3.0, 2.0], dtype=torch.float64).expand_as(ref), atol=1e-9)


def emu_corr_volume(f0, f1, flow, radius, pix, defect=None):
    B, h, w, _ = f0.shape
    b, y, x = pix
    fl = flow[b, y, x].float()
    u, v = (fl[:, 0], fl[:, 1]) if fl.shape[-1] == 2 else ((fl[:, 0] if defect == "disp_plus" else -fl[:, 0]), 0 * fl[:, 0])
    cx = unnorm(norm_window(x.float() + u, w), w)
    cy = unnorm(norm_window(y.float() + v, h), h)
    fx, fy = torch.floor(cx), torch.floor(cy)
    xe, ye = fx + 1.0, fy + 1.0
    wnw, wne, wsw, wse = (xe - cx) * (ye - cy), (cx - fx) * (ye - cy), (xe - cx) * (cy - fy), (cx - fx) * (cy - fy)
    if defect == "nesw_swap":
        wne, wsw = wsw, wne
    G = 2 * radius + 2
    gy, gx = torch.meshgrid(torch.arange(G), torch.arange(G), indexing="ij")
    yy = fy.long()[:, None] - radius + gy.reshape(-1)
    xx = fx.long()[:, None] - radius + gx.reshape(-1)
    ok = (yy >= 0) & (yy < h) & (xx >= 0) & (xx < w)
    if defect == "replicate":
        ok = torch.ones_like(ok)
    rows = f1[b[:, None].expand_as(yy), yy.clamp(0, h - 1), xx.clamp(0, w - 1)] * ok[..., None]
    d = emu_dot8(f0[b, y, x], rows).view(-1, G, G)
    n = 2 * radius + 1
    r = d[:, :n, :n] * wnw[:, None, None]
    r = fma(d[:, :n, 1:], wne[:, None, None], r)
    r = fma(d[:, 1:, :n], wsw[:, None, None], r)
    r = fma(d[:, 1:, 1:], wse[:, None, None], r)
    return (r / SQRT_C32).reshape(-1, n * n)


def _flows(kind, B, h, w, fd, seed):
    gen = g(seed)
    shp = (B, h, w, fd)
    if kind == "sigma12":
        return torch.randn(shp, generator=gen) * 12
    if kind == "frac":
        return torch.randint(-6, 7, shp, generator=gen).float() + torch.rand(shp, generator=gen) * 0.8 + 0.1
    if kind == "half":
        return torch.randint(-3, 4, shp, generator=gen).float() + 0.5
    if kind == "near_int":
        return torch.randint(-4, 5, shp, generator=gen).float() + (torch.rand(shp, generator=gen) - 0.5) * 2e-6
    raise ValueError(kind)


CV_CPU = [("sigma12", 2), ("frac", 2), ("frac", 1), ("near_int", 2)]


@pytest.mark.parametrize("kind,fd", CV_CPU)
def test_corr_volume64_and_flow_warp64_match_oracle_and_emulation(kind, fd):
    B, h, w = 2, 14, 40
    f0, f1 = _feat(B, h, w, 220 + fd)
    fl = _flows(kind, B, h, w, fd, 221)
    pix = _sub(B, h, w, 222)
    ref, bnd = ref64.local_corr_volume64(f0, f1, fl, 4, pix)
    ref64.check("corr volume %s fd %d oracle" % (kind, fd), refops.local_corr_volume(f0, f1, fl, h, w, 4)[pix], ref, bnd)
    r = ref64.check("corr volume %s fd %d emulation" % (kind, fd), emu_corr_volume(f0, f1, fl, 4, pix), ref, bnd)
    assert r < 0.5
    ref, bnd = ref64.flow_warp64(f1, fl, pix)
    ref64.check("flow warp %s fd %d oracle" % (kind, fd), refops.flow_warp(f1, fl, h, w)[pix], ref, bnd)
    r = ref64.check("flow warp %s fd %d emulation" % (kind, fd), emu_flow_warp(f1, fl, pix), ref, bnd)
    assert r < 0.5


def emu_flow_warp(f, flow, pix, defect=None):
    B, h, w, _ = f.shape
    b, y, x = pix
    fl = flow[b, y, x].float()
    u, v = (fl[:, 0], fl[:, 1]) if fl.shape[-1] == 2 else ((fl[:, 0] if defect == "disp_plus" else -fl[:, 0]), 0 * fl[:, 0])
    ix = unnorm(norm_sample(x.float() + u, w), w)[:, None]
    iy = unnorm(norm_sample(y.float() + v, h), h)[:, None]
    return emu_taps(f, b, ix, iy, defect)[:, 0]


@pytest.mark.parametrize("defect,kind,fd", [("replicate", "sigma12", 2), ("nesw_swap", "frac", 2),
                                            ("disp_plus", "frac", 1)])
def test_corr_volume64_and_flow_warp64_reject_defects(defect, kind, fd):
    B, h, w = 2, 14, 40
    f0, f1 = _feat(B, h, w, 220 + fd)
    fl = _flows(kind, B, h, w, fd, 221)
    pix = _sub(B, h, w, 222)
    ref, bnd = ref64.local_corr_volume64(f0, f1, fl, 4, pix)
    rejects("corr volume " + defect, emu_corr_volume(f0, f1, fl, 4, pix, defect), ref, bnd)
    if defect != "nesw_swap":
        ref, bnd = ref64.flow_warp64(f1, fl, pix)
        rejects("flow warp " + defect, emu_flow_warp(f1, fl, pix, defect), ref, bnd)


def emu_propagate(q, k, flow, radius, pix, defect=None):
    B, h, w, _ = q.shape
    b, y, x = pix
    dy, dx = ref64.window_offsets(radius, radius)
    sy, sx = y[:, None] + dy, x[:, None] + dx
    ok = (sx >= 0) & (sx < w) & (sy >= 0) & (sy < h)
    bb = b[:, None].expand_as(sy)
    kv = k[bb, sy.clamp(0, h - 1), sx.clamp(0, w - 1)] * ok[..., None]
    s = emu_dot8(q[b, y, x].contiguous(), kv) / SQRT_C32
    s = torch.where(ok, s, torch.full_like(s, -1e9) if defect == "exclude_oob" else torch.zeros_like(s))
    vals = flow[bb, sy.clamp(0, h - 1), sx.clamp(0, w - 1)] * ok[..., None]
    l, acc, _ = emu_online(s, vals)
    return acc / l[:, None]


@pytest.mark.parametrize("fd", [1, 2])
def test_propagate_local64_matches_oracle_and_emulation(fd):
    B, h, w = 2, 12, 30
    gen = g(230 + fd)
    qk = torch.randn((B, h * w, 256), generator=gen) * 1.5
    q, k = qk[..., :128].reshape(B, h, w, C), qk[..., 128:].reshape(B, h, w, C)
    fl = torch.randn((B, h, w, fd), generator=gen) * 5
    pix = _sub(B, h, w, 231)
    ref, bnd = ref64.propagate_local64(q, k, fl, 1, pix)
    oracle = refops.propagate_local(q.contiguous(), k.contiguous(), fl, h, w, 1)[pix]
    ref64.check("propagate fd %d oracle" % fd, oracle, ref, bnd)
    r = ref64.check("propagate fd %d emulation" % fd, emu_propagate(q, k, fl, 1, pix), ref, bnd)
    assert r < 0.5
    rejects("propagate exclude out-of-image keys", emu_propagate(q, k, fl, 1, pix, "exclude_oob"), ref, bnd)


def depth_setup(B, h, w, seed, kind="bidir", neg=False):
    """Features, cameras built by UniMatch.depth_cameras (at 1/8 resolution, bidirectional) and the workloads' 64
    inverse-depth candidates.  kind: "bidir" (small motion), "rotated", "forward" (2 units forward: near candidates project
    behind the camera)."""
    import types
    from unimatch_b200 import UniMatch
    gen = g(seed)
    f0 = torch.randn((B, h, w, C), generator=gen) * 1.5
    f1 = torch.randn((B, h, w, C), generator=gen) * 1.5
    if neg:                                                 # every in-image correlation negative: ties at logit 0 decide
        f0, f1 = f0.abs(), -f1.abs()
    n = (B + 1) // 2
    intr = torch.tensor([[500.0, 0, 8 * w / 2 - 3], [0, 490.0, 8 * h / 2 + 2], [0, 0, 1]]).repeat(n, 1, 1)
    pose = torch.eye(4).repeat(n, 1, 1)
    ang = 0.15 if kind == "rotated" else 0.02
    ca, sa = math.cos(ang), math.sin(ang)
    pose[:, 0, 0], pose[:, 0, 2], pose[:, 2, 0], pose[:, 2, 2] = ca, sa, -sa, ca
    # "forward": the mirror image of a point behind the camera lands inside the image, so only the z clamp keeps it out
    pose[:, :3, 3] = torch.tensor([0.0, 0.0, -2.0] if kind == "forward" else [0.3, -0.05, 0.1])
    cams = UniMatch.depth_cameras(types.SimpleNamespace(_cands={}), intr, pose, 8, 1.0 / 10, 1.0 / 0.5, 64, True)
    return f0, f1, cams


def emu_depth(f0, f1, cams, pix, from_argmax, defect=None):
    B, h, w, _ = f0.shape
    b, y, x = pix
    Ki, Kb, Pm, cand = cams["K_inv"][b], cams["K"][b], cams["pose"][b], cams["cand"]
    fx, fy = x.float(), y.float()
    X = [fma(Ki[:, r, 2], torch.ones(()), fma(Ki[:, r, 1], fy, Ki[:, r, 0] * fx)) for r in range(3)]
    Xr = [fma(Pm[:, r, 2], X[2], fma(Pm[:, r, 1], X[1], Pm[:, r, 0] * X[0])) for r in range(3)]
    a = f0[b, y, x]
    logits = []
    for d in range(cand.numel()):
        depth = 1.0 / cand[d]
        Pt = [fma(Xr[r], depth, Pm[:, r, 3]) for r in range(3)]
        pr = [fma(Kb[:, r, 2], Pt[2], fma(Kb[:, r, 1], Pt[1], Kb[:, r, 0] * Pt[0])) for r in range(3)]
        z = pr[2] if defect == "no_zclamp" else torch.clamp(pr[2], min=1e-3)
        ix = unnorm(norm_sample(pr[0] / z, w), w)[:, None]
        iy = unnorm(norm_sample(pr[1] / z, h), h)[:, None]
        logits.append(emu_dot8(a, emu_taps(f1, b, ix, iy))[:, 0] / SQRT_C32)
    s = torch.stack(logits, 1)
    if from_argmax:
        best = torch.zeros(s.shape[0])
        m = torch.full((s.shape[0],), -math.inf)
        for d in range(cand.numel()):
            better = s[:, d] >= m if defect == "last_max" else s[:, d] > m
            best = torch.where(better, cand[d], best)
            m = torch.maximum(m, s[:, d])
        return best
    l, acc, _ = emu_online(s, cand.view(1, -1, 1).expand(s.shape[0], -1, 1))
    return (acc / l[:, None])[:, 0]


@pytest.mark.parametrize("kind", ["bidir", "rotated", "forward"])
def test_depth_corr64_matches_oracle_and_emulation(kind):
    B, h, w = 2, 12, 16
    f0, f1, cams = depth_setup(B, h, w, 240, kind)
    pix = _sub(B, h, w, 241)
    ref, bnd, s, ds = ref64.depth_corr64(f0, f1, cams["K"], cams["K_inv"], cams["pose"], cams["cand"], pix)
    args = (f0, f1, cams["K"], cams["K_inv"], cams["pose"], cams["cand"], h, w)
    ref64.check("depth %s oracle" % kind, refops.depth_corr_softmax(*args, False)[pix][:, 0], ref, bnd)
    r = ref64.check("depth %s emulation" % kind, emu_depth(f0, f1, cams, pix, False), ref, bnd)
    assert r < 0.5
    ref64.check_argmax("depth %s oracle argmax" % kind, refops.depth_corr_softmax(*args, True)[pix][:, 0], cams["cand"], s,
                       ds)
    ref64.check_argmax("depth %s emulation argmax" % kind, emu_depth(f0, f1, cams, pix, True), cams["cand"], s, ds)
    if kind == "forward":
        rejects("depth without the z clamp", emu_depth(f0, f1, cams, pix, False, "no_zclamp"), ref, bnd)


def test_depth_corr64_argmax_rejects_last_maximum():
    """Negative in-image correlations: candidates projecting outside (logit exactly 0) tie for the maximum, and
    torch.argmax takes the first of them."""
    B, h, w = 2, 12, 16
    f0, f1, cams = depth_setup(B, h, w, 250, "forward", neg=True)
    pix = _sub(B, h, w, 251)
    _, _, s, ds = ref64.depth_corr64(f0, f1, cams["K"], cams["K_inv"], cams["pose"], cams["cand"], pix)
    ref64.check_argmax("depth argmax ties", emu_depth(f0, f1, cams, pix, True), cams["cand"], s, ds)
    with pytest.raises(AssertionError):
        ref64.check_argmax("depth argmax last max", emu_depth(f0, f1, cams, pix, True, "last_max"), cams["cand"], s, ds)


def emu_convex(flow, mask, factor, mult, defect=None):
    B, h, w, fd = flow.shape
    FF = factor * factor
    m = mask.view(B, h, w, 9, FF)
    e = torch.exp(m - m.amax(3, keepdim=True))
    fl = torch.nn.functional.pad(flow * mult, (0, 0, 1, 1, 1, 1))
    inside = torch.nn.functional.pad(torch.ones((B, h, w, 1)), (0, 0, 1, 1, 1, 1))
    nb = torch.stack([fl[:, ty:ty + h, tx:tx + w] for ty in range(3) for tx in range(3)], 3)      # [B, h, w, 9, fd]
    ins = torch.stack([inside[:, ty:ty + h, tx:tx + w] for ty in range(3) for tx in range(3)], 3)
    den = torch.zeros((B, h, w, FF))
    for t in range(9):
        den = den + e[:, :, :, t] * (ins[:, :, :, t] if defect == "inimage_norm" else 1.0)
    acc = torch.zeros((B, h, w, FF, fd))
    for t in range(9):
        acc = fma((e[:, :, :, t] / den)[..., None], nb[:, :, :, t, None, :], acc)
    return acc.view(B, h, w, factor, factor, fd).permute(0, 5, 1, 3, 2, 4).reshape(B, fd, h * factor, w * factor)


@pytest.mark.parametrize("factor,fd,mult,scale", [(4, 2, 4, 3.0), (8, 1, 1, 3.0), (4, 2, 4, 60.0)])
def test_convex_upsample64_matches_oracle_and_emulation(factor, fd, mult, scale):
    B, h, w = 2, 5, 7
    gen = g(260 + factor + fd)
    fl = torch.randn((B, h, w, fd), generator=gen) * 4
    mask = torch.randn((B, h, w, 9 * factor * factor), generator=gen) * scale
    ref, bnd = ref64.convex_upsample64(fl, mask, factor, mult)
    name = "convex F %d fd %d mult %d scale %g" % (factor, fd, mult, scale)
    ref64.check(name + " oracle", refops.convex_upsample(fl, mask, factor, float(mult)), ref, bnd)
    assert ref64.check(name + " emulation", emu_convex(fl, mask, factor, mult), ref, bnd) < 0.5
    rejects(name + " in-image normalisation", emu_convex(fl, mask, factor, mult, "inimage_norm"), ref, bnd)


def emu_upsample2x(flow, mult, defect=None):
    B, h, w, fd = flow.shape
    H, W = 2 * h, 2 * w
    f32 = lambda v: torch.tensor(float(v), dtype=F32)
    Y, X = torch.arange(H).float(), torch.arange(W).float()
    if defect == "align_false":
        fy, fx = ((Y + 0.5) * 0.5 - 0.5).clamp(min=0), ((X + 0.5) * 0.5 - 0.5).clamp(min=0)
    else:
        fy = (f32(h - 1) / f32(H - 1) if H > 1 else f32(0)) * Y
        fx = (f32(w - 1) / f32(W - 1) if W > 1 else f32(0)) * X
    y0, x0 = fy.long(), fx.long()
    y1, x1 = y0 + (y0 < h - 1).long(), x0 + (x0 < w - 1).long()
    ly, lx = (fy - y0.float())[:, None, None], (fx - x0.float())[None, :, None]
    hy, hx = 1.0 - ly, 1.0 - lx
    v = lambda yy, xx: flow[:, yy][:, :, xx]
    return (hy * (hx * v(y0, x0) + lx * v(y0, x1)) + ly * (hx * v(y1, x0) + lx * v(y1, x1))) * mult


@pytest.mark.parametrize("h,w,fd", [(6, 9, 2), (1, 12, 1), (7, 5, 1)])
def test_upsample2x64_matches_oracle_and_emulation(h, w, fd):
    fl = torch.randn((2, h, w, fd), generator=g(270 + h)) * 6
    ref, bnd = ref64.upsample2x64(fl, 2.0)
    ref64.check("upsample2x %dx%d oracle" % (h, w), refops.upsample2x(fl, 2.0), ref, bnd)
    assert ref64.check("upsample2x %dx%d emulation" % (h, w), emu_upsample2x(fl, 2.0), ref, bnd) < 0.5
    rejects("upsample2x align_corners=False", emu_upsample2x(fl, 2.0, "align_false"), ref, bnd)


def test_add_position_ref_matches_refops():
    gen = g(280)
    x = torch.randn((3, 12, 20, C), generator=gen)
    table = torch.randn((6, 5, C), generator=gen)
    want = torch.empty_like(x)
    for yy in range(12):
        for xx in range(20):
            want[:, yy, xx] = x[:, yy, xx] + table[yy % 6, xx % 5]
    assert torch.equal(ref64.add_position_ref(x, table, 12, 20), want)
    assert torch.equal(refops.add_position(x, table, 12, 20), want)


STEM_SCALE = [1.0 / (255.0 * s_) for s_ in (0.229, 0.224, 0.225)]
STEM_SHIFT = [-m_ / s_ for m_, s_ in zip((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))]


def stem_images(n, H, W, seed):
    """Raw pixels in [0, 255] with saturated 0 and 255 blocks."""
    gen = g(seed)
    x = torch.rand((n, 3, H, W), generator=gen) * 255
    x[:, :, :H // 3, :W // 4] = 0.0
    x[:, :, H // 2:, W // 2:W // 2 + W // 5] = 255.0
    return x.round()


def emu_stem(x, weight, bias, stride, relu, scale, shift, defect=None):
    F_ = torch.nn.functional
    if scale is not None:
        sc, sh = torch.tensor(scale).view(1, -1, 1, 1), torch.tensor(shift).view(1, -1, 1, 1)
        if defect == "pad_shift":                           # normalising after the zero padding
            v = F_.pad(x, (3, 3, 3, 3)) * sc + sh
            y = F_.conv2d(v, weight, bias, stride=stride)
        else:
            y = F_.conv2d(fma(x, sc.expand_as(x), sh.expand_as(x)), weight, bias, stride=stride, padding=3)
    else:
        y = F_.conv2d(x, weight, bias, stride=stride, padding=3)
    y = torch.relu(y) if relu else y
    return y.permute(0, 2, 3, 1)


@pytest.mark.parametrize("norm", [True, False])
def test_conv7x7_64_stem_matches_oracle_and_emulation(norm):
    x = stem_images(2, 37, 54, 290)
    if not norm:
        x = x / 255.0
    wt = torch.randn((64, 3, 7, 7), generator=g(291)) * (2.0 / 147) ** 0.5
    sc, sh = (STEM_SCALE, STEM_SHIFT) if norm else (None, None)
    ref, bnd = ref64.conv7x7_64(x, wt, None, 2, False, sc, sh)
    out = torch.empty(ref.shape, dtype=F32)
    refops.conv7x7_small(x[:1], x[1:], True, wt, None, 2, False, sc, sh, out, None)
    ref64.check("stem norm %s oracle" % norm, out, ref, bnd)
    assert ref64.check("stem norm %s emulation" % norm, emu_stem(x, wt, None, 2, False, sc, sh), ref, bnd) < 0.5
    if norm:
        rejects("stem padded with the shift", emu_stem(x, wt, None, 2, False, sc, sh, "pad_shift"), ref, bnd)


@pytest.mark.parametrize("cin", [1, 2])
def test_conv7x7_64_flow_encoder_matches_oracle(cin):
    gen = g(295 + cin)
    fl = torch.randn((2, 15, 22, cin), generator=gen) * 20
    wt = torch.randn((128, cin, 7, 7), generator=gen) * (2.0 / (49 * cin)) ** 0.5
    bias = torch.randn(128, generator=gen) * 0.1
    ref, bnd = ref64.conv7x7_64(fl.permute(0, 3, 1, 2), wt, bias, 1, True)
    out = torch.empty(ref.shape, dtype=F32)
    split = torch.empty((2,) + ref.shape, dtype=torch.float16)
    refops.conv7x7_small(fl, None, False, wt, bias, 1, True, None, None, out, split)
    ref64.check("flow encoder cin %d oracle" % cin, out, ref, bnd)
    ref64.check("flow encoder cin %d oracle split" % cin, split[0].double() + split[1].double(), ref,
                ref64.split_out_bound(ref, bnd))
