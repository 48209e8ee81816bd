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
