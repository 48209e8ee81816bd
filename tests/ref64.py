"""Float64 references of the tensor-core kernels, each with a per-element error bound derived from the arithmetic the kernel
promises.  Written from the math (Swin windows, softmax, convolution, LayerNorm, GELU), not through the fp32 oracle.

Arithmetic model ("fp32-faithful", README): every fp32 operand x is split into fp16 (hi, lo) = (rn16(x), rn16(x - hi));
products are hi*hi + hi*lo + lo*hi formed exactly on the tensor cores and accumulated in fp32.  The bound of a GEMM-like
output y = sum_k x_k w_k is

    |err| <= G0 * A  +  steps * 2^-23 * (|y| + 3 R)  +  REP

  A    = sum |x||w|               the dropped lo*lo term (<= 2^-22 |x||w| each) and the alignment of the products inside one
                                  MMA: G0 = 2^-21.
  steps                           accumulate steps of the fp32 accumulator (one wgmma of K = 16 each, 3 split products):
                                  tensor-core accumulation truncates, so each step may lose up to one ulp (2^-23 relative)
                                  of the running sum.  The running sum stays within |y| + 3 R, R = sqrt(sum (x w)^2), for
                                  operands of random sign (the partial sums of a random walk stay within about 3 of its
                                  standard deviations of the straight line to y); for one-signed sums R << |y| = A.
  REP  = sum |x - (x_hi + x_lo)||w| + sum |x_hi + x_lo||w - (w_hi + w_lo)|
                                  what the fp16 split itself cannot represent, computed exactly here from the split: fp16
                                  subnormals (small operands) are counted as what they are, not hidden under a floor.

Attention / softmax-expectation outputs o = sum_k p_k v_k add a logit term sum_k p_k |v_k - o| ds_k (first-order
sensitivity of the softmax; ds_k = the GEMM bound of the logit scaled by 1/sqrt(128), plus the fp32 rounding of the
exponent argument), a value term for P V (the same GEMM bound over the keys) and the (hi, lo) split of P:
2^-22 p_k + 2^-25 / l per key, l = sum_k exp(s_k - max s) >= 1.

`check` compares a kernel output with (ref, bound), prints the headroom max(err / bound) and on failure names the worst
element by its tile coordinates.
"""
import math

import torch

C = 128
EPS_IN = 1e-5              # InstanceNorm2d eps
EPS_LN = 1e-5              # LayerNorm eps
G0 = 2.0 ** -21            # per-product term (lo*lo dropped, alignment inside one MMA)
U_STEP = 2.0 ** -23        # one truncated accumulate step, relative to the running sum
U32 = 2.0 ** -24           # fp32 unit roundoff
WALK = 3.0                 # running-sum excursion in units of R
SPLIT_OUT = (2.0 ** -21, 2.0 ** -24)   # fp32 value stored as fp16 (hi, lo) planes: twice the worst loss (2^-22 rel, 2^-25 abs)
ACT_ABS = {"tanh": 1e-6, "sigmoid": 5e-7, "gelu": 5e-7}   # fast-intrinsic epilogue functions, absolute error
ACT_SLOPE = {"none": 1.0, "relu": 1.0, "tanh": 1.0, "sigmoid": 0.25, "gelu": 1.13}
L_SUM = 4.0                # fp32 sums of the softmax weights: L_SUM * 2^-24 * sqrt(keys) relative
UFLOW = 2.0 ** -100        # absolute error of a weight that underflows fp32 (peaked or saturated logits), per |value|

ACT_NAMES = {0: "none", 1: "relu", 2: "tanh", 3: "sigmoid", 4: "gelu"}
MASK_NONE, MASK_SWIN, MASK_CAUSAL = 0, 1, 2
VALUE_TENSOR, VALUE_COORDS, VALUE_XCOORD = 0, 1, 2
POST_NONE, POST_MINUS_OWN, POST_OWN_MINUS = 0, 1, 2
CONV_LINEAR, CONV_GRU_ZR, CONV_GRU_Q, CONV_LN = 0, 1, 2, 3


# ---- the fp16 (hi, lo) split -----------------------------------------------------------------------------------------
def split_sum(x):
    """fp32 tensor -> float64 value of hi + lo, the operand the tensor cores actually see."""
    x = x.float()
    hi = x.half()
    lo = (x - hi.float()).half()
    return hi.double() + lo.double()


def split_out_bound(val, bound):
    """bound of an output written as fp16 (hi, lo) planes instead of fp32."""
    return bound + SPLIT_OUT[0] * val.abs() + SPLIT_OUT[1]


def gemm_steps(k):
    """accumulate steps of one output: 3 split products x K / 16."""
    return 3 * ((k + 15) // 16)


# ---- activations (float64, exact) ----------------------------------------------------------------------------------
def act64(y, name):
    if name == "relu":
        return torch.relu(y)
    if name == "tanh":
        return torch.tanh(y)
    if name == "sigmoid":
        return torch.sigmoid(y)
    if name == "gelu":
        return 0.5 * y * (1.0 + torch.erf(y / math.sqrt(2.0)))
    return y


def act_bound(y, e, name):
    out = act64(y, name)
    return out, ACT_SLOPE[name] * e + ACT_ABS.get(name, 0.0) + 2 * U32 * out.abs() + (U32 * y.abs() if name == "gelu" else 0.0)


def layernorm64(y, e, gamma, beta, res=None):
    """LayerNorm over the last dim (n = 128) of y with per-element input bound e -> (out, bound).

    The kernels take two-pass fp32 statistics: mean = fl(sum y) / n, then var = fl(sum (y - mean)^2) / n, then
    out = (y - mean) * rsqrt(var + eps) * gamma + beta (+ residual).
      * The fp32 sum of n terms, in any order, is off by at most (n - 1) u sum |y| (u = 2^-24), and / n is exact, so the
        mean carries an absolute error dm <= n u mean|y| besides the input's em.  Every centred value moves by the same dm,
        so the output moves by |gamma| rstd dm -- independently of |d|: a channel that sits exactly on the mean (a
        constant row, the zero padding rows) still sees it.
      * That shift changes the centred sum of squares by n dm^2 (the cross term sums to 0), i.e. rstd by at most
        (dm rstd)^2 relative; the fp32 sum of squares adds n u relative, rsqrt and the products 2^-21.
    Exact input (e = 0, a constant row of a value whose multiples up to n are exact in fp32) makes dm's actual value 0,
    so the output is beta (+ residual) bit for bit."""
    g, b = gamma.double(), beta.double()
    n = y.shape[-1]
    mean = y.mean(-1, keepdim=True)
    d = y - mean
    var = (d * d).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + EPS_LN)
    out = d * rstd * g + b
    em = e.mean(-1, keepdim=True)
    dm = n * U32 * y.abs().mean(-1, keepdim=True)
    rho = ((d.abs() * (e + em)).sum(-1, keepdim=True) / (d * d + EPS_LN).sum(-1, keepdim=True) + 2.0 ** -21 +
           n * U32 + (dm * rstd) ** 2)
    bound = g.abs() * rstd * (e + em + dm) + g.abs() * d.abs() * rstd * rho + 4 * U32 * (g.abs() * d.abs() * rstd + b.abs())
    if res is not None:
        out = out + res.double()
        bound = bound + U32 * out.abs()
    return out, bound


# ---- convolution / Linear (um_conv2d_tc) ----------------------------------------------------------------------------
def _c2(x, w, stride, pad):
    return torch.nn.functional.conv2d(x, w, None, stride=stride, padding=pad)


def patches(x, kh, kw, stride, pad, pix):
    """Input patches [P, c * kh * kw] (channel-major, the order of weight.flatten(1)) of the output pixels pix = (b, y, x) of
    a convolution over the channel-last map x [B, H, W, c], zeros outside the image."""
    b, yo, xo = pix
    H, W = x.shape[1], x.shape[2]
    Y = (yo[:, None] * stride - pad[0] + torch.arange(kh))[:, :, None].expand(-1, kh, kw)
    X = (xo[:, None] * stride - pad[1] + torch.arange(kw))[:, None, :].expand(-1, kh, kw)
    ok = (Y >= 0) & (Y < H) & (X >= 0) & (X < W)
    v = x[b[:, None, None].expand_as(Y), Y.clamp(0, H - 1), X.clamp(0, W - 1)] * ok[..., None].to(x.dtype)
    return v.permute(0, 3, 1, 2).reshape(b.numel(), -1)


def conv64(xs, wt, bias=None, pad=(0, 0), stride=1, mode=CONV_LINEAR, act=0, aux0=None, aux1=None, gamma=None, beta=None,
           pre=None, pix=None):
    """xs: channel-last fp32 sources [B, H, W, c_i] (concatenated along channels), wt: fp32 [cout, sum c_i, kh, kw].
    Returns (out, bound) channel-last float64 [B, Ho, Wo, cout] of what um_conv2d_tc writes: GRU_ZR -> [z | r * h].
    pix = (b, y, x) output pixels: (out, bound) [P, cout] at those pixels only (aux0, aux1 and pre stay whole maps)."""
    kh, kw = wt.shape[2], wt.shape[3]
    w, wh = wt.double(), split_sum(wt)
    if pix is None:
        x32 = torch.cat([x.float() for x in xs], -1).permute(0, 3, 1, 2)
        x, xh = x32.double(), split_sum(x32)
        y = _c2(x, w, stride, pad)
        a = _c2(x.abs(), w.abs(), stride, pad)
        r = torch.sqrt(_c2(x * x, w * w, stride, pad))
        rep = _c2((x - xh).abs(), w.abs(), stride, pad) + _c2(xh.abs(), (w - wh).abs(), stride, pad)
    else:
        p32 = patches(torch.cat([x.float() for x in xs], -1), kh, kw, stride, pad, pix)
        x, xh = p32.double(), split_sum(p32)
        w, wh = w.flatten(1), wh.flatten(1)
        y = x @ w.T
        a = x.abs() @ w.abs().T
        r = torch.sqrt((x * x) @ (w * w).T)
        rep = (x - xh).abs() @ w.abs().T + xh.abs() @ (w - wh).abs().T
        aux0, aux1, pre = (None if t is None else t[pix] for t in (aux0, aux1, pre))
    ktot = sum((c.shape[-1] + 63) // 64 * 64 for c in xs) * kh * kw
    nk = ktot // 64
    steps = 12 + nk if nk >= 8 else 12 * nk          # K >= 512: fresh accumulator per 64-wide stage, then fp32 adds
    e = G0 * a + steps * U_STEP * (y.abs() + WALK * r) + rep
    if pix is None:
        y, e = y.permute(0, 2, 3, 1), e.permute(0, 2, 3, 1)
    if bias is not None:
        y = y + bias.double()
        e = e + U32 * y.abs()
    if pre is not None:
        y = y + pre.double()[..., :y.shape[-1]]
        e = e + U32 * y.abs()
    if mode == CONV_LINEAR:
        return act_bound(y, e, ACT_NAMES[act])
    if mode == CONV_LN:
        return layernorm64(y, e, gamma, beta, aux0)
    if mode == CONV_GRU_ZR:
        z, ez = act_bound(y[..., :128], e[..., :128], "sigmoid")
        rr, er = act_bound(y[..., 128:], e[..., 128:], "sigmoid")
        h = aux0.double()
        return torch.cat((z, rr * h), -1), torch.cat((ez, er * h.abs() + U32 * (rr * h).abs()), -1)
    h, z = aux0.double(), aux1.double()
    t, et = act_bound(y, e, "tanh")
    out = (1 - z) * h + z * t
    return out, z.abs() * et + 4 * U32 * ((1 - z).abs() * h.abs() + (z * t).abs())


def ffn64(x0, x1, w1, w2, residual, gamma, beta):
    """Fused FFN on token rows: residual + LayerNorm(GELU([x0 | x1] W1^T) W2^T) -> (out, bound) [rows, 128]."""
    xx = torch.cat((x0, x1), -1).float()

    def gemm(x32, xd, wt):
        w, wh = wt.double().flatten(1), split_sum(wt.flatten(1))
        x, xh = xd, split_sum(x32)
        y = x @ w.T
        a = x.abs() @ w.abs().T
        r = torch.sqrt((x * x) @ (w * w).T)
        rep = (x - xh).abs() @ w.abs().T + xh.abs() @ (w - wh).abs().T
        return y, G0 * a + gemm_steps(w.shape[1]) * U_STEP * (y.abs() + WALK * r) + rep, w
    a, ea, _ = gemm(xx, xx.double(), w1)
    hdn, eh = act_bound(a, ea, "gelu")
    eh = split_out_bound(hdn, eh)                    # the hidden activation travels as fp16 (hi, lo) register operands
    y, ey, w2d = gemm(hdn.float(), hdn, w2)
    ey = ey + eh @ w2d.abs().T
    return layernorm64(y, ey, gamma, beta, residual)


# ---- window attention ---------------------------------------------------------------------------------------------
def window_layout(h, w, kh, kw, sh, sw):
    """[nwin, lw] token index (y * w + x of the un-shifted map) of every window position after the cyclic shift, and the
    Swin shift region (3 bands per shifted axis) of every position."""
    wh, ww = h // kh, w // kw
    yr = torch.arange(h).view(kh, wh)                 # rolled row -> (window row, offset)
    xr = torch.arange(w).view(kw, ww)
    Y = yr.view(kh, 1, wh, 1).expand(kh, kw, wh, ww)
    X = xr.view(1, kw, 1, ww).expand(kh, kw, wh, ww)
    tok = ((Y + sh) % h) * w + (X + sw) % w
    ry = torch.zeros_like(Y) if sh == 0 else (Y >= h - wh).long() + (Y >= h - sh).long()
    rx = torch.zeros_like(X) if sw == 0 else (X >= w - ww).long() + (X >= w - sw).long()
    return tok.reshape(kh * kw, wh * ww), (ry * 3 + rx).reshape(kh * kw, wh * ww)


def _logit_bound(qw, kw_):
    """raw logits q.k and their GEMM bound (24 accumulate steps over 128 channels)."""
    qh, kh_ = split_sum(qw), split_sum(kw_)
    q, k = qw.double(), kw_.double()
    s = q @ k.T
    a = q.abs() @ k.abs().T
    r = torch.sqrt((q * q) @ (k * k).T)
    rep = (q - qh).abs() @ k.abs().T + qh.abs() @ (k - kh_).abs().T
    return s, G0 * a + gemm_steps(C) * U_STEP * (s.abs() + WALK * r) + rep


def _pv(p, vals):
    """p [M, N] times vals: [N, d] shared by every row, or [M, N, d] per row."""
    return p @ vals if vals.dim() == 2 else torch.einsum("mn,mnd->md", p, vals)


def softmax_weighted(s, ds, vals, v_rep=None, tc_pv=True):
    """s: [M, N] scaled logits (-inf = excluded), ds: their bound, vals: [N, d] (or [M, N, d]: values per row) float64.
    Returns (o, bound) [M, d].  tc_pv: P V on the tensor cores (P split into fp16 (hi, lo), truncating accumulation over
    64-key tiles); otherwise fp32 CUDA-core sums of p * value."""
    smax = s.max(-1, keepdim=True).values
    e = torch.exp(s - smax)
    l = e.sum(-1, keepdim=True)
    p = e / l
    o = _pv(p, vals)
    va = vals.abs()
    pv = _pv(p, va)
    n = s.shape[-1]
    ds = torch.where(torch.isfinite(s), ds + U_STEP * (s.abs() + smax.abs()), torch.zeros_like(ds))
    pds = p * ds
    b = _pv(pds, va) + pds.sum(-1, keepdim=True) * o.abs()               # sum_k p_k ds_k |v_k - o|
    b = b + 2 * G0 * pv + 2 * U32 * o.abs() + L_SUM * U32 * math.sqrt(n) * (o.abs() + pv)
    b = b + UFLOW * _pv(torch.ones_like(p), va)                          # weights near and below the fp32 underflow
    if tc_pv:
        tiles = (n + 63) // 64
        b = b + 12 * tiles * U_STEP * (o.abs() + WALK * torch.sqrt((p * p) @ (vals * vals)))
        b = b + 2.0 ** -22 * pv + 2.0 ** -25 / l * va.sum(0, keepdim=True)
    if v_rep is not None:
        b = b + _pv(p, v_rep)
    return o, b


def attention64(q, k, v, kv_shift, h, w, kh, kw, sh, sw, mask_mode, tc=True, rows=None):
    """softmax(Q K^T / sqrt(128) + Swin mask) V per window with the cyclic shift and the roll back; key / value stream of
    stream n is (n + kv_shift) mod n_streams.  q, k, v: fp32 [n, h*w, 128].  Returns (out, bound, locate), [n, h*w, 128],
    or [n, R, 128] for the query tokens `rows` (sorted, distinct) only."""
    n = q.shape[0]
    tok, reg = window_layout(h, w, kh, kw, sh, sw)
    nwin, lw = tok.shape
    rows = torch.arange(h * w) if rows is None else rows
    slot = torch.full((h * w,), -1, dtype=torch.long)                  # token -> index into rows
    slot[rows] = torch.arange(rows.numel())
    out = torch.zeros((n, rows.numel(), C), dtype=torch.float64)
    bnd = torch.zeros_like(out)
    for wi in range(nwin):
        t = tok[wi]
        sel = (slot[t] >= 0).nonzero().view(-1)                        # window positions of the queries evaluated
        if sel.numel() == 0:
            continue
        m = reg[wi][sel][:, None] != reg[wi][None, :]
        for s_ in range(n):
            ks = (s_ + kv_shift) % n
            qw, kk, vv = q[s_, t[sel]], k[ks, t], v[ks, t]
            s, e = _logit_bound(qw, kk)
            s, e = s / math.sqrt(C), e / math.sqrt(C)
            if mask_mode == MASK_SWIN:
                s = s - 100.0 * m
                e = e + U_STEP * 100.0 * m
            vd = vv.double()
            o, b = softmax_weighted(s, e, vd, (vd - split_sum(vv)).abs(), tc_pv=tc)
            out[s_, slot[t[sel]]] = o
            bnd[s_, slot[t[sel]]] = b

    pos = torch.empty(h * w, dtype=torch.long)
    win = torch.empty(h * w, dtype=torch.long)
    for wi in range(nwin):
        pos[tok[wi]] = torch.arange(lw)
        win[tok[wi]] = wi

    def locate(idx):
        st, r, c = idx
        t = rows[r]
        return "stream %d, window %d, query tile %d, row %d, channel %d" % (st, win[t], pos[t] // 128, pos[t] % 128, c)
    return out, bnd, locate


def expectation64(q, k, values, n_streams, kv_shift, vdim, value_mode, post_op, h, w, kh, kw, mask_mode, rows=None):
    """sum_k softmax_k(q.k / sqrt(128)) value_k over the whole map (kh = kw = 1) or one window per image row (kh = h,
    kw = 1), causal mask = keys right of the query excluded (weight exp(-1e9)); value = a tensor, (x, y) or x of the key;
    post-op subtracts the query's own coordinates.  rows: query token subset.  Returns (out, bound) [n_streams, R, vdim]."""
    n_total, L, _ = q.shape
    rows = torch.arange(L) if rows is None else rows
    ys, xs = torch.div(torch.arange(L), w, rounding_mode="floor"), torch.arange(L) % w
    outs, bnds = [], []
    for s_ in range(n_streams):
        ks = (s_ + kv_shift) % n_total
        if value_mode == VALUE_TENSOR:
            vals = values[ks].double()
        elif value_mode == VALUE_COORDS:
            vals = torch.stack((xs, ys), -1).double()
        else:
            vals = xs[:, None].double()
        s, e = _logit_bound(q[s_, rows], k[ks])
        s, e = s / math.sqrt(C), e / math.sqrt(C)
        if kh != 1:
            s = torch.where(ys[rows][:, None] == ys[None, :], s, torch.full_like(s, -math.inf))
        if mask_mode == MASK_CAUSAL:
            s = torch.where(xs[None, :] > xs[rows][:, None], torch.full_like(s, -1e9), s)
        o, b = softmax_weighted(s, e, vals, tc_pv=False)
        own = torch.stack((xs[rows], ys[rows]), -1).double()[:, :vdim]
        if post_op == POST_MINUS_OWN:
            o = o - own
        elif post_op == POST_OWN_MINUS:
            o = own - o
        outs.append(o)
        bnds.append(b + U32 * o.abs())
    return torch.stack(outs), torch.stack(bnds)


# ---- instance norm ------------------------------------------------------------------------------------------------
def instance_norm_stats64(x):
    """x: [N, h, w, C] -> (mean, rstd) float64 [N, C] (biased variance, eps 1e-5) and the channels' std."""
    v = x.reshape(x.shape[0], -1, x.shape[-1]).double()
    mean = v.mean(1)
    var = ((v - mean[:, None]) ** 2).mean(1)
    return mean, 1.0 / torch.sqrt(var + EPS_IN), torch.sqrt(var)


# ---- matching-path kernels on the CUDA cores (um_local.cu, um_local_stencil.cu, um_misc.cu, um_stem.cu) ------------
# These run fp32 FMAs (no fp16 split, no fast math), so the bounds are the classical ones:
#   dot product over n sequential roundings     gamma_n * sum |a||b|, gamma_n = n u / (1 - n u), u = 2^-24
#     gather kernels: 16 FMAs per lane + 3 shuffle adds (n = 19); the stencil: one FMA chain over 128 channels
#   bilinear blend of 4 taps with fp32 weights   BLEND_N more roundings on the blend of |values|
#   coordinates                                  the kernels form positions in fp32 the way the reference does (normalise
#                                                to [-1, 1], un-normalise with align_corners=True), which moves a tap by a
#                                                few ulps of (size - 1) and of the position itself: COORD_REL * (size - 1 +
#                                                |p|).  The output moves by |d out / d x| dx + |d out / d y| dy, with the
#                                                derivative bounded by the largest finite difference of the four-tap cells
#                                                the rounding can reach (the cell of the position and its neighbours).
#   online softmax                               softmax_weighted(..., tc_pv=False)
SQRT_C = math.sqrt(C)
DOT_N_GATHER = 19
DOT_N_STENCIL = 128
BLEND_N = 6
COORD_REL = 2.0 ** -21


def gamma(n):
    return n * U32 / (1 - n * U32)


def coord_err(p, size):
    return COORD_REL * ((size - 1) + p.abs())


def bilerp(val, ix, iy):
    """Bilinear interpolation at float64 positions (ix, iy) [P, K] of val(yy, xx) -> [P, K, ...] (values at integer pixels,
    padding done by val), with the weights of the kernels' make_tap.  Returns (out, |d/dx| bound, |d/dy| bound, blend of
    |values|)."""
    x0, y0 = torch.floor(ix), torch.floor(iy)
    wx, wy = ix - x0, iy - y0
    x0, y0 = x0.long(), y0.long()
    V = [[val(y0 + j, x0 + i) for i in range(-1, 3)] for j in range(-1, 3)]
    ex = lambda t: t.view(t.shape + (1,) * (V[0][0].dim() - t.dim()))
    wx, wy = ex(wx), ex(wy)
    ws = ((1 - wx) * (1 - wy), wx * (1 - wy), (1 - wx) * wy, wx * wy)
    taps = (V[1][1], V[1][2], V[2][1], V[2][2])
    out = sum(w_ * t for w_, t in zip(ws, taps))
    mag = sum(w_ * t.abs() for w_, t in zip(ws, taps))
    gx = torch.stack([(V[j][i + 1] - V[j][i]).abs() for j in range(4) for i in range(3)]).amax(0)
    gy = torch.stack([(V[j + 1][i] - V[j][i]).abs() for j in range(3) for i in range(4)]).amax(0)
    return out, gx, gy, mag


def _zero_pad(img, b):
    """val(yy, xx) of bilerp on channel-last float64 images img [B, h, w, c] (query p in image b[p]), zeros outside."""
    h, w = img.shape[1], img.shape[2]

    def val(yy, xx):
        ok = (yy >= 0) & (yy < h) & (xx >= 0) & (xx < w)
        v = img[b.view(-1, *([1] * (yy.dim() - 1))).expand_as(yy), yy.clamp(0, h - 1), xx.clamp(0, w - 1)]
        return v * ok.unsqueeze(-1)
    return val


def _dot_val(a, img, b):
    """val(yy, xx) -> (a_p . img[b_p, yy, xx], sum |a_p||img|) stacked on the last dim, zeros outside the image."""
    sample = _zero_pad(img, b)

    def val(yy, xx):
        v = sample(yy, xx)
        return torch.stack((torch.einsum("pc,pkc->pk", a, v), torch.einsum("pc,pkc->pk", a.abs(), v.abs())), -1)
    return val


def _chunks(n, size=256):
    return [slice(i, min(i + size, n)) for i in range(0, n, size)]


def _logits(a, img, b, ix, iy, exact_coords, dot_n, h, w):
    """Scaled correlation logits a . bilinear(img, (ix, iy)) / sqrt(C) [P, K] and their bound."""
    v, gx, gy, mag = bilerp(_dot_val(a, img, b), ix, iy)
    s, A = v[..., 0] / SQRT_C, mag[..., 1] / SQRT_C
    ds = gamma(dot_n + (0 if exact_coords else BLEND_N)) * A + 2 * U32 * s.abs()
    if not exact_coords:
        ds = ds + (gx[..., 0] * coord_err(ix, w) + gy[..., 0] * coord_err(iy, h)) / SQRT_C
    return s, ds


def window_offsets(ry, rx):
    dy, dx = torch.meshgrid(torch.arange(-ry, ry + 1), torch.arange(-rx, rx + 1), indexing="ij")
    return dy.reshape(-1), dx.reshape(-1)


def local_corr_softmax64(f0, f1, ry, rx, stereo, pix, stencil):
    """local_correlation_softmax / _stereo (matching.py): softmax over the integer window (out-of-image taps excluded, weight
    exp(-1e9)) of f0 . f1 / sqrt(C), expectation of the tap coordinates minus the pixel's own; stereo returns x - E[x].
    f0, f1: [B, h, w, C] fp32, pix = (b, y, x) of the query pixels.  stencil: integer taps on exact coordinates and one FMA
    chain per dot product (um_local_stencil.cu); otherwise the gather kernel.  Returns (out, bound) [P, 2 or 1]."""
    B, h, w, _ = f0.shape
    f0d, f1d = f0.double(), f1.double()
    b, y, x = pix
    dy, dx = window_offsets(ry, rx)
    outs, bnds = [], []
    for sl in _chunks(b.numel()):
        bb, yy, xx = b[sl], y[sl], x[sl]
        sy, sx = yy[:, None] + dy, xx[:, None] + dx
        s, ds = _logits(f0d[bb, yy, xx], f1d, bb, sx.double(), sy.double(), stencil,
                        DOT_N_STENCIL if stencil else DOT_N_GATHER, h, w)
        valid = (sx >= 0) & (sx < w) & (sy >= 0) & (sy < h)
        s = torch.where(valid, s, torch.full_like(s, -math.inf))
        vals = torch.stack((sx, sy), -1).double()[..., :1 if stereo else 2]
        o, bd = softmax_weighted(s, ds, vals, tc_pv=False)
        own = torch.stack((xx, yy), -1).double()[:, :o.shape[-1]]
        o = own - o if stereo else o - own
        outs.append(o)
        bnds.append(bd + U32 * o.abs())
    return torch.cat(outs), torch.cat(bnds)


def as_flow2(flow):
    """[..., 2] flow or [..., 1] disparity -> float64 (u, v); a disparity d moves a pixel by (-d, 0)."""
    flow = flow.double()
    return flow if flow.shape[-1] == 2 else torch.cat((-flow, torch.zeros_like(flow)), -1)


def local_corr_volume64(f0, f1, flow, radius, pix):
    """local_correlation_with_flow (matching.py): f0 . bilinear(f1, (x + dx + u, y + dy + v)) / sqrt(C) for the (2r+1)^2
    offsets, zeros padding, exact coordinates.  The kernel blends all taps with the centre tap's weights, which is the same
    function of the same positions up to the coordinate rounding the bound carries.  Returns (out, bound) [P, (2r+1)^2]."""
    B, h, w, _ = f0.shape
    f0d, f1d, fl = f0.double(), f1.double(), as_flow2(flow)
    b, y, x = pix
    dy, dx = window_offsets(radius, radius)
    outs, bnds = [], []
    for sl in _chunks(b.numel()):
        bb, yy, xx = b[sl], y[sl], x[sl]
        u = fl[bb, yy, xx]
        ix = (xx.double() + u[:, 0])[:, None] + dx
        iy = (yy.double() + u[:, 1])[:, None] + dy
        s, ds = _logits(f0d[bb, yy, xx], f1d, bb, ix, iy, False, DOT_N_GATHER, h, w)
        outs.append(s)
        bnds.append(ds)
    return torch.cat(outs), torch.cat(bnds)


def flow_warp64(f, flow, pix):
    """bilinear_sample of f [B, h, w, C] at (x + u, y + v) (geometry.py: zeros padding, align_corners=True) -> (out, bound)
    [P, C]."""
    B, h, w, _ = f.shape
    fd, fl = f.double(), as_flow2(flow)
    b, y, x = pix
    outs, bnds = [], []
    for sl in _chunks(b.numel()):
        bb, yy, xx = b[sl], y[sl], x[sl]
        u = fl[bb, yy, xx]
        ix, iy = (xx.double() + u[:, 0])[:, None], (yy.double() + u[:, 1])[:, None]
        v, gx, gy, mag = bilerp(_zero_pad(fd, bb), ix, iy)
        bd = gamma(BLEND_N) * mag + gx * coord_err(ix, w)[..., None] + gy * coord_err(iy, h)[..., None]
        outs.append(v[:, 0])
        bnds.append(bd[:, 0])
    return torch.cat(outs), torch.cat(bnds)


def propagate_local64(q, k, flow, radius, pix):
    """SelfAttnPropagation.forward_local_window_attn (attention.py) on projected q / k [B, h, w, C] (any strides): softmax
    over the (2r+1)^2 window of q . k / sqrt(C), zero-padded unfold, so an out-of-image key is a zero vector with logit 0 and
    value 0.  Returns (out, bound) [P, fd]."""
    B, h, w, _ = q.shape
    qd, kd, fl = q.double(), k.double(), flow.double()
    b, y, x = pix
    dy, dx = window_offsets(radius, radius)
    outs, bnds = [], []
    for sl in _chunks(b.numel()):
        bb, yy, xx = b[sl], y[sl], x[sl]
        sy, sx = yy[:, None] + dy, xx[:, None] + dx
        kv = _zero_pad(kd, bb)(sy, sx)
        a = qd[bb, yy, xx]
        s = torch.einsum("pc,pkc->pk", a, kv) / SQRT_C
        ds = gamma(DOT_N_GATHER) * torch.einsum("pc,pkc->pk", a.abs(), kv.abs()) / SQRT_C + 2 * U32 * s.abs()
        o, bd = softmax_weighted(s, ds, _zero_pad(fl, bb)(sy, sx), tc_pv=False)
        outs.append(o)
        bnds.append(bd)
    return torch.cat(outs), torch.cat(bnds)


def _project64(K, Kinv, pose, x, y, depth):
    """warp_with_pose_depth_candidates (matching.py) in float64 on the fp32 camera matrices: pixel (x, y) [P] at depths
    [P, D] -> image positions (u, v) [P, D] (z clamped at 1e-3) and a bound of their fp32 rounding."""
    X = Kinv[:, :, 0] * x[:, None] + Kinv[:, :, 1] * y[:, None] + Kinv[:, :, 2]                       # [P, 3]
    Xa = Kinv[:, :, 0].abs() * x[:, None].abs() + Kinv[:, :, 1].abs() * y[:, None].abs() + Kinv[:, :, 2].abs()
    R, t = pose[:, :3, :3], pose[:, :3, 3]
    Xr = torch.einsum("prc,pc->pr", R, X)
    Xra = torch.einsum("prc,pc->pr", R.abs(), Xa)
    eXr = 6 * U32 * Xra                                                                               # two 3-term FMA chains
    Pt = Xr[:, None, :] * depth[..., None] + t[:, None, :]                                            # [P, D, 3]
    Pta = Xra[:, None, :] * depth[..., None] + t[:, None, :].abs()
    ePt = eXr[:, None, :] * depth[..., None] + 4 * U32 * Pta                                          # 1 / c, * and +
    pr = torch.einsum("prc,pdc->pdr", K, Pt)
    pra = torch.einsum("prc,pdc->pdr", K.abs(), Pta)
    epr = torch.einsum("prc,pdc->pdr", K.abs(), ePt) + 3 * U32 * pra
    z = pr[..., 2].clamp(min=1e-3)
    ez = torch.where(pr[..., 2] + epr[..., 2] >= 1e-3, epr[..., 2], torch.zeros_like(z))
    u, v = pr[..., 0] / z, pr[..., 1] / z
    eu = (epr[..., 0] + u.abs() * ez) / (z - ez).clamp(min=1e-3) + U32 * u.abs()
    ev = (epr[..., 1] + v.abs() * ez) / (z - ez).clamp(min=1e-3) + U32 * v.abs()
    return u, v, eu, ev


def depth_corr64(f0, f1, K, Kinv, pose, cand, pix):
    """correlation_softmax_depth (matching.py): f0 . bilinear(f1, project(pixel, 1 / c)) / sqrt(C) for every inverse-depth
    candidate c (zeros padding: a candidate projecting outside has logit 0), softmax over the candidates and the expected
    candidate.  Returns (softmax out [P], bound [P], logits [P, D], their bound [P, D])."""
    B, h, w, _ = f0.shape
    f0d, f1d = f0.double(), f1.double()
    Kd, Kid, Pd, cd = K.double(), Kinv.double(), pose.double(), cand.double()
    b, y, x = pix
    outs, bnds, ss, dss = [], [], [], []
    for sl in _chunks(b.numel(), 128):
        bb, yy, xx = b[sl], y[sl], x[sl]
        depth = (1.0 / cd)[None].expand(bb.numel(), -1)
        u, v, eu, ev = _project64(Kd[bb], Kid[bb], Pd[bb], xx.double(), yy.double(), depth)
        val, gx, gy, mag = bilerp(_dot_val(f0d[bb, yy, xx], f1d, bb), u, v)
        s, A = val[..., 0] / SQRT_C, mag[..., 1] / SQRT_C
        ds = (gamma(DOT_N_GATHER + BLEND_N) * A + 2 * U32 * s.abs() +
              (gx[..., 0] * (eu + coord_err(u, w)) + gy[..., 0] * (ev + coord_err(v, h))) / SQRT_C)
        o, bd = softmax_weighted(s, ds, cd[:, None], tc_pv=False)
        outs.append(o[:, 0])
        bnds.append(bd[:, 0])
        ss.append(s)
        dss.append(ds)
    return torch.cat(outs), torch.cat(bnds), torch.cat(ss), torch.cat(dss)


def argmax_admissible(s, ds):
    """[P, D] bool: the candidates a first-maximum argmax over logits within ds of s may return.  d qualifies if no earlier
    candidate is surely >= it and no later one surely > it; where the top two differ by more than their bounds only the
    true argmax qualifies."""
    lo, hi = s - ds, s + ds
    neg = torch.full_like(lo[:, :1], -math.inf)
    before = torch.cat((neg, torch.cummax(lo, 1).values[:, :-1]), 1)
    after = torch.cat((torch.cummax(lo.flip(1), 1).values.flip(1)[:, 1:], neg), 1)
    return (before < hi) & (after <= hi)


def check_argmax(name, got, cand, s, ds):
    """got [P] candidate values the kernel returned; every one must be admissible.  Prints how many were decided exactly."""
    got = got.detach().double().cpu().view(-1, 1)
    hit = got == cand.double().view(1, -1)
    assert (hit.sum(1) == 1).all(), "%s: output is not one of the candidates" % name
    adm = argmax_admissible(s, ds)
    ok = (hit & adm).any(1)
    exact = adm.sum(1) == 1
    print("%-60s argmax: %d of %d pixels decided exactly, %d near-tied" % (name, int(exact.sum()), got.shape[0],
                                                                          int((~exact).sum())))
    if not ok.all():
        i = int((~ok).nonzero()[0])
        raise AssertionError("%s: pixel %d chose candidate %d, admissible %s" % (
            name, i, int(hit[i].nonzero()), adm[i].nonzero().view(-1).tolist()))


def convex_upsample64(flow, mask, factor, mult, rows=None):
    """upsample_flow_with_mask (utils.py): softmax over the 9 mask logits of each sub-pixel, convex combination of the 3x3
    neighbourhood of mult * flow (zero-padded unfold, the softmax still over all 9).  flow [B, h, w, fd], mask
    [B, h, w, 9 F F] (logit t * F * F + ky * F + kx).  rows: low-resolution rows to evaluate.  Returns (out, bound)
    [B, fd, len(rows) * F, w * F]."""
    B, h, w, fd = flow.shape
    rows = torch.arange(h) if rows is None else rows
    F_ = factor
    m = mask.double()[:, rows].view(B, len(rows), w, 9, F_ * F_)
    e = torch.exp(m - m.amax(3, keepdim=True))
    p = e / e.sum(3, keepdim=True)
    fl = torch.nn.functional.pad(flow.double() * mult, (0, 0, 1, 1, 1, 1))                     # [B, h+2, w+2, fd]
    nb = torch.stack([fl[:, rows + ty][:, :, tx:tx + w] for ty in range(3) for tx in range(3)], 3)   # [B, R, w, 9, fd]
    o = torch.einsum("brwts,brwtd->brwsd", p, nb)
    pv = torch.einsum("brwts,brwtd->brwsd", p, nb.abs())
    dev = (nb[:, :, :, :, None, :] - o[:, :, :, None]).abs()                                  # [B, R, w, 9, FF, fd]
    arg = (m - m.amax(3, keepdim=True)).abs()
    bd = 24 * U32 * pv + torch.einsum("brwts,brwtsd->brwsd", p * (4 * U32 + U32 * arg), dev)
    bd = bd + UFLOW * nb.abs().sum(3, keepdim=True)                # weights near and below the fp32 underflow
    fix = lambda t: t.view(B, len(rows), w, F_, F_, fd).permute(0, 5, 1, 3, 2, 4).reshape(B, fd, len(rows) * F_, w * F_)
    return fix(o), fix(bd)


def upsample2x64(flow, mult):
    """F.interpolate(scale_factor=2, bilinear, align_corners=True) * mult of channel-last flow [B, h, w, fd] -> (out,
    bound) [B, 2h, 2w, fd]."""
    B, h, w, fd = flow.shape
    H, W = 2 * h, 2 * w
    fy = torch.arange(H, dtype=torch.float64) * ((h - 1) / (H - 1) if H > 1 else 0.0)
    fx = torch.arange(W, dtype=torch.float64) * ((w - 1) / (W - 1) if W > 1 else 0.0)
    iy, ix = (t.reshape(-1, 1) for t in torch.meshgrid(fy, fx, indexing="ij"))
    img = flow.double()

    def val(yy, xx):                                               # ATen clamps the second tap at the last row / column
        return img[:, yy.clamp(0, h - 1), xx.clamp(0, w - 1)].permute(1, 2, 0, 3)          # [H W, 1, B, fd]
    out, gx, gy, mag = (t.view(H, W, B, fd).permute(2, 0, 1, 3) for t in bilerp(val, ix, iy))
    bd = 6 * U32 * mag + gx * COORD_REL * (w - 1) + gy * COORD_REL * (h - 1)
    return out * mult, (bd + U32 * out.abs()) * abs(mult)


def add_position_ref(x, table, h, w):
    """feature_add_position: x + table[y mod wh, x mod ww] -- one fp32 addition per element, so the result is exact."""
    wh, ww = table.shape[0], table.shape[1]
    return x + table.repeat(h // wh, w // ww, 1)[None]


def conv7x7_64(x, weight, bias, stride, relu, scale=None, shift=None, pix=None):
    """The 7x7 stem / flow-encoder convolution, padding 3, on planar [N, cin, H, W] input: x * scale + shift per channel
    inside the image (the folded ImageNet normalisation), zeros outside, then + bias and ReLU.  The kernel is one fp32 FMA
    chain of 49 cin products per output.  Returns (out, bound) channel-last [N, Ho, Wo, cout], or [P, cout] at the output
    pixels pix = (b, y, x)."""
    xd = x.double()
    if scale is not None:
        xd = xd * torch.tensor(scale, dtype=torch.float32).double().view(1, -1, 1, 1) + \
             torch.tensor(shift, dtype=torch.float32).double().view(1, -1, 1, 1)
    wd = weight.double()
    if pix is None:
        y = torch.nn.functional.conv2d(xd, wd, None, stride=stride, padding=3).permute(0, 2, 3, 1)
        a = torch.nn.functional.conv2d(xd.abs(), wd.abs(), None, stride=stride, padding=3).permute(0, 2, 3, 1)
    else:
        p = patches(xd.permute(0, 2, 3, 1), 7, 7, stride, (3, 3), pix)
        y, a = p @ wd.flatten(1).T, p.abs() @ wd.flatten(1).abs().T
    e = gamma(49 * x.shape[1] + 3) * a
    if bias is not None:
        y = y + bias.double()
        e = e + gamma(49 * x.shape[1] + 3) * bias.double().abs()
    if relu:
        y = torch.relu(y)
    return y, e


def pixel_subset(B, h, w, gen, seam_x=(), seam_y=(), n_seam=2000, n_rand=300):
    """(b, y, x) of the pixels a reference is evaluated on: every border pixel, up to n_seam pixels on the columns / rows
    x mod sx in (0, sx - 1), y mod sy in (0, sy - 1) of the given tile seams, and n_rand random pixels."""
    ys, xs = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    border = (ys == 0) | (ys == h - 1) | (xs == 0) | (xs == w - 1)
    seam = torch.zeros_like(border)
    for s in seam_x:
        seam |= (xs % s == 0) | (xs % s == s - 1)
    for s in seam_y:
        seam |= (ys % s == 0) | (ys % s == s - 1)
    seam &= ~border
    idx = [border.reshape(-1).nonzero().view(-1)]
    si = seam.reshape(-1).nonzero().view(-1)
    idx.append(si[torch.randperm(si.numel(), generator=gen)[:n_seam]])
    idx = torch.cat(idx)
    flat = torch.cat([idx + i * h * w for i in range(B)] + [torch.randperm(B * h * w, generator=gen)[:n_rand]]).unique()
    return flat // (h * w), (flat % (h * w)) // w, flat % w


# ---- the assertion ------------------------------------------------------------------------------------------------
def check(name, got, ref, bound, locate=None):
    """max |got - ref| / bound <= 1 elementwise; prints the headroom; on failure names the worst element."""
    got = got.detach().double().cpu()
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    assert torch.isfinite(got).all(), "%s: non-finite output" % name
    err = (got - ref).abs()
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound).nan_to_num(nan=math.inf)
    worst = int(ratio.reshape(-1).argmax())
    idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(worst), ratio.shape))
    r = ratio.reshape(-1)[worst].item()
    print("%-60s max err/bound = %.3f" % (name, r))
    if r > 1.0:
        where = locate(idx) if locate else "index %s" % (idx,)
        raise AssertionError("%s: err/bound = %.3f at %s (got %.9g, ref %.9g, bound %.3g)" % (
            name, r, where, got[idx].item(), ref[idx].item(), bound[idx].item()))
    return r


def conv_locator(bn):
    def locate(idx):
        b, y, x, c = idx
        return "batch %d, y %d, x %d, channel tile %d (channel %d)" % (b, y, x, c // bn, c)
    return locate
