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
    """LayerNorm over the last dim (128) of y with per-element input bound e -> (out, bound)."""
    g, b = gamma.double(), beta.double()
    mean = y.mean(-1, keepdim=True)
    d = y - mean
    var = (d * d).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + EPS_LN)
    out = d * rstd * g + b
    em = e.mean(-1, keepdim=True)
    rho = ((d.abs() * (e + em)).sum(-1, keepdim=True) / (d * d + EPS_LN).sum(-1, keepdim=True) + 2.0 ** -21 +
           y.shape[-1] * U32 * (1 + mean.abs() * rstd))
    bound = g.abs() * rstd * (e + em) + g.abs() * d.abs() * rstd * rho + 4 * U32 * (g.abs() * d.abs() * rstd + b.abs())
    if res is not None:
        out = out + res.double()
        bound = bound + U32 * out.abs()
    return out, bound


# ---- convolution / Linear (um_conv2d_tc) ----------------------------------------------------------------------------
def _c2(x, w, stride, pad):
    return torch.nn.functional.conv2d(x, w, None, stride=stride, padding=pad)


def conv64(xs, wt, bias=None, pad=(0, 0), stride=1, mode=CONV_LINEAR, act=0, aux0=None, aux1=None, gamma=None, beta=None,
           pre=None):
    """xs: channel-last fp32 sources [B, H, W, c_i] (concatenated along channels), wt: fp32 [cout, sum c_i, kh, kw].
    Returns (out, bound) channel-last float64 [B, Ho, Wo, cout] of what um_conv2d_tc writes: GRU_ZR -> [z | r * h]."""
    x32 = torch.cat([x.float() for x in xs], -1).permute(0, 3, 1, 2)
    x, xh = x32.double(), split_sum(x32)
    w, wh = wt.double(), split_sum(wt)
    y = _c2(x, w, stride, pad)
    a = _c2(x.abs(), w.abs(), stride, pad)
    r = torch.sqrt(_c2(x * x, w * w, stride, pad))
    rep = _c2((x - xh).abs(), w.abs(), stride, pad) + _c2(xh.abs(), (w - wh).abs(), stride, pad)
    kh, kw = wt.shape[2], wt.shape[3]
    ktot = sum((c.shape[-1] + 63) // 64 * 64 for c in xs) * kh * kw
    nk = ktot // 64
    steps = 12 + nk if nk >= 8 else 12 * nk          # K >= 512: fresh accumulator per 64-wide stage, then fp32 adds
    e = G0 * a + steps * U_STEP * (y.abs() + WALK * r) + rep
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


def softmax_weighted(s, ds, vals, v_rep=None, tc_pv=True):
    """s: [M, N] scaled logits (-inf = excluded), ds: their bound, vals: [N, d] float64.  Returns (o, bound) [M, d].
    tc_pv: P V on the tensor cores (P split into fp16 (hi, lo), truncating accumulation over 64-key tiles); otherwise fp32
    CUDA-core sums of p * value."""
    smax = s.max(-1, keepdim=True).values
    e = torch.exp(s - smax)
    l = e.sum(-1, keepdim=True)
    p = e / l
    o = p @ vals
    va = vals.abs()
    pv = p @ va
    n = s.shape[-1]
    ds = torch.where(torch.isfinite(s), ds + U_STEP * (s.abs() + smax.abs()), torch.zeros_like(ds))
    pds = p * ds
    b = pds @ va + pds.sum(-1, keepdim=True) * o.abs()                   # sum_k p_k ds_k |v_k - o|
    b = b + 2 * G0 * pv + 2 * U32 * o.abs() + L_SUM * U32 * math.sqrt(n) * (o.abs() + pv)
    if tc_pv:
        tiles = (n + 63) // 64
        b = b + 12 * tiles * U_STEP * (o.abs() + WALK * torch.sqrt((p * p) @ (vals * vals)))
        b = b + 2.0 ** -22 * pv + 2.0 ** -25 / l * va.sum(0, keepdim=True)
    if v_rep is not None:
        b = b + p @ v_rep
    return o, b


def attention64(q, k, v, kv_shift, h, w, kh, kw, sh, sw, mask_mode, tc=True):
    """softmax(Q K^T / sqrt(128) + Swin mask) V per window with the cyclic shift and the roll back; key / value stream of
    stream n is (n + kv_shift) mod n_streams.  q, k, v: fp32 [n, h*w, 128].  Returns (out, bound, locate)."""
    n = q.shape[0]
    tok, reg = window_layout(h, w, kh, kw, sh, sw)
    nwin, lw = tok.shape
    out = torch.zeros((n, h * w, C), dtype=torch.float64)
    bnd = torch.zeros_like(out)
    for s_ in range(n):
        ks = (s_ + kv_shift) % n
        for wi in range(nwin):
            t = tok[wi]
            qw, kk, vv = q[s_, t], k[ks, t], v[ks, t]
            s, e = _logit_bound(qw, kk)
            s, e = s / math.sqrt(C), e / math.sqrt(C)
            if mask_mode == MASK_SWIN:
                m = reg[wi][:, None] != reg[wi][None, :]
                s = s - 100.0 * m
                e = e + U_STEP * 100.0 * m
            vd = vv.double()
            o, b = softmax_weighted(s, e, vd, (vd - split_sum(vv)).abs(), tc_pv=tc)
            out[s_, t] = o
            bnd[s_, t] = b

    pos = torch.empty(h * w, dtype=torch.long)
    win = torch.empty(h * w, dtype=torch.long)
    for wi in range(nwin):
        pos[tok[wi]] = torch.arange(lw)
        win[tok[wi]] = wi

    def locate(idx):
        st, t, c = idx
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
