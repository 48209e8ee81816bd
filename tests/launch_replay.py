"""Every launch of a forward, checked against float64 as it happens.

`Replay` stands in for `unimatch_b200.unimatch._OPS` (the op table the module calls, as `_Census` of
tests/test_kernel_edges_gpu.py does).  For each launch of an op in `CHECKS` it builds a signature (the op, its scalar
arguments, the shapes, strides and dtypes of its tensors); the first launch of every signature is checked, later ones (the
refinement iterations, the repeated transformer blocks) run unchecked.  A checked launch:

  1. copies every tensor argument to the host BEFORE the call (`pre`, the residual and in-place outputs alias inputs);
  2. runs the real op and copies its outputs back;
  3. compares them with the float64 reference and per-element bound of tests/ref64.py, reading fp16 (hi, lo) operand
     planes as hi + lo and bounding outputs written as planes with `split_out_bound`.

Large maps are evaluated on `ref64.pixel_subset` (every border pixel, the op's tile seams, random pixels), token rows on
their first rows, every row of the last (ragged) query tile and key tile, and random rows; windows on the first and last
windows and random ones.  Each check prints `max err/bound` and raises an AssertionError naming the op and its signature.

`NO_NUMERICS` lists the ops the module calls that compute nothing to check; tests/test_driver_resolutions_cpu.py requires
every `_OPS.<name>` of unimatch_b200/unimatch.py to be in one of the two tables."""
import inspect
import time

import torch

import ref64
from unimatch_b200 import ops

C = 128
TILE_Q = 128                  # query rows per tile of the attention / expectation kernels
TILE_K = 64                   # keys per tile
CONV_TILE = (8, 16)           # output pixels per tile of um_conv2d_tc (rows, columns)

NO_NUMERICS = {}              # op -> why it needs no check (the module calls none such today)


def host(t):
    """A host copy that shares no storage with t (also for a CPU tensor)."""
    return t.detach().to("cpu", copy=True)


def planes_value(p):
    """fp16 (hi, lo) planes [2, ...] -> the fp32 value hi + lo they hold."""
    return p[0].float() + p[1].float()


def describe(v):
    if isinstance(v, torch.Tensor):
        return ("tensor", tuple(v.shape), tuple(v.stride()), str(v.dtype))
    if isinstance(v, (list, tuple)):
        return tuple(v)
    return v


def signature(name, args):
    """(op, (argument, scalar or (shape, strides, dtype)) ...) of a launch; args: the bound arguments, defaults applied."""
    return (name,) + tuple((k, describe(v)) for k, v in args.items())


def short(sig):
    """The signature without the tensor tags, for messages."""
    return "%s(%s)" % (sig[0], ", ".join("%s=%s" % (k, v[1:] if isinstance(v, tuple) and v[:1] == ("tensor",) else v)
                                           for k, v in sig[1:]))


# ---- row / pixel subsets ---------------------------------------------------------------------------------------------
def tail_rows(n, tile):
    """Every row of the last tile of n rows (a whole tile when n is a multiple of it)."""
    return torch.arange((n - 1) // tile * tile, n)


def token_rows(n, gen, head=64, n_rand=256):
    """Rows of an [n, ...] token matrix to evaluate: the first `head`, every row of the last query and key tile, random."""
    return torch.cat((torch.arange(min(head, n)), tail_rows(n, TILE_Q), tail_rows(n, TILE_K),
                      torch.randperm(n, generator=gen)[:n_rand])).unique()


def attention_rows(h, w, kh, kw, sh, sw, gen, n_win=24, n_rand=16):
    """Query tokens of a windowed attention to evaluate: in the first two, the last two and random windows, the first 8
    positions, every position of the last query tile and random positions."""
    tok, _ = ref64.window_layout(h, w, kh, kw, sh, sw)
    nwin, lw = tok.shape
    wins = torch.cat((torch.tensor([0, 1, nwin - 2, nwin - 1]).clamp(0, nwin - 1),
                      torch.randperm(nwin, generator=gen)[:n_win])).unique()
    pos = torch.cat((torch.arange(min(8, lw)), tail_rows(lw, TILE_Q), torch.randperm(lw, generator=gen)[:n_rand])).unique()
    return tok[wins][:, pos].reshape(-1).sort().values


def grid_pixels(B, h, w, gen, seam_x=(), seam_y=()):
    return ref64.pixel_subset(B, h, w, gen, seam_x, seam_y, n_seam=1000, n_rand=300)


def rows_as_pixels(rows):
    """Token rows of a [rows / 16, 16] pixel grid (the tensor-core GEMM over token rows) -> (b, y, x)."""
    return torch.zeros_like(rows), rows // 16, rows % 16


# ---- the checks (one per op; `a` = host copies of the arguments taken before the call, `out` = the op's return) ----------
class _Check:
    def __init__(self, replay, name, sig, a, live, out):
        self.replay, self.name, self.sig, self.a, self.live, self.out = replay, name, sig, a, live, out
        self.gen = torch.Generator().manual_seed(len(replay.checked) + 17)
        self.worst = 0.0

    def check(self, what, got, ref, bound, locate=None):
        label = "%s #%d %s" % (self.name, len(self.replay.checked), what)
        try:
            r = ref64.check(label, got, ref, bound, locate)
        except AssertionError as e:
            raise AssertionError("%s: %s\n  signature: %s" % (self.name, e, short(self.sig))) from None
        self.worst = max(self.worst, r)

    def exact(self, what, got, ref):
        label = "%s #%d %s" % (self.name, len(self.replay.checked), what)
        if not torch.equal(got, ref):
            d = (got.double() - ref.double()).abs()
            raise AssertionError("%s: %s not bit-exact, max |diff| %.3g\n  signature: %s" % (self.name, label, d.max(),
                                                                                              short(self.sig)))
        print("%-60s bit-exact" % label)

    def result(self, key):
        """the live output argument `key`, read back after the call"""
        return host(self.live[key])


def check_conv2d_tc(c):
    a = c.a
    kh, kw, cout, mode, stride, rows = a["kh"], a["kw"], a["cout"], a["mode"], a["stride"], a["rows"]
    srcs = [s for s in (a["src0"], a["src1"]) if s is not None]
    if rows:
        xs = [planes_value(s[:, :rows]).view(1, rows // 16, 16, s.shape[-1]) for s in srcs]
        grid = lambda t: None if t is None else t[:rows].reshape(1, rows // 16, 16, t.shape[-1])
    else:
        xs = [planes_value(s) for s in srcs]
        grid = lambda t: t
    wv = planes_value(a["weights"])                                    # [cout_p, ktot], K = (source, tap, channel)
    blocks, off = [], 0
    for x in xs:
        n = kh * kw * x.shape[-1]
        blocks.append(wv[:, off:off + n].view(wv.shape[0], kh, kw, x.shape[-1]).permute(0, 3, 1, 2))
        off += n
    wt = torch.cat(blocks, 1)[:cout].contiguous()
    _, Hi, Wi, _ = xs[0].shape
    ho, wo = (Hi + 2 * a["pad_h"] - kh) // stride + 1, (Wi + 2 * a["pad_w"] - kw) // stride + 1
    if rows:
        r = token_rows(rows, c.gen)
        pix = rows_as_pixels(r)
        at = lambda t: t[r]
    else:
        pix = grid_pixels(xs[0].shape[0], ho, wo, c.gen, (CONV_TILE[1],), (CONV_TILE[0],))
        at = lambda t: t[pix]
    ref, bnd = ref64.conv64(xs, wt, a["bias"], (a["pad_h"], a["pad_w"]), stride, mode, a["act"], grid(a["aux0"]),
                            grid(a["aux1"]), a["gamma"], a["beta"], grid(a["pre"]), pix)
    loc = lambda idx: "pixel (b %d, y %d, x %d), channel %d" % (int(pix[0][idx[0]]), int(pix[1][idx[0]]),
                                                                 int(pix[2][idx[0]]), idx[1])
    zr = mode == ops.CONV_GRU_ZR
    # output channel ranges: GRU_ZR writes z (fp32) and r * h (planes); the others write every channel to both
    f_cols, s_cols = ((0, 128), (128, 256)) if zr else ((0, cout), (0, cout))
    win = a["win_dst"] is not None
    wc0, wc1 = (a["win_c0"], a["win_c1"]) if win else (0, 0)
    if a["out_f32"] is not None:
        got = at(c.result("out_f32"))
        cols = [ch for ch in range(*f_cols) if not wc0 <= ch < wc1]
        if cols:
            sel = torch.tensor(cols)
            c.check("out_f32", got[:, a["off_f32"] + sel - f_cols[0]], ref[:, sel], bnd[:, sel], loc)
    if a["out_split"] is not None:
        o = c.live["out_split"]
        got = at(planes_value(host(o[:, :rows] if rows else o)))
        lo_, hi_ = s_cols
        got = got[:, a["off_split"]:a["off_split"] + hi_ - lo_]
        c.check("out_split", got, ref[:, lo_:hi_], ref64.split_out_bound(ref[:, lo_:hi_], bnd[:, lo_:hi_]), loc)
    if win:
        h, w, wkh, wkw, sh, sw, _ = a["win_geom"]
        tok, _ = ref64.window_layout(h, w, wkh, wkw, sh, sw)
        lw = tok.shape[1]
        where = torch.empty(h * w, dtype=torch.long)                   # token -> window * lw + position
        where[tok.reshape(-1)] = torch.arange(tok.numel())
        dst = c.result("win_dst")                                      # [ops, 2, streams, windows, lp, 128]
        keep = r < a["win_streams"] * h * w
        st, t = r[keep] // (h * w), r[keep] % (h * w)
        for o in range((wc1 - wc0) // 128):
            pl = dst[o][:, :, :, :lw].reshape(2, a["win_streams"], -1, C)[:, st, where[t]]
            ch = slice(wc0 + 128 * o, wc0 + 128 * (o + 1))
            c.check("window planes %d" % o, planes_value(pl), ref[keep][:, ch],
                    ref64.split_out_bound(ref[keep][:, ch], bnd[keep][:, ch]))


def check_window_attention(c):
    a = c.a
    geo = (a["h"], a["w"], a["kh"], a["kw"], a["sh"], a["sw"], a["mask_mode"])
    rows = attention_rows(*geo[:6], c.gen)
    tc = ops.attention_planes_lp(*geo) > 0 and not ops._force_cuda_cores
    ref, bnd, loc = ref64.attention64(a["q"], a["k"], a["v"], a["kv_shift"], *geo, tc=tc, rows=rows)
    c.check("out", host(c.out)[:, rows], ref, bnd, loc)


def _from_planes(p, n, h, w, geo):
    """window-major (hi, lo) planes [2, n, windows, lp, 128] -> fp32 tokens [n, h*w, 128]"""
    tok, _ = ref64.window_layout(h, w, *geo)
    lw = tok.shape[1]
    out = torch.empty((n, h * w, C))
    out[:, tok.reshape(-1)] = planes_value(p)[:, :, :lw].reshape(n, -1, C)
    return out


def check_window_attention_planes(c):
    a = c.a
    n, h, w = a["n"], a["h"], a["w"]
    geo = (a["kh"], a["kw"], a["sh"], a["sw"])
    q, k, v = (_from_planes(a[x], n, h, w, geo) for x in ("qp", "kp", "vp"))
    rows = attention_rows(h, w, *geo, c.gen)
    ref, bnd, loc = ref64.attention64(q, k, v, a["kv_shift"], h, w, *geo, a["mask_mode"], rows=rows)
    if a["out_f32"] is not None:
        got = c.result("out_f32")[:n * h * w].view(n, h * w, C)[:, rows]
        c.check("out_f32", got, ref, bnd, loc)
    if a["out_split"] is not None:
        got = planes_value(c.result("out_split"))[:n * h * w].view(n, h * w, C)[:, rows]
        c.check("out_split", got, ref, ref64.split_out_bound(ref, bnd), loc)


def expectation_rows(L, h, w, kh, gen):
    """token_rows, and for one window per image row (kh = h) every token of the first, the last and two random rows"""
    rows = token_rows(L, gen)
    if kh != 1:
        ys = torch.cat((torch.tensor([0, h - 1]), torch.randint(0, h, (2,), generator=gen)))
        rows = torch.cat((rows, (ys[:, None] * w + torch.arange(w)).reshape(-1))).unique()
    return rows


def check_softmax_expectation(c):
    a = c.a
    L = a["q"].shape[1]
    rows = expectation_rows(L, a["h"], a["w"], a["kh"], c.gen)
    ref, bnd = ref64.expectation64(a["q"], a["k"], a["values"], a["n_streams"], a["kv_shift"], a["vdim"], a["value_mode"],
                                   a["post_op"], a["h"], a["w"], a["kh"], a["kw"], a["mask_mode"], rows)
    loc = lambda idx: "stream %d, token %d (query tile %d), column %d" % (idx[0], int(rows[idx[1]]), int(rows[idx[1]]) // TILE_Q,
                                                                          idx[2])
    c.check("out", host(c.out)[:, rows], ref, bnd, loc)


def check_ffn_tc(c):
    a = c.a
    rows = a["rows"]
    hidden = a["w1"].shape[1]
    w1 = planes_value(a["w1"]).view(hidden, 256, 1, 1)
    w2 = planes_value(a["w2"]).view(C, hidden, 1, 1)
    r = token_rows(rows, c.gen, head=256, n_rand=512)
    x0, x1 = (planes_value(a[s][:, r]) for s in ("src0", "src1"))
    res = a["residual"][r] if a["residual"] is not None else torch.zeros_like(x0)
    ref, bnd = ref64.ffn64(x0, x1, w1, w2, res, a["gamma"], a["beta"])
    loc = lambda idx: "row %d (tile %d), channel %d" % (int(r[idx[0]]), int(r[idx[0]]) // TILE_Q, idx[1])
    if a["out_f32"] is not None:
        c.check("out_f32", c.result("out_f32")[r], ref, bnd, loc)
    if a["out_split"] is not None:
        c.check("out_split", planes_value(c.result("out_split")[:, r]), ref, ref64.split_out_bound(ref, bnd), loc)


def check_instance_norm_stats(c):
    x = c.a["x"]
    st = host(c.out).double()
    for i in range(x.shape[0]):                                        # one image at a time: bounded host memory
        mean, rstd, sd = ref64.instance_norm_stats64(x[i:i + 1])
        c.check("rstd image %d" % i, st[i:i + 1, 1], rstd, 1e-6 * rstd)
        c.check("mean image %d" % i, st[i:i + 1, 0], mean, 2.0 ** -24 * mean.abs() + 2.0 ** -22 * sd)


def check_instance_norm_apply(c):
    """y = [ReLU]((a - mean) rstd) + [(res - mean_r) rstd_r | res], [ReLU], with the given statistics: a few fp32
    operations per element, bounded by 4 ulp of every term's magnitude."""
    a = c.a
    x = a["a"]
    n, cc = x.shape[0], x.shape[-1]
    x = x.reshape(n, -1, cc)
    hw = x.shape[1]
    p = token_rows(hw, c.gen, n_rand=512)                              # per image: first, last and random pixels
    b, p = torch.arange(n).repeat_interleave(p.numel()), p.repeat(n)
    U = ref64.U32

    def norm(t, st):
        t = t.reshape(n, -1, cc)[b, p].double()
        if st is None:
            return t, t.abs()
        m, rs = st[b, 0].double(), st[b, 1].double()
        return (t - m) * rs, (t.abs() + m.abs()) * rs
    y, mag = norm(a["a"], a["stats_a"])
    if a["relu_a"]:
        y = torch.relu(y)
    if a["res"] is not None:
        yr, mr = norm(a["res"], a["stats_res"])
        y, mag = y + yr, mag + mr
    if a["relu_out"]:
        y = torch.relu(y)
    bnd = 4 * U * (mag + y.abs())
    if a["out_f32"] is not None:
        c.check("out_f32", c.result("out_f32").reshape(n, hw, -1)[b, p][:, :cc], y, bnd)
    if a["out_split"] is not None:
        o = c.result("out_split")
        got = planes_value(o.reshape(2, n, hw, o.shape[-1])[:, b, p])[:, a["off"]:a["off"] + cc]
        c.check("out_split", got, y, ref64.split_out_bound(y, bnd))


def check_split_planes(c):
    a = c.a
    src = a["src"].reshape(-1, a["src"].shape[-1])
    rows, cc = src.shape
    cp = a["dst"].shape[-1]
    dst = c.result("dst").reshape(2, -1, cp)[:, :rows, a["off"]:a["off"] + cc]
    hi = src.half()
    c.exact("hi", dst[0], hi)
    c.exact("lo", dst[1], (src - hi.float()).half())


def _maps(t, h, w):
    return t.reshape(t.shape[0], h, w, t.shape[-1])


def check_local_corr_softmax(c):
    a = c.a
    h, w = a["h"], a["w"]
    f0, f1 = _maps(a["f0"], h, w), _maps(a["f1"], h, w)
    stencil = not a["stereo"] and a["ry"] == 4 and a["rx"] == 4
    pix = grid_pixels(f0.shape[0], h, w, c.gen, (32,) if stencil else (), (8,) if stencil else ())
    ref, bnd = ref64.local_corr_softmax64(f0, f1, a["ry"], a["rx"], a["stereo"], pix, stencil)
    c.check("out", host(c.out)[pix], ref, bnd)


def check_local_corr_volume(c):
    a = c.a
    h, w = a["h"], a["w"]
    f0, f1 = _maps(a["f0"], h, w), _maps(a["f1"], h, w)
    pix = grid_pixels(f0.shape[0], h, w, c.gen)
    ref, bnd = ref64.local_corr_volume64(f0, f1, _maps(a["flow"], h, w), a["radius"], pix)
    c.check("out", host(c.out)[pix], ref, bnd)


def check_flow_warp(c):
    a = c.a
    h, w = a["h"], a["w"]
    f = _maps(a["f"], h, w)
    pix = grid_pixels(f.shape[0], h, w, c.gen)
    ref, bnd = ref64.flow_warp64(f, _maps(a["flow"], h, w), pix)
    c.check("out", _maps(host(c.out), h, w)[pix], ref, bnd)


def check_propagate_local(c):
    a = c.a
    h, w = a["h"], a["w"]
    q, k = _maps(a["q"], h, w), _maps(a["k"], h, w)
    pix = grid_pixels(q.shape[0], h, w, c.gen)
    ref, bnd = ref64.propagate_local64(q, k, _maps(a["flow"], h, w), a["radius"], pix)
    c.check("out", _maps(host(c.out), h, w)[pix], ref, bnd)


def check_depth_corr_softmax(c):
    a = c.a
    h, w = a["h"], a["w"]
    f0, f1 = _maps(a["f0"], h, w), _maps(a["f1"], h, w)
    pix = grid_pixels(f0.shape[0], h, w, c.gen)
    ref, bnd, s, ds = ref64.depth_corr64(f0, f1, a["K"], a["Kinv"], a["pose"], a["cand"], pix)
    got = host(c.out)[..., 0][pix]
    if a["from_argmax"]:
        ref64.check_argmax("%s #%d argmax" % (c.name, len(c.replay.checked)), got, a["cand"], s, ds)
    else:
        c.check("softmax", got, ref, bnd)


def check_convex_upsample(c):
    a = c.a
    fl, mask, F = a["flow"], a["mask"], a["factor"]
    h = fl.shape[1]
    rows = torch.cat((torch.tensor([0, 1, h - 2, h - 1]).clamp(0, h - 1), torch.randperm(h, generator=c.gen)[:6])).unique()
    ref, bnd = ref64.convex_upsample64(fl, mask, F, a["mult"], rows)
    sel = (rows[:, None] * F + torch.arange(F)).reshape(-1)
    c.check("out", host(c.out)[:, :, sel], ref, bnd)


def check_upsample2x(c):
    ref, bnd = ref64.upsample2x64(c.a["flow"], c.a["mult"])
    c.check("out", host(c.out), ref, bnd)


def check_add_position(c):
    a = c.a
    x = _maps(a["x"], a["h"], a["w"])
    c.exact("out", _maps(host(c.out), a["h"], a["w"]), ref64.add_position_ref(x, a["table"], a["h"], a["w"]))


def check_conv7x7_small(c):
    a = c.a
    if a["nchw"]:
        x = a["in0"] if a["in1"] is None else torch.cat((a["in0"], a["in1"]), 0)
    else:
        x = a["in0"].permute(0, 3, 1, 2)
    N, _, H, W = x.shape
    s = a["stride"]
    ho, wo = (H - 1) // s + 1, (W - 1) // s + 1
    pix = grid_pixels(N, ho, wo, c.gen, (8, 32), (8, 32))
    ref, bnd = ref64.conv7x7_64(x, a["weight"], a["bias"], s, a["relu"], a["scale"], a["shift"], pix)
    if a["out_f32"] is not None:
        c.check("out_f32", c.result("out_f32")[pix], ref, bnd)
    if a["out_split"] is not None:
        got = planes_value(c.result("out_split")[:, pix[0], pix[1], pix[2]])
        c.check("out_split", got, ref, ref64.split_out_bound(ref, bnd))


CHECKS = {name[len("check_"):]: fn for name, fn in list(globals().items()) if name.startswith("check_")}


class Replay:
    """Stands in for torch.ops.unimatch_sm100 in unimatch_b200.unimatch (see the module docstring).  `only`: check just
    these ops (the others run unchecked).  `checked`: [(signature, worst err/bound)] in launch order; `host_s`: seconds
    spent copying arguments and evaluating the references."""

    def __init__(self, real, only=None):
        self.real, self.only = real, only
        self.seen, self.checked, self.host_s = set(), [], 0.0

    def __getattr__(self, name):
        fn = getattr(self.real, name)
        if name not in CHECKS or (self.only is not None and name not in self.only):
            return fn
        params = inspect.signature(getattr(ops, "_" + name))

        def wrapped(*args, **kwargs):
            bound = params.bind(*args, **kwargs)
            bound.apply_defaults()
            live = dict(bound.arguments)
            sig = signature(name, live)
            if sig in self.seen:
                return fn(*args, **kwargs)
            self.seen.add(sig)
            t0 = time.perf_counter()
            pre = {k: host(v) if isinstance(v, torch.Tensor) else v for k, v in live.items()}
            t1 = time.perf_counter()
            out = fn(*args, **kwargs)
            t2 = time.perf_counter()
            chk = _Check(self, name, sig, pre, live, out)
            CHECKS[name](chk)
            self.checked.append((sig, chk.worst))
            self.host_s += time.perf_counter() - t2 + t1 - t0
            return out
        return wrapped
