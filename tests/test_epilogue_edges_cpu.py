"""The GEMM epilogue functions -- exact-erf GELU, the fast tanh / sigmoid, the two LayerNorm epilogues and the fused FFN --
checked on the CPU against their float64 references in tests/ref64.py, over the inputs tests/test_epilogue_edges_gpu.py
feeds the kernels:
  * an fp32 emulation of each epilogue (the kernels' formulas, fast intrinsics modelled as below) passes its bound;
  * the same emulation with one defect injected fails it, or the docstring says why the bound cannot see that defect.

Intrinsics: ex2.approx.ftz is modelled as the correctly rounded 2^x with results below 2^-126 flushed to 0 (the hardware
adds up to 2 ulp, which the GPU tests measure); __expf(x) = ex2(fl(x * log2 e)); __fdividef(a, b) = a * fl(1 / b), and 0
for 2^126 < |b| < 2^128, as the CUDA programming guide documents; fmaf is the exact product plus c rounded once."""
import math

import numpy as np
import pytest
import torch

import ref64

C = 128
F32 = torch.float32
FLT_MAX = float(np.finfo(np.float32).max)
LOG2E = 1.4426950408889634


def g(seed):
    return torch.Generator().manual_seed(seed)


def hl(x):
    x = x.float()
    hi = x.half().float()
    return hi, (x - hi).half().float()


def f32(x):
    return torch.as_tensor(x, dtype=torch.float64).float()


def fma(a, b, c):
    """fmaf: the product of two fp32 values is exact in float64; the sum is rounded to fp32 (via float64, which double
    rounds only on exact float64 ties -- never met by these inputs at the precision the bounds look at)."""
    return (a.double() * b.double() + c.double()).float()


def rejects(name, got, ref, bound):
    with pytest.raises(AssertionError):
        ref64.check(name, got, ref, bound)


# ---- the activation sweep (§ a of the GPU tests) ----------------------------------------------------------------------
def act_sweep():
    """fp32 arguments of the activation sweep, all finite: a dense grid over [-16, 16] at step 2^-12; log-spaced
    magnitudes 2^-30 ... 2^100 of both signs; +-0 and fp32 subnormals; the neighbourhoods of GELU's clamp (|y| = 8.5) and
    of the end of its stated range (|y| = 12); tanh's __fdividef window (1 + e^2y in (2^126, 2^128): y in 43.6 ... 44.4);
    sigmoid's (y in -88.8 ... -87.3); +-FLT_MAX."""
    parts = [torch.arange(-16 * 4096, 16 * 4096 + 1, dtype=torch.float64) / 4096]
    mags = 2.0 ** torch.linspace(-30, 100, 2601, dtype=torch.float64)
    parts += [mags, -mags]
    sub = torch.tensor([2.0 ** -149, 2.0 ** -140, 2.0 ** -130, 2.0 ** -127, 2.0 ** -126 * (1 - 2.0 ** -23)],
                       dtype=torch.float64)
    parts += [torch.tensor([0.0, -0.0], dtype=torch.float64), sub, -sub]
    for c in (8.5, 12.0):
        near = torch.tensor(np.nextafter(np.float32(c), np.float32(np.inf)).item(), dtype=torch.float64)
        ulp = near - c
        k = torch.arange(-256, 257, dtype=torch.float64)
        parts += [c + k * ulp, -(c + k * ulp), c + k / 2 ** 16, -(c + k / 2 ** 16)]
    parts.append(torch.linspace(43.6, 44.4, 4097, dtype=torch.float64))
    parts.append(torch.linspace(-88.8, -87.3, 4097, dtype=torch.float64))
    parts.append(torch.tensor([FLT_MAX, -FLT_MAX], dtype=torch.float64))
    return f32(torch.cat(parts))


# ---- fp32 emulations of the fast activations (um_tc.cuh act_gelu, um_conv_tc.cu sigmoid_fast / tanh_fast) ------------
GELU_Q = (3.151970304e-06, 2.940293484e-07, -6.359316176e-04, 7.810713258e-03, -5.312381312e-02, -4.589283466e-01,
          -1.151162863e+00, -9.999961257e-01)


def ex2(x):
    x = x.float()
    x = torch.where(x.abs() < 2.0 ** -126, torch.zeros_like(x), x)       # .ftz: subnormal inputs are 0
    r = f32(torch.exp2(x.double()))
    return torch.where(r.abs() < 2.0 ** -126, torch.zeros_like(r), r)    # .ftz: subnormal results are 0


def expf_fast(x):
    return ex2(x.float() * f32(LOG2E))


def fdividef(a, b):
    a, b = torch.broadcast_to(f32(a), b.shape), b.float()
    q = a * f32(1.0 / b.double())
    return torch.where((b.abs() > 2.0 ** 126) & (b.abs() < 2.0 ** 128), torch.zeros_like(q), q)


def gelu_fast(y):
    y = y.float()
    a = torch.clamp(y.abs(), max=8.5)
    q = torch.full_like(a, GELU_Q[0])
    for c in GELU_Q[1:]:
        q = fma(q, a, torch.full_like(a, c))
    return fma(-y.abs(), ex2(q), torch.clamp(y, min=0.0))


def tanh_fast(y):
    return 1.0 - fdividef(2.0, 1.0 + expf_fast(2.0 * y.float()))


def sigmoid_fast(y):
    return fdividef(1.0, 1.0 + expf_fast(-y.float()))


def gelu_tanh_form(y):
    """defect: the tanh approximation of GELU (nn.GELU(approximate="tanh")) instead of the exact-erf one."""
    y = y.float()
    return 0.5 * y * (1.0 + torch.tanh(f32(math.sqrt(2.0 / math.pi)) * (y + f32(0.044715) * y * y * y)))


def tanh_unguarded(y):
    """defect: tanh = (e^2y - 1) / (e^2y + 1), with no guard for e^2y overflowing (y > 44.4: inf / inf)."""
    e = expf_fast(2.0 * y.float())
    return (e - 1.0) / (e + 1.0)


FAST = {"gelu": gelu_fast, "tanh": tanh_fast, "sigmoid": sigmoid_fast}


def act_report(name, got, y):
    """worst |got - exact| over the sweep and its argument"""
    ref = ref64.act64(y.double(), name)
    err = (got.double() - ref).abs()
    i = int(err.argmax())
    return err[i].item(), y[i].item()


@pytest.mark.parametrize("name", ["gelu", "tanh", "sigmoid"])
def test_fast_activations_pass_act_bound_on_sweep(name):
    y = act_sweep()
    ref, bnd = ref64.act_bound(y.double(), torch.zeros(y.shape, dtype=torch.float64), name)
    got = FAST[name](y)
    ref64.check("%s emulation on the sweep" % name, got, ref, bnd)
    inr = y.abs() <= 12
    err, arg = act_report(name, got[inr], y[inr])
    print("%s emulation: worst |err| %.3g at y = %.9g (|y| <= 12)" % (name, err, arg))


def test_gelu_fit_meets_its_stated_error():
    """um_tc.cuh states |act_gelu - exact| <= 2.7e-7 for |y| <= 12.  With exact exp2, the fitted polynomial and its fp32
    evaluation alone must stay inside that figure (the GPU tests add ex2.approx's own error)."""
    y = act_sweep()
    y = y[y.abs() <= 12]
    err, arg = act_report("gelu", gelu_fast(y), y)
    print("gelu fit (exact exp2): worst |err| %.3g at y = %.9g" % (err, arg))
    assert err <= 2.7e-7, (err, arg)


def test_act_bound_rejects_tanh_form_gelu():
    y = act_sweep()
    ref, bnd = ref64.act_bound(y.double(), torch.zeros(y.shape, dtype=torch.float64), "gelu")
    rejects("tanh-form gelu", gelu_tanh_form(y), ref, bnd)


def test_act_bound_rejects_unguarded_tanh():
    """The unguarded quotient overflows to inf / inf = NaN in tanh's __fdividef window and beyond; the check refuses
    non-finite outputs."""
    y = act_sweep()
    got = tanh_unguarded(y)
    assert torch.isnan(got[(y > 44.4) & (y < 1e30)]).all()
    ref, bnd = ref64.act_bound(y.double(), torch.zeros(y.shape, dtype=torch.float64), "tanh")
    rejects("unguarded tanh", got, ref, bnd)


# ---- LayerNorm rows (§ b of the GPU tests) ---------------------------------------------------------------------------
# family name -> rows built from standard-normal z [n, 128] and per-row signs s (every value exact in fp16 after
# fp16 rounding, so a GEMM with an identity weight reproduces the row exactly)
LN_FAMILIES = {
    "mean/std 0": lambda z, s: z,
    "mean/std 10": lambda z, s: 10.0 * s + z,
    "mean/std 1e2": lambda z, s: 1e2 * s + z,
    "mean/std 1e3": lambda z, s: 1e3 * s + z,
    "std 1": lambda z, s: z,
    "std 1e-2": lambda z, s: 1e-2 * z,
    "std 3e-3": lambda z, s: 3e-3 * z,
    "std 1e-3": lambda z, s: 1e-3 * z,
    "constant": lambda z, s: (z[:, :1] * 2.0 ** torch.arange(-8, 8, 2).repeat(z.shape[0])[:z.shape[0], None]).expand_as(z),
    "outlier channel x100": lambda z, s: torch.cat((z[:, :37], 100.0 * z[:, 37:38], z[:, 38:]), 1),
    "mag 2^-8": lambda z, s: 2.0 ** -8 * z,
    "mag 2^-4": lambda z, s: 2.0 ** -4 * z,
    "mag 2^4": lambda z, s: 2.0 ** 4 * z,
    "mag 2^8": lambda z, s: 2.0 ** 8 * z,
    "mag 2^12": lambda z, s: 2.0 ** 12 * z,
}


def ln_rows(family, n, seed, positive=False):
    """[n, 128] fp32 rows of a family, exact in fp16.  positive: the mean offsets all positive (the FFN's rows, where
    GELU is the identity for large positive arguments)."""
    gen = g(seed)
    z = torch.randn((n, C), generator=gen)
    s = torch.ones((n, 1)) if positive else torch.where(torch.rand((n, 1), generator=gen) < 0.5, -1.0, 1.0)
    return LN_FAMILIES[family](z, s).contiguous().half().float()


def ln_params(kind, seed):
    """gamma, beta: "random" (standard normal) or "identity" (1, 0)"""
    if kind == "identity":
        return torch.ones(C), torch.zeros(C)
    gen = g(seed)
    return torch.randn(C, generator=gen), torch.randn(C, generator=gen)


def _seqsum(v):
    s = torch.zeros(v.shape[:-1], dtype=F32)
    for i in range(v.shape[-1]):
        s = s + v[..., i]
    return s


HALVES = (list(range(0, 32)) + list(range(64, 96)), list(range(32, 64)) + list(range(96, 128)))


def emu_layernorm(y, gamma, beta, res=None, defect=None):
    """The conv UM_CONV_LN epilogue in fp32: two partial sums over channels {0-31, 64-95} and {32-63, 96-127} for the mean,
    then the centred sum of squares as FMAs, rsqrt(var + 1e-5) (rsqrtf modelled as correctly rounded), then
    (y - mean) * rstd * gamma + beta, + residual.
    defects: "one_pass" var = E[y^2] - mean^2 in fp32; "no_eps" / "eps1e-6"; "res_first" residual added before the
    normalisation."""
    y = y.float()
    if defect == "res_first" and res is not None:
        y = y + res
    mean = (_seqsum(y[:, HALVES[0]]) + _seqsum(y[:, HALVES[1]])) * f32(1.0 / C)
    if defect == "one_pass":
        sq = _seqsum(y[:, HALVES[0]] * y[:, HALVES[0]]) + _seqsum(y[:, HALVES[1]] * y[:, HALVES[1]])
        var = torch.clamp(sq * f32(1.0 / C) - mean * mean, min=0.0)
    else:
        parts = []
        for idx in HALVES:
            s = torch.zeros(y.shape[0], dtype=F32)
            for i in idx:
                d = y[:, i] - mean
                s = fma(d, d, s)
            parts.append(s)
        var = (parts[0] + parts[1]) * f32(1.0 / C)
    eps = {"no_eps": 0.0, "eps1e-6": 1e-6}.get(defect, 1e-5)
    rstd = f32(1.0 / torch.sqrt((var + f32(eps)).double()))
    out = (y - mean[:, None]) * rstd[:, None] * gamma + beta
    if res is not None and defect != "res_first":
        out = out + res
    return out


def _ln_case(family, params, with_res, seed, exact=True):
    y = ln_rows(family, 64, seed)
    if not exact:                                      # rows as fp32 GEMM outputs: the fp32 mean is no longer exact
        y = (y + torch.randn(y.shape, generator=g(seed + 1)) * y.abs() * 2.0 ** -14).float()
    gamma, beta = ln_params(params, seed + 2)
    res = torch.randn((64, C), generator=g(seed + 3)) if with_res else None
    ref, bnd = ref64.layernorm64(y.double(), torch.zeros(y.shape, dtype=torch.float64), gamma, beta, res)
    return y, gamma, beta, res, ref, bnd


@pytest.mark.parametrize("with_res", [True, False])
@pytest.mark.parametrize("params", ["random", "identity"])
@pytest.mark.parametrize("family", list(LN_FAMILIES))
def test_layernorm64_passes_emulation_on_row_families(family, params, with_res):
    """Exact input (e = 0): the bound has to carry the fp32 statistics alone.  Rows exact in fp16 (what the GPU tests
    feed through an identity weight) and the same rows perturbed to full fp32 precision (what a GEMM hands the
    epilogue), where the fp32 row mean is inexact."""
    seed = 300 + list(LN_FAMILIES).index(family)
    for exact in (True, False):
        y, gamma, beta, res, ref, bnd = _ln_case(family, params, with_res, seed, exact)
        ref64.check("layernorm %s %s res %s %s" % (family, params, with_res, "fp16" if exact else "fp32"),
                    emu_layernorm(y, gamma, beta, res), ref, bnd)


def test_layernorm_constant_rows_are_beta_plus_residual():
    """A constant row of fp16-exact values has an exact fp32 mean, centred values 0 and output beta (+ residual) bit for
    bit -- the zero padding rows of the transformer's token buffers are such rows."""
    y = ln_rows("constant", 64, 310)
    gamma, beta = ln_params("random", 311)
    res = torch.randn((64, C), generator=g(312))
    assert torch.equal(emu_layernorm(y, gamma, beta), beta.expand_as(y))
    assert torch.equal(emu_layernorm(y, gamma, beta, res), beta + res)


# defect -> the families whose rows must expose it.  Out of the bound's reach, by construction:
#   one_pass   for |mean| / std <= 10: E[y^2] - mean^2 loses about (mean / std)^2 n u of var, under the bound's n u;
#   no_eps / eps1e-6   where var >> eps: eps moves rstd by eps / (2 var) relative, under 2^-21 + n u once var >~ 1e-1
#              (std 1, mean/std rows, mag >= 2^4); eps1e-6 on constant rows: centred values are exactly 0 either way.
LN_DEFECTS = [
    ("one_pass", ["mean/std 1e2", "mean/std 1e3"]),
    ("no_eps", ["std 1e-2", "std 3e-3", "std 1e-3", "constant", "mag 2^-8", "mag 2^-4"]),
    ("eps1e-6", ["std 1e-2", "std 3e-3", "std 1e-3", "mag 2^-8", "mag 2^-4"]),
    ("res_first", list(LN_FAMILIES)),
]


@pytest.mark.parametrize("params", ["random", "identity"])
@pytest.mark.parametrize("defect,families", LN_DEFECTS)
def test_layernorm64_rejects_defects(defect, families, params):
    for family in families:
        seed = 300 + list(LN_FAMILIES).index(family)
        y, gamma, beta, res, ref, bnd = _ln_case(family, params, True, seed)
        rejects("layernorm %s %s" % (family, defect), emu_layernorm(y, gamma, beta, res, defect), ref, bnd)


# ---- fused FFN (§ c of the GPU tests) --------------------------------------------------------------------------------
def emu_ffn(x0, x1, w1, w2, res, gamma, beta, defect=None):
    """ffn_tc_kernel in fp32: H = X W1^T from the split products lo*hi + hi*lo + hi*hi, P = act_gelu(H) as fp16 (hi, lo),
    O = P W2^T the same way, then the LayerNorm epilogue.
    defects: "p_hi_only" the lo plane of P dropped; "tanh_gelu" the tanh-form GELU; "h_fp16" H rounded to fp16 before
    GELU."""
    xh, xl = hl(torch.cat((x0, x1), -1))
    w1h, w1l = hl(w1.flatten(1))
    w2h, w2l = hl(w2.flatten(1))
    h = xl @ w1h.T + xh @ w1l.T + xh @ w1h.T
    if defect == "h_fp16":
        h = h.half().float()
    p = gelu_tanh_form(h) if defect == "tanh_gelu" else gelu_fast(h)
    ph, pl = hl(p)
    if defect == "p_hi_only":
        pl = torch.zeros_like(pl)
    o = pl @ w2h.T + ph @ w2l.T + ph @ w2h.T
    return emu_layernorm(o, gamma.float(), beta.float(), res)


def _selecting(rows, cols, gen, signed):
    """[rows, cols, 1, 1] weight with one +-1 (signed) or +1 per row, in distinct columns where cols >= rows"""
    w = torch.zeros((rows, cols, 1, 1))
    col = torch.randperm(cols, generator=gen)[:rows] if cols >= rows else torch.randint(0, cols, (rows,), generator=gen)
    w[torch.arange(rows), col, 0, 0] = torch.where(torch.rand(rows, generator=gen) < 0.5, -1.0, 1.0) if signed else 1.0
    return w


def ffn_case(kind, rows, hidden, seed, residual=True):
    """Inputs of one FFN edge case.
      "mag 2^k"      standard-normal sources x 2^k, fan-in weights;
      "hidden +-60"  W1 selects one source channel per hidden channel (weight +-1), sources exact in fp16 and spread
                     over [-60, 60]: the hidden pre-activations reach GELU's tail and its clamp at 8.5; fan-in W2;
      "select"       W1 and W2 both select (one +-1 / +1 per row), standard-normal sources: every output is one hidden
                     channel's GELU, with no sum over the hidden dimension to average a defect's rounding away."""
    gen = g(seed)
    gamma, beta = torch.randn(C, generator=gen), torch.randn(C, generator=gen)
    res = torch.randn((rows, C), generator=gen) if residual else None
    if kind == "select":
        xs = [torch.randn((rows, C), generator=gen) for _ in range(2)]
        return xs, _selecting(hidden, 2 * C, gen, True), _selecting(C, hidden, gen, False), res, gamma, beta
    w2 = torch.randn((C, hidden, 1, 1), generator=gen) * (1.0 / hidden) ** 0.5
    if kind == "hidden +-60":
        xs = [(torch.rand((rows, C), generator=gen) * 120 - 60).half().float() for _ in range(2)]
        return xs, _selecting(hidden, 2 * C, gen, True), w2, res, gamma, beta
    scale = 2.0 ** float(kind.split("^")[1])
    xs = [torch.randn((rows, C), generator=gen) * scale for _ in range(2)]
    w1 = torch.randn((hidden, 2 * C, 1, 1), generator=gen) * (2.0 / (2 * C)) ** 0.5
    return xs, w1, w2, res, gamma, beta


FFN_KINDS = ["mag 2^-8", "mag 2^-4", "mag 2^0", "mag 2^4", "mag 2^8", "hidden +-60", "select"]


@pytest.mark.parametrize("hidden", [128, 1024])
@pytest.mark.parametrize("kind", FFN_KINDS)
def test_ffn64_passes_emulation(kind, hidden):
    xs, w1, w2, res, gamma, beta = ffn_case(kind, 256, hidden, 400 + FFN_KINDS.index(kind))
    ref, bnd = ref64.ffn64(xs[0], xs[1], w1, w2, res, gamma, beta)
    r = ref64.check("ffn %s hidden %d emulation" % (kind, hidden), emu_ffn(xs[0], xs[1], w1, w2, res, gamma, beta), ref,
                    bnd)
    assert r < 0.5                                     # headroom for the GPU's truncating accumulation


@pytest.mark.parametrize("hidden", [128, 1024])
@pytest.mark.parametrize("defect", ["p_hi_only", "tanh_gelu", "h_fp16"])
def test_ffn64_rejects_defects(defect, hidden):
    """Each defect is rejected on the "select" case (1.6x to 4.7x the bound with these inputs).

    Out of the bound's reach: all three defects with fan-in W2 (the "mag" and "hidden +-60" cases stay at 0.01 to 0.32 of
    the bound).  ffn64 adds the hidden channels' GELU and split bounds linearly through |W2| (eh @ |W2|^T: a worst case
    over signs), while a defect's rounding errors have random signs and add as sqrt(hidden), 11x to 32x less.  A
    tighter bound would have to assume random signs, which the truncating tensor-core accumulation does not give.  The
    activation sweep of the GPU tests sees a tanh-form act_gelu directly (test_act_bound_rejects_tanh_form_gelu)."""
    xs, w1, w2, res, gamma, beta = ffn_case("select", 256, hidden, 400 + FFN_KINDS.index("select"))
    ref, bnd = ref64.ffn64(xs[0], xs[1], w1, w2, res, gamma, beta)
    rejects("ffn select hidden %d %s" % (hidden, defect), emu_ffn(xs[0], xs[1], w1, w2, res, gamma, beta, defect), ref,
            bnd)
