"""The GEMM epilogue functions on the device, each against float64 (tests/ref64.py) over its whole input range:
  a. GELU, tanh and sigmoid through um_conv2d_tc's epilogue, with the argument set exactly: a 1x1 Linear over zero input
     planes with no bias, the sweep values passed as the pre-accumulated input, so the epilogue sees exactly y;
  b. the LayerNorm epilogues (conv UM_CONV_LN at G = 1 and G = 2, and the fused FFN's) on row families with large means,
     variance near eps, constant rows and outlier channels, the GEMM output set exactly by identity / selecting weights;
  c. the fused FFN at its edges against ffn64;
  d. a census of the FFN launches of the bench workloads, each of which must have a case here or in
     tests/test_kernel_edges_gpu.py.
The cases and the fp32 emulations that show the bounds reject defective epilogues are in tests/test_epilogue_edges_cpu.py."""
import math

import pytest
import torch

import ref64
import test_epilogue_edges_cpu as E
import test_kernel_edges_gpu as K
from unimatch_b200 import ops

pytestmark = pytest.mark.gpu
OPS = torch.ops.unimatch_sm100
C = 128
FP16_MAX = 65504.0
L_, LN = ops.CONV_LINEAR, ops.CONV_LN
ACTS = {"tanh": ops.ACT_TANH, "sigmoid": ops.ACT_SIGMOID, "gelu": ops.ACT_GELU}


# ---- a. activation sweeps ---------------------------------------------------------------------------------------------
def run_act(y, act, bn):
    """y [N] fp32 through a 1x1 Linear (cout = bn, 64 zero input channels, no bias) with pre = y: the accumulator is 0,
    so the epilogue's argument is 0 + y = y exactly.  Returns (fp32 output, fp16 (hi + lo) split output) [N]."""
    n = y.numel()
    pix = ((n + bn - 1) // bn + 15) // 16 * 16
    h = pix // 16
    pre = torch.zeros(pix * bn)
    pre[:n] = y
    dev = "cuda"
    src = torch.zeros((2, 1, h, 16, 64), dtype=torch.float16, device=dev)
    wt = ops.prep_conv_weight(torch.zeros((bn, 64, 1, 1)), [64], bn).to(dev)
    out_f = torch.zeros((1, h, 16, bn), device=dev)
    out_s = torch.zeros((2, 1, h, 16, bn), dtype=torch.float16, device=dev)
    OPS.conv2d_tc(src, None, wt, None, 1, 1, 0, 0, bn, bn, L_, act, out_f, 0, out_s, 0, None, None, None, None, 1, 0, None,
                  None, 0, 0, 0, pre.view(1, h, 16, bn).to(dev))
    return out_f.view(-1)[:n].cpu(), (out_s[0].double() + out_s[1].double()).view(-1)[:n].cpu()


# name, act, bn: bn 128 / GELU is the fixed (128, 1, LINEAR, GELU) instantiation; the others run the run-time-mode one
ACT_CASES = [("gelu", 128), ("gelu", 64), ("tanh", 128), ("sigmoid", 128)]


@pytest.mark.parametrize("name,bn", ACT_CASES)
def test_activation_sweep(name, bn):
    """Every sweep value of test_epilogue_edges_cpu.act_sweep against ref64.act_bound(y, 0).  The split output is checked
    where the fp32 output and the exact result fit fp16 (<= 65504 in magnitude).
    Non-finite arguments: NaN must give NaN.  The header promises nothing for +-inf; what they give is printed
    (act_gelu(+inf) = fmaf(-inf, 2^q(8.5), +inf) = NaN, act_gelu(-inf) = -inf; tanh_fast(+-inf) = +-1 and
    sigmoid_fast(+inf) = 1, sigmoid_fast(-inf) = 0 through __expf(+-inf) = inf / 0)."""
    y = E.act_sweep()
    got_f, got_s = run_act(y, ACTS[name], bn)
    y64 = y.double()
    ref, bnd = ref64.act_bound(y64, torch.zeros_like(y64), name)
    tag = "%s bn %d (%s)" % (name, bn, "fixed" if (name, bn) == ("gelu", 128) else "run-time mode")
    ref64.check(tag + " f32", got_f, ref, bnd)
    # the split planes hold the fp32 output: where that exceeds fp16's range (including act_gelu(y) = -|y| 2^q(8.5), not
    # ~0, for y << -8.5: -9.5e12 at y = -1e30, inside the bound's U32 |y| term) hi is inf by the format
    fits = (ref.abs() <= FP16_MAX) & (got_f.double().abs() <= FP16_MAX)
    ref64.check(tag + " split", got_s[fits], ref[fits], ref64.split_out_bound(ref[fits], bnd[fits]))
    err = (got_f.double() - ref).abs()
    inr = y.abs() <= 12
    i = int(torch.where(inr, err, torch.zeros_like(err)).argmax())
    j = int((err / y64.abs().clamp(min=1.0)).argmax())
    print("%s: worst |err| %.3g at y = %.9g (|y| <= 12); worst |err| / max(|y|, 1) %.3g at y = %.9g" % (
        tag, err[i].item(), y[i].item(), err[j].item() / max(abs(y[j].item()), 1.0), y[j].item()))
    nf_f, nf_s = run_act(torch.tensor([math.nan, -math.nan, math.inf, -math.inf]), ACTS[name], bn)
    assert torch.isnan(nf_f[:2]).all() and torch.isnan(nf_s[:2]).all(), (tag, nf_f, nf_s)
    print("%s: (+inf, -inf) -> %s" % (tag, nf_f[2:].tolist()))


# ---- b. LayerNorm rows ------------------------------------------------------------------------------------------------
ROWS_PER_FAMILY = 64


def family_rows(positive=False):
    """[families x 64, 128] fp32 rows, exact in fp16, and the row range of each family"""
    rows, spans = [], {}
    for i, fam in enumerate(E.LN_FAMILIES):
        spans[fam] = slice(i * ROWS_PER_FAMILY, (i + 1) * ROWS_PER_FAMILY)
        rows.append(E.ln_rows(fam, ROWS_PER_FAMILY, 500 + i, positive))
    return torch.cat(rows), spans


def _planes(x, cp):
    buf = torch.zeros((2, x.shape[0], cp), dtype=torch.float16, device="cuda")
    OPS.split_planes(x.cuda(), buf, 0)
    return buf


def _check_rows(tag, spans, got_f, got_s, ref, bnd):
    for fam, sl in spans.items():
        if got_f is not None:
            ref64.check("%s %s f32" % (tag, fam), got_f[sl], ref[sl], bnd[sl])
        if got_s is not None:
            ref64.check("%s %s split" % (tag, fam), got_s[sl], ref[sl], ref64.split_out_bound(ref[sl], bnd[sl]))


LN_VARIANTS = [("random", True), ("random", False), ("identity", True), ("identity", False)]


@pytest.mark.parametrize("params,with_res", LN_VARIANTS)
@pytest.mark.parametrize("cin", [128, 512])
def test_conv_layernorm_rows(cin, params, with_res):
    """UM_CONV_LN over token rows with an identity weight (cin 128: G = 1; cin 512, the extra channels zero: G = 2,
    per-stage accumulators): every row reaches the epilogue exactly, so layernorm64 runs with e = 0.  Constant rows must
    come out as beta (+ residual) bit for bit."""
    y, spans = family_rows()
    R = y.shape[0]
    gamma, beta = E.ln_params(params, 600)
    res = torch.randn((R, C), generator=E.g(601)) if with_res else None
    x = torch.zeros((R, cin))
    x[:, :C] = y
    wt = torch.zeros((C, cin, 1, 1))
    wt[torch.arange(C), torch.arange(C), 0, 0] = 1.0
    out_f = torch.zeros((R, C), device="cuda")
    out_s = torch.zeros((2, R, C), dtype=torch.float16, device="cuda")
    OPS.conv2d_tc(_planes(x, cin), None, ops.prep_conv_weight(wt, [cin], C).cuda(), None, 1, 1, 0, 0, C, C, LN, 0, out_f, 0,
                  out_s, 0, None if res is None else res.cuda(), None, gamma.cuda(), beta.cuda(), 1, R)
    ref, bnd = ref64.layernorm64(y.double(), torch.zeros((R, C), dtype=torch.float64), gamma, beta, res)
    got_f = out_f.cpu()
    _check_rows("conv LN G=%d %s res %s" % (1 if cin < 512 else 2, params, with_res), spans, got_f,
                (out_s[0].double() + out_s[1].double()).cpu(), ref, bnd)
    const = got_f[spans["constant"]]
    want = beta.expand_as(const) if res is None else beta + res[spans["constant"]]
    assert torch.equal(const, want), (const - want).abs().max()


def run_ffn(xs, w1, w2, res, gamma, beta, outputs=("f32", "split")):
    rows, hidden = xs[0].shape[0], w1.shape[0]
    out_f = torch.zeros((rows, C), device="cuda") if "f32" in outputs else None
    out_s = torch.zeros((2, rows, C), dtype=torch.float16, device="cuda") if "split" in outputs else None
    OPS.ffn_tc(_planes(xs[0], C), _planes(xs[1], C), ops.prep_conv_weight(w1, [C, C], hidden).cuda(),
               ops.prep_conv_weight(w2, [hidden], C).cuda(), None if res is None else res.cuda(), gamma.cuda(), beta.cuda(),
               out_f, out_s, rows)
    return (None if out_f is None else out_f.cpu(),
            None if out_s is None else (out_s[0].double() + out_s[1].double()).cpu())


@pytest.mark.parametrize("params,with_res", LN_VARIANTS)
def test_ffn_layernorm_rows(params, with_res):
    """The FFN's LayerNorm on the same families (mean offsets positive, where GELU is the identity for large arguments):
    hidden 128, W1 = [I | 0] and W2 = I, so O = the (hi, lo) split of GELU(row), checked against ffn64.  The last 64
    rows are zero, like the padding rows of the transformer's token buffers: beta (+ residual) bit for bit."""
    y, spans = family_rows(positive=True)
    R = y.shape[0] + 64
    x0 = torch.cat((y, torch.zeros((64, C))))
    x1 = torch.zeros((R, C))
    gamma, beta = E.ln_params(params, 610)
    res = torch.randn((R, C), generator=E.g(611)) if with_res else None
    w1 = torch.zeros((C, 2 * C, 1, 1))
    w1[torch.arange(C), torch.arange(C), 0, 0] = 1.0
    w2 = torch.zeros((C, C, 1, 1))
    w2[torch.arange(C), torch.arange(C), 0, 0] = 1.0
    got_f, got_s = run_ffn((x0, x1), w1, w2, res, gamma, beta)
    ref, bnd = ref64.ffn64(x0, x1, w1, w2, res, gamma, beta)
    spans["zero rows"] = slice(R - 64, R)
    _check_rows("ffn LN %s res %s" % (params, with_res), spans, got_f, got_s, ref, bnd)
    zero = got_f[spans["zero rows"]]
    want = beta.expand_as(zero) if res is None else beta + res[spans["zero rows"]]
    assert torch.equal(zero, want), (zero - want).abs().max()


# ---- c. the fused FFN at its edges -------------------------------------------------------------------------------------
FFN_EDGE = [
    # kind (test_epilogue_edges_cpu.ffn_case), hidden, rows, outputs / residual
    ("mag 2^-8", 128, 256, "res"),
    ("mag 2^-8", 1024, 256, "no_res"),
    ("mag 2^-4", 128, 256, "f32_only"),
    ("mag 2^-4", 1024, 256, "split_only"),
    ("mag 2^4", 128, 256, "no_res"),
    ("mag 2^4", 1024, 256, "res"),
    ("mag 2^8", 128, 256, "split_only"),
    ("mag 2^8", 1024, 256, "f32_only"),
    ("hidden +-60", 128, 256, "res"),
    ("hidden +-60", 1024, 256, "no_res"),
    ("select", 128, 256, "f32_only"),
    ("select", 1024, 256, "res"),
    ("hidden +-60", 1024, 256 * 77, "split_only"),
    ("select", 1024, 256 * 77, "no_res"),
    ("mag 2^8", 128, 256 * 77, "res"),
]


@pytest.mark.parametrize("kind,hidden,rows,variant", FFN_EDGE)
def test_ffn_edges(kind, hidden, rows, variant):
    xs, w1, w2, res, gamma, beta = E.ffn_case(kind, rows, hidden, 700 + E.FFN_KINDS.index(kind) + hidden,
                                              residual=variant != "no_res")
    outputs = {"f32_only": ("f32",), "split_only": ("split",)}.get(variant, ("f32", "split"))
    got_f, got_s = run_ffn(xs, w1, w2, res, gamma, beta, outputs)
    sel = torch.arange(rows) if rows <= 1024 else torch.cat((torch.arange(256), torch.arange(rows - 256, rows),
                                                             torch.randperm(rows, generator=E.g(rows))[:512])).unique()
    ref, bnd = ref64.ffn64(xs[0][sel], xs[1][sel], w1, w2, None if res is None else res[sel], gamma, beta)
    tag = "ffn %s hidden %d rows %d %s" % (kind, hidden, rows, variant)
    if got_f is not None:
        ref64.check(tag + " f32", got_f[sel], ref, bnd)
    if got_s is not None:
        ref64.check(tag + " split", got_s[sel], ref, ref64.split_out_bound(ref, bnd))


# ---- d. census of the FFN launches -------------------------------------------------------------------------------------
def ffn_key(hidden, rows):
    return ("ffn", hidden, rows % 256 == 0)


def covered_ffn_keys():
    keys = {ffn_key(hidden, rows) for _, hidden, rows, _ in FFN_EDGE}
    return keys | {ffn_key(hidden, rows) for rows, hidden in K.FFN_F64}       # test_kernel_edges_gpu.test_ffn_tc_vs_float64


class _FfnCensus(K._Census):
    """The conv / attention census of tests/test_kernel_edges_gpu.py, plus the transformer FFN of every launch: the fused
    kernel (ffn_tc) or the two GEMMs (W1 + GELU over two sources, then W2 + LayerNorm) when the rows are not a multiple of
    256."""

    def __init__(self, real):
        super().__init__(real)
        self.ffn = []

    def _key_ffn_tc(self, src0, src1, w1, w2, residual, gamma, beta, out_f32, out_split, rows):
        self.ffn.append(("fused kernel", w1.shape[1], rows))
        return ffn_key(w1.shape[1], rows)

    def _key_conv2d_tc(self, *a, **kw):
        b = self.conv_sig.bind(*a, **kw)
        b.apply_defaults()
        p = b.arguments
        if p["src1"] is not None and p["rows"] and p["act"] == ops.ACT_GELU:
            self.ffn.append(("two GEMMs", p["cout"], p["rows"]))
        return super()._key_conv2d_tc(*a, **kw)


def census_batches():
    """workload -> batch sizes of the census: 1, and the pairs per GPU bench.py runs it at"""
    from bench import BENCH_WORKLOADS
    from unimatch_b200.spec import WORKLOADS
    batches = {wl: {1} for wl in WORKLOADS}
    for wl, H, W, ppg, *_ in BENCH_WORKLOADS.values():
        batches[wl].add(ppg)
    return batches


def test_ffn_census_of_bench_workloads(monkeypatch):
    """Every workload of spec.WORKLOADS at its bench resolution, at batch 1 and at bench.py's batch: each fused-FFN
    launch (hidden, rows % 256 == 0) must have a case in FFN_EDGE or test_ffn_tc_vs_float64.  Prints which path each
    workload's FFN takes: the fused kernel needs token rows (2 x batch x tokens per view) that are a multiple of 256."""
    import unimatch_b200.unimatch as um
    from unimatch_b200.spec import WORKLOADS
    from unimatch_b200.synthetic import synthetic_batch, synthetic_model
    census = _FfnCensus(um._OPS)
    monkeypatch.setattr(um, "_OPS", census)
    for wl, batches in census_batches().items():
        cfg = WORKLOADS[wl]
        H, W = K.CENSUS_RES[cfg["model"]["task"]]
        model = synthetic_model(wl)
        for B in sorted(batches):
            inp = {k: v.cuda() for k, v in synthetic_batch(cfg["model"]["task"], B, H, W).items()}
            census.ffn = []
            with torch.no_grad():
                model(inp["img0"], inp["img1"], intrinsics=inp.get("intrinsics"), pose=inp.get("pose"), **cfg["call"])
            torch.cuda.synchronize()
            paths = sorted(set(census.ffn))
            assert paths, "%s: no FFN launch recorded" % wl
            print("ffn census: %s batch %d at %dx%d: %s" % (wl, B, H, W, "; ".join(
                "%s, hidden %d, rows %d" % p for p in paths)))
        del model
        torch.cuda.empty_cache()
    fused = {k for k in census.keys if k[0] == "ffn"}
    missing = fused - covered_ffn_keys()
    assert not missing, "fused FFN launches without an edge case: %s" % sorted(missing)
