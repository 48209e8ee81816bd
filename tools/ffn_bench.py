#!/usr/bin/env python
"""The fused transformer FFN kernel (`ops.ffn_tc`, um_ffn_tc.cu) on its own, on one GPU.

    python tools/ffn_bench.py [--rows 399360,99840] [--hidden 1024] [--iters 200] [--warmup 20] [--rounds 3]
                              [--baseline path/to/libunimatch_sm100.so ...]

The default row counts are the flagship workload's FFN calls (8 pairs of 480x832: 399,360 token rows at 1/4 resolution,
99,840 at 1/8), each made 6 times per step.  Operands are synthetic and seeded: [source | message] as fp16 (hi, lo) planes,
W1 [hidden, 256] and W2 [128, hidden] as prepared weight planes, an fp32 residual, and both outputs (fp32 rows and fp16
planes) written as the transformer does.  Each timing is CUDA events around `--iters` back-to-back launches after
`--warmup` launches of the same shape.

Each --baseline (repeatable; reported as base0, base1, ...) is another build of the library, for instance the parent
commit's, loaded next to the in-tree one and called through its C entry point `um_ffn_tc` with the same descriptor; all
builds alternate `--rounds` times per row count, in reversed order every other round, and each baseline's output is
compared with the in-tree build's (largest absolute difference over the largest value).

Prints the card, its power limit and SM clocks (query-only nvidia-smi), one line per timing (ms per launch, useful
TFLOP/s = 2 x rows x hidden x (256 + 128) per launch, MMA TFLOP/s = 3 x that for the three fp16 products of the hi/lo
split, and that as a share of the 989 TFLOP/s dense FP16 data-sheet figure of the H100 SXM), then ONE JSON line.
Fails without a CUDA device.  Writes nothing.
"""
import argparse
import ctypes
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.common import card  # noqa: E402
from unimatch_b200 import ops  # noqa: E402

PEAK_FP16_TFLOPS = 989.0


def operands(rows, hidden, dev, seed):
    gen = torch.Generator().manual_seed(seed)
    w1 = torch.randn((hidden, 256, 1, 1), generator=gen) * (2.0 / 256) ** 0.5
    w2 = torch.randn((128, hidden, 1, 1), generator=gen) * (1.0 / hidden) ** 0.5
    srcs = []
    for _ in range(2):
        buf = torch.zeros((2, rows, 128), dtype=torch.float16, device=dev)
        torch.ops.unimatch_sm100.split_planes(torch.randn((rows, 128), generator=gen).to(dev), buf, 0)
        srcs.append(buf)
    return {"src0": srcs[0], "src1": srcs[1],
            "w1": ops.prep_conv_weight(w1, [128, 128], hidden).to(dev), "w2": ops.prep_conv_weight(w2, [hidden], 128).to(dev),
            "residual": torch.randn((rows, 128), generator=gen).to(dev),
            "gamma": torch.randn(128, generator=gen).to(dev), "beta": torch.randn(128, generator=gen).to(dev),
            "out_f32": torch.empty((rows, 128), device=dev), "out_split": torch.empty((2, rows, 128), dtype=torch.float16, device=dev),
            "rows": rows}


def tree_launcher(t):
    op = torch.ops.unimatch_sm100.ffn_tc
    return lambda: op(t["src0"], t["src1"], t["w1"], t["w2"], t["residual"], t["gamma"], t["beta"], t["out_f32"],
                      t["out_split"], t["rows"])


def lib_launcher(lib, t):
    """The same call through another build's C entry point (the descriptor ops.ffn_tc fills)."""
    d = ops.FfnDesc()
    d.src[0] = t["src0"].data_ptr(); d.src[1] = t["src1"].data_ptr(); d.src_plane_stride = t["src0"].stride(0)
    d.rows = t["rows"]; d.w1 = t["w1"].data_ptr(); d.w2 = t["w2"].data_ptr(); d.hidden = t["w1"].shape[1]
    d.residual = t["residual"].data_ptr(); d.ld_res = t["residual"].stride(0)
    d.gamma = t["gamma"].data_ptr(); d.beta = t["beta"].data_ptr()
    d.out_f32 = t["out_f32"].data_ptr(); d.ld_f32 = t["out_f32"].stride(0)
    d.out_split = t["out_split"].data_ptr(); d.split_plane_stride = t["out_split"].stride(0)

    def run():
        rc = lib.um_ffn_tc(ctypes.byref(d), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        if rc:
            raise RuntimeError("baseline um_ffn_tc failed (%d)" % rc)
    return run


def time_ms(launch, iters, warmup):
    """mean device time of one launch, from CUDA events around `iters` back-to-back launches (common.timed is host time)"""
    for _ in range(warmup):
        launch()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        launch()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", default="399360,99840", help="comma-separated row counts (multiples of 256)")
    ap.add_argument("--hidden", type=int, default=1024)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--baseline", action="append", default=[],
                    help="another libunimatch_sm100.so to alternate with the in-tree build (repeatable)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("ffn_bench needs a CUDA device")
    if args.iters < 1 or args.rounds < 1:
        ap.error("--iters and --rounds must be positive")
    dev = torch.device("cuda", 0)
    bases = []
    for i, path in enumerate(args.baseline):
        lib = ctypes.CDLL(os.path.abspath(path))
        lib.um_ffn_tc.restype = ctypes.c_int
        lib.um_ffn_tc.argtypes = [ctypes.POINTER(ops.FfnDesc), ctypes.c_void_p]
        bases.append(("base%d" % i, path, lib))
    gpu = ", ".join(card().values())
    print("card: %s" % gpu, flush=True)
    result = {"card": gpu, "hidden": args.hidden, "iters": args.iters, "rounds": args.rounds,
              "baselines": {k: path for k, path, _ in bases}, "shapes": []}
    for rows in [int(r) for r in args.rows.split(",")]:
        t = operands(rows, args.hidden, dev, seed=1234 + rows % 1000)
        runs = {"tree": tree_launcher(t)}
        for k, _, lib in bases:
            runs[k] = lib_launcher(lib, t)
        ms = {k: [] for k in runs}
        useful = 2.0 * rows * args.hidden * (256 + 128)
        for r in range(args.rounds):
            order = list(runs) if r % 2 == 0 else list(reversed(runs))
            for k in order:
                m = time_ms(runs[k], args.iters, args.warmup)
                ms[k].append(m)
                tf = useful / m * 1e-9
                print("rows %7d  %-5s round %d: %.4f ms/launch  useful %.1f TFLOP/s  MMA %.1f TFLOP/s  (%.1f %% of %.0f)"
                      % (rows, k, r, m, tf, 3 * tf, 100 * 3 * tf / PEAK_FP16_TFLOPS, PEAK_FP16_TFLOPS), flush=True)
        entry = {"rows": rows, "useful_tflop": useful * 1e-12}
        for k, v in ms.items():
            mean = sum(v) / len(v)
            entry[k] = {"ms": [round(x, 5) for x in v], "ms_mean": round(mean, 5), "spread_ms": round(max(v) - min(v), 5),
                        "mma_tflops": round(3 * useful / mean * 1e-9, 1),
                        "share_of_peak": round(3 * useful / mean * 1e-9 / PEAK_FP16_TFLOPS, 4)}
        for k, _, _ in bases:
            outs = []
            for run in (runs["tree"], runs[k]):
                t["out_f32"].zero_(); t["out_split"].zero_()
                run()
                outs.append((t["out_f32"].clone(), t["out_split"].float().sum(0)))
            scale = outs[1][0].abs().max().item()
            entry[k]["speedup_of_tree"] = round(entry[k]["ms_mean"] / entry["tree"]["ms_mean"], 4)
            entry[k]["max_abs_diff_rel"] = {"f32": (outs[0][0] - outs[1][0]).abs().max().item() / scale,
                                            "split": (outs[0][1] - outs[1][1]).abs().max().item() / scale}
        result["shapes"].append(entry)
        del t
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
