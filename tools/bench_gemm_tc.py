#!/usr/bin/env python
"""Time every wgmma GEMM plan of the cfg3 MLPs on its own, in bf16x3 and in plain bf16 mode.

    python tools/bench_gemm_tc.py [--batch 8192] [--iters 200] [--warmup 20] [--tile-m 128,256] [--json OUT]

The plans are the ones a cfg3 `Engine(gemm="tc")` builds for one batch (`eng.tc_plans`: forward, dgrad and
weight-gradient plans of the bottom and top MLPs).  Only the dense dimensions decide a plan, so the engine is
built with small embedding tables.  Every plan is re-created from its own descriptor with `mode_x3=0`, and the
forward and dgrad plans also with `tile_m=128` and `tile_m=256` (where the library has the field).

Per plan: the median of `--iters` back-to-back launches, each bracketed by CUDA events on one stream, after
`--warmup` launches.  FLOP counts: 2 M N K per product (fp32-equivalent); x3 issues three bf16 MMAs per
product, so its bf16 MMA rate is 3x that over the time.  The share is of the data sheet's dense BF16 rate
(989 TFLOP/s for the H100 SXM at 700 W).  The x3/bf16 column is the time ratio at the same shape: about 3 when
the kernel is bound by the tensor cores (x3 issues 3x the MMAs), about 2 when it is bound by operand traffic
(x3 moves 2x the operand bytes).
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_BF16 = 989e12


def gpu_state():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "nvidia-smi unavailable (%s)" % e


def time_plan(plan, iters, warmup, stream):
    for _ in range(warmup):
        plan.run(stream.cuda_stream)
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    with torch.cuda.stream(stream):
        for a, b in ev:
            a.record(stream)
            plan.run(stream.cuda_stream)
            b.record(stream)
    stream.synchronize()
    return float(np.median([a.elapsed_time(b) for a, b in ev])) * 1e3   # us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8192)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--json", default=None, help="also write the rows as JSON here")
    ap.add_argument("--tile-m", default="128,256", help="tile heights the forward and dgrad plans are also timed at")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gemm_tc: no CUDA device")

    from dlrm_b200 import _lib
    from dlrm_b200 import mlperf as M
    from dlrm_b200.engine import Engine

    torch.cuda.set_device(0)
    dev = "cuda:0"
    B = args.batch
    tms = [int(t) for t in args.tile_m.split(",") if t]
    ln_emb = [1000] * len(M.TABLE_ROWS)
    ln_top = M.ln_top()
    eng = Engine(M.DIM, ln_emb, list(M.LN_BOT), ln_top, loss="bce", sigmoid_top=len(ln_top) - 2, device=dev,
                 max_batch=B, gemm="tc")
    eng.init_params(0)
    eng._tc_setup(B)
    torch.cuda.synchronize()
    has_tile_m = any(f == "tile_m" for f, _ in _lib.GemmTcDesc._fields_)
    fields = [f for f, _ in _lib.GemmTcDesc._fields_]

    def variant(plan, **over):
        kw = {f: getattr(plan.desc, f) for f in fields}
        kw.update(over)
        return _lib.GemmTcPlan(**kw)

    stream = torch.cuda.Stream()
    rows = []
    for kind in ("fwd", "dgrad", "wgrad"):
        for (which, i), plan in sorted(eng.tc_plans[kind].items()):
            d = plan.desc
            Mm, N, K = d.M, d.N, d.K
            flop = 2.0 * Mm * N * K
            r = dict(kind=kind, mlp=which, layer=i, M=Mm, N=N, K=K, info=plan.info())
            r["us_x3"] = time_plan(plan, args.iters, args.warmup, stream)
            r["us_bf16"] = time_plan(variant(plan, mode_x3=0), args.iters, args.warmup, stream)
            if has_tile_m and kind != "wgrad":
                for tm in tms:
                    try:
                        p = variant(plan, tile_m=tm)
                    except RuntimeError as e:
                        r["x3_tm%d" % tm] = str(e)
                        continue
                    r["us_x3_tm%d" % tm] = time_plan(p, args.iters, args.warmup, stream)
                    r["us_bf16_tm%d" % tm] = time_plan(variant(plan, tile_m=tm, mode_x3=0), args.iters, args.warmup,
                                                       stream)
            r["flop"] = flop
            rows.append(r)
    state = gpu_state()

    def share(us, mult, flop):
        tf = mult * flop / (us * 1e-6) / 1e12
        return tf, tf * 1e12 / PEAK_BF16

    print("# %s | batch %d | %d launches per point (median), %d warm-up" % (state, B, args.iters, args.warmup))
    print("# bf16 MMA TFLOP/s: x3 counts 3 MMAs per product; share = of 989 TFLOP/s (H100 SXM data sheet, dense BF16)")
    hdr = "%-6s %-4s %2s %5s %5s %5s %4s %3s %4s %9s %7s %5s %9s %7s %5s %6s" % (
        "kind", "mlp", "L", "M", "N", "K", "tn", "tm", "ctas", "x3 us", "TF/s", "share", "bf16 us", "TF/s", "share",
        "x3/bf")
    print(hdr)
    for r in rows:
        info = r["info"]
        tx, sx = share(r["us_x3"], 3, r["flop"])
        tb, sb = share(r["us_bf16"], 1, r["flop"])
        print("%-6s %-4s %2d %5d %5d %5d %4d %3s %4d %9.1f %7.1f %5.2f %9.1f %7.1f %5.2f %6.2f" % (
            r["kind"], r["mlp"], r["layer"], r["M"], r["N"], r["K"], info["tile_n"], info.get("tile_m", 128),
            info["ctas"], r["us_x3"], tx, sx, r["us_bf16"], tb, sb, r["us_x3"] / r["us_bf16"]))
        for tm in tms:
            if "us_x3_tm%d" % tm in r:
                tx, sx = share(r["us_x3_tm%d" % tm], 3, r["flop"])
                tb, sb = share(r["us_bf16_tm%d" % tm], 1, r["flop"])
                print("%-6s %-4s %2s %5s %5s %5s %4s %3d %4s %9.1f %7.1f %5.2f %9.1f %7.1f %5.2f %6.2f" % (
                    "", "", "", "", "", "", "", tm, "", r["us_x3_tm%d" % tm], tx, sx, r["us_bf16_tm%d" % tm], tb, sb,
                    r["us_x3_tm%d" % tm] / r["us_bf16_tm%d" % tm]))
            elif "x3_tm%d" % tm in r:
                print("%-6s tile_m=%d refused: %s" % ("", tm, r["x3_tm%d" % tm]))
    for kind in ("fwd", "dgrad", "wgrad"):
        ks = [r for r in rows if r["kind"] == kind]
        print("# %-5s total: x3 %.1f us, bf16 %.1f us" % (kind, sum(r["us_x3"] for r in ks), sum(r["us_bf16"] for r in ks)))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(gpu=state, batch=B, iters=args.iters, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
