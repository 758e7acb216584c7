#!/usr/bin/env python
"""Inference with row-wise quantized embedding tables on the MLPerf-DLRM model, one H100.

    python tools/bench_quantized_tables.py [--iters 50] [--repeats 2] [--batches 8192,16384] [--out FILE]

Configurations, each built, timed and freed in turn, alternated a, b, c, d, e, a, b, c, d, e:
  (a) the MLPerf tables (204.2 M rows, dim 128), fp16 rows           (55.5 GB)
  (b) the same tables, 8-bit rows                                   (27.8 GB)
  (c) the same tables, 4-bit rows                                   (13.9 GB)
  (d) the tables capped at 20 M rows, fp32 rows (the engine's [w | 4 words] rows)
  (e) the capped tables, 8-bit rows
One-hot lookups (uniform random rows), the MLPerf MLPs on the tensor-core path, forward only.  For every test batch
size: ms per batch and samples/s of a replayed forward graph, and the gather kernel alone -- its launches captured in a
CUDA graph of their own, so no host work is inside the timed span -- in us, with its bandwidth computed from each
format's bytes (rows read, indices and offsets read, pooled rows written) over the H100 SXM data sheet's 3.35 TB/s.
Also the quantize kernel's rate on 8 M fp32 rows, and the GPU name, power limit and SM clock read in the same run.  The tables are left zero: the kernels' memory traffic does not
depend on the values.  Loading and quantizing an fp32 checkpoint of the MLPerf size is not measured here (it needs a
108 GB checkpoint on disk).
"""
import argparse
import json
import os
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (ClockSampler)
from tools.bench_fp16_tables import gpu_info  # noqa: E402

HBM_PEAK = 3.35e12
CONFIGS = {"a": ("full", "fp16"), "b": ("full", "int8"), "c": ("full", "int4"), "d": ("cap20M", "fp32"),
           "e": ("cap20M", "int8")}


def row_read_bytes(dtype, D):
    return {"fp32": 4 * D, "fp16": 2 * D, "int8": D + 8, "int4": D // 2 + 4}[dtype]


def build(cap, dtype, max_batch):
    from dlrm_b200 import mlperf as M
    from dlrm_b200.engine import Engine

    rows = list(M.TABLE_ROWS) if cap == "full" else [min(n, 20_000_000) for n in M.TABLE_ROWS]
    e = Engine(M.DIM, rows, M.LN_BOT, M.ln_top(len(rows)), sigmoid_top=len(M.ln_top(len(rows))) - 2,
               device="cuda:0", max_batch=max_batch, gemm="tc", emb_dtype=dtype)
    return e, rows


def time_events(fn, iters):
    s, t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    s.record()
    for _ in range(iters):
        fn()
    t.record()
    torch.cuda.synchronize()
    return s.elapsed_time(t) / iters


def measure(name, batches, iters):
    from dlrm_b200.engine import GraphedTrainStep, sparse_from_reference

    cap, dtype = CONFIGS[name]
    e, rows = build(cap, dtype, max(batches))
    tbytes = (e.qtables if e.quant_only else e.tables).numel() * (1 if e.quant_only else e.esize)
    g = torch.Generator(device="cuda:0").manual_seed(1)
    res = []
    for B in batches:
        X = torch.rand((B, 13), device="cuda:0", generator=g)
        idx = [torch.randint(0, n, (B,), device="cuda:0", generator=g) for n in rows]
        off = torch.arange(B, device="cuda:0").repeat(len(rows), 1)
        sp = sparse_from_reference(off, idx, "cuda:0")
        e.emb_forward(sp)                        # warm-up outside the capture
        torch.cuda.synchronize()
        gather_graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gather_graph):
            e.emb_forward(sp)
        gather_ms = time_events(gather_graph.replay, iters)
        del gather_graph
        stage = types.SimpleNamespace(X=X, sparse=sp, target=None)
        graph = GraphedTrainStep(e, stage, 0.0, "sgd", warmup=2, train=False)
        step_ms = time_events(graph.replay, iters)
        nbytes = B * len(rows) * (row_read_bytes(dtype, e.D) + 2 * 8 + 4 * e.D)
        res.append(dict(config=name, tables=cap, dtype=dtype, table_gb=round(tbytes / 1e9, 2), batch=B,
                        ms_per_batch=round(step_ms, 4), samples_per_s=round(B / step_ms * 1e3),
                        gather_us=round(gather_ms * 1e3, 1), gather_gb_s=round(nbytes / (gather_ms * 1e-3) / 1e9, 1),
                        gather_share_of_hbm_peak=round(nbytes / (gather_ms * 1e-3) / HBM_PEAK, 3)))
        del graph
    assert e.lib.dlrm_b200_check_device_errors(None) == 0
    del e
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return res


def quantize_rate(iters):
    from dlrm_b200 import _lib

    n, D = 8_000_000, 128
    src = torch.rand((n, D), device="cuda:0")
    out = {}
    for bits, qd in ((8, _lib.DTYPE_Q8), (4, _lib.DTYPE_Q4)):
        dst = torch.empty((n, D + 8 if bits == 8 else D // 2 + 4), dtype=torch.uint8, device="cuda:0")

        def run():
            _lib.check(_lib.lib().dlrm_b200_emb_quantize_rows(src.data_ptr(), _lib.DTYPE_F32, D, n, D, dst.data_ptr(),
                                                              qd, 0, torch.cuda.current_stream().cuda_stream), "q")
        ms = time_events(run, iters)
        out["quantize_int%d" % bits] = dict(rows=n, ms=round(ms, 3), rows_per_s=round(n / ms * 1e3),
                                            gb_s=round(n * (4 * D + dst.shape[1]) / (ms * 1e-3) / 1e9, 1))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--batches", default="8192,16384")
    ap.add_argument("--configs", default="abcde")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    batches = [int(b) for b in a.batches.split(",")]
    info = gpu_info()
    clocks = bench.ClockSampler()
    clocks.start()
    t0 = time.time()
    lines = []
    try:
        for r in range(a.repeats):
            for name in a.configs:
                for row in measure(name, batches, a.iters):
                    row["repeat"] = r
                    lines.append(row)
                    print(json.dumps(row), flush=True)
        q = quantize_rate(a.iters)
        print(json.dumps(q), flush=True)
    finally:
        clk = clocks.stop(t0, time.time())
    summary = dict(info, clocks=clk, quantize=q,
                   checkpoint_load="not measured (needs a 108 GB fp32 checkpoint on disk)")
    print(json.dumps(summary), flush=True)
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(dict(summary, rows=lines), fh, indent=1)


if __name__ == "__main__":
    main()
