#!/usr/bin/env python
"""fp32 vs fp16 embedding tables on the MLPerf-DLRM workload (cfg3), one H100.

    python tools/bench_fp16_tables.py [--steps K] [--warmup W] [--repeats 2] [--runs a,b,c]

Runs, each in its own process (the tables of one run must be freed before the next), alternating
  (a) cfg3 with bench.py's 20 M-row cap, fp32 tables     (53.3 GB of weights)
  (b) cfg3 with the cap, fp16 tables                     (28.3 GB with the per-row words)
  (c) cfg3 uncapped (204.2 M rows), fp16 tables          (55.5 GB; fp32 would need 104.5 GB)
as a,b,a,b,...,c, and prints one JSON line per run: ms/step, samples/s, the training gather+link and update times
(CUDA events around those launches, as bench.py's kernel section measures them), table bytes, and the GPU name,
power limit and median SM clock read during the run.

Every run drives the sharded engine at N = 1 the way bench.py does (placement, peer-mapped exchange, multi-hot
index exchange, device-resident ring of batches, RWSAdagrad, lr 0.01), with eager steps: a captured training step
would replay one step's stochastic-rounding bits, so fp16 tables train eagerly and the fp32 run does the same.
"""
import argparse
import json
import os
import subprocess
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload, lookups_per_sample, ClockSampler, measure_rooflines)

RUNS = {"a": ("capped", "fp32"), "b": ("capped", "fp16"), "c": ("uncapped", "fp16")}


def gpu_info(index=0):
    """Name and power limit of the GPU (nvidia-smi, read only)."""
    info = {"gpu": torch.cuda.get_device_name(index), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        info["power_limit_w"] = float(out.splitlines()[0])
    except Exception:
        pass
    return info


def one_run(name, steps, warmup, ring):
    from dlrm_b200 import dist as ddist, mlperf as M, placement as P

    cap, dtype = RUNS[name]
    os.environ.update(RANK="0", WORLD_SIZE="1", LOCAL_RANK="0", MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(bench._free_port()))
    os.environ.setdefault("NCCL_NVLS_ENABLE", "0")
    ddist.init_distributed("nccl")
    torch.cuda.set_device(0)
    dev = "cuda:0"
    W = bench.workload("cfg3")
    if cap == "uncapped":
        W["rows"] = list(M.TABLE_ROWS)
    D, rows, ln_bot, ln_top = bench.model_dims(W)
    B = W["B"]
    cost = bench.lookups_per_sample(W)
    pl = P.plan(rows, cost, 1, bytes_per_row=P.row_bytes(D, dtype))
    de = ddist.DistEngine(D, rows, ln_bot, ln_top, local_batch=B, device=dev, gemm="tc", exchange="p2p",
                          placement=pl, emb_dtype=dtype)
    eng = de.eng
    eng.init_params(100)
    eng.ensure_optimizer_state("rwsadagrad")
    lr, nsets = 0.01, 2
    mh = ddist.MultiHotExchange(de, W["hot"], 13, nsets)
    host = [mh.fill_host(mh.host_buffer(), 1234, i, rows) for i in range(ring)]
    devr = [h.to(dev) for h in host]
    stages = [types.SimpleNamespace(sparse=mh.sparse[k], X=mh.X[k], target=mh.target[k]) for k in range(nsets)]

    def pre(k):
        return lambda: mh.exchange(k)

    def load_dev(k, i):
        mh.stage[k].copy_(devr[i % ring], non_blocking=True)

    def step(i):
        k = i % nsets
        load_dev(k, i)
        mh.exchange(k)
        return eng.train_step(stages[k].X, stages[k].sparse, stages[k].target, lr, "rwsadagrad")

    for i in range(warmup):
        step(i)
    torch.cuda.synchronize()
    sampler = bench.ClockSampler(0)
    sampler.start()
    time.sleep(0.25)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.time()
    ev0.record()
    for r in range(steps):
        loss = step(warmup + r)
    ev1.record()
    torch.cuda.synchronize()
    t1 = time.time()
    ms = ev0.elapsed_time(ev1) / steps
    clocks = sampler.stop(t0, t1)
    args = types.SimpleNamespace(steps=steps)
    # only the two times are taken: bench.py's byte model behind its GB/s figures counts 4-byte elements
    _, roof_upd = bench.measure_rooflines(de, stages, load_dev, pre, args, W, cost, 3350.0, "data sheet", True)
    line = {"run": name, "tables": "cfg3 %s (%.1f M rows x %d)" % (cap, sum(rows) / 1e6, D), "emb_dtype": dtype,
            "ms_per_step": ms, "samples_per_s": B / (ms * 1e-3), "steps": steps, "warmup": warmup,
            "gather_link_us": roof_upd["train_gather_plus_link_us"], "update_us": roof_upd["avg_launch_us"],
            "table_bytes": int(eng.tables.numel() * eng.tables.element_size()),
            "loss_last_step": float(loss.item()), "sm_clock_mhz": clocks.get("sm_mhz"),
            "clock_reasons": clocks.get("reasons"), "cuda_graph": False}
    line.update(gpu_info(0))
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--ring", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=2, help="how many times (a) and (b) alternate")
    ap.add_argument("--runs", default="a,b,c", help="which of a, b, c to run")
    ap.add_argument("--one", default=None, help=argparse.SUPPRESS)     # internal: run one configuration here
    args = ap.parse_args()
    if args.one:
        return one_run(args.one, args.steps, max(args.warmup, 3), args.ring)
    want = [r for r in args.runs.split(",") if r]
    order = [r for _ in range(args.repeats) for r in ("a", "b") if r in want] + (["c"] if "c" in want else [])
    failed = 0
    for name in order:
        cmd = [sys.executable, os.path.abspath(__file__), "--one", name, "--steps", str(args.steps),
               "--warmup", str(args.warmup), "--ring", str(args.ring)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
        if r.returncode != 0 or not lines:
            failed += 1
            print(json.dumps({"run": name, "error": (r.stderr or r.stdout)[-1500:]}), flush=True)
        else:
            print(lines[-1], flush=True)
    sys.exit(1 if failed else 0)


if __name__ == "__main__":
    main()
