#!/usr/bin/env python
"""Element-wise Adagrad against row-wise Adagrad on one H100.

    python tools/bench_adagrad.py [--steps K] [--warmup W] [--repeats 2] [--runs a,b,c,d]

Runs, each in its own process (the tables of one run are freed before the next), alternated a,b,c,a,b,c then d:
  (a) cfg2 (26 x 1e6 x 128, batch 2048, random bags Lmax 10), fp32 tables, RWSAdagrad
  (b) cfg2, fp32 tables, Adagrad (one fp32 accumulator per element: a separate [rows, 128] arena)
  (c) cfg2, fp16 tables, Adagrad
  (d) cfg3-shaped (MLPerf multi-hot, batch 8192) with the row cap lowered until the fp32 tables plus the Adagrad
      accumulators fit, fp32 tables, Adagrad
and prints one JSON line per run: ms/step, samples/s, the median time of the embedding update alone (CUDA events around
the update launches, cfg2 runs), the row cap and the GB of tables and accumulators, and the GPU's name and power
limit.  Eager steps throughout (fp16 tables train eagerly; the fp32 runs do the same).
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

import bench  # noqa: E402  (workload, model_dims, lookups_per_sample)

RUNS = {"a": ("cfg2", "fp32", "rwsadagrad"), "b": ("cfg2", "fp32", "adagrad"), "c": ("cfg2", "fp16", "adagrad"),
        "d": ("cfg3", "fp32", "adagrad")}
FIT_BYTES = 70e9      # tables + accumulators of run (d), leaving room for activations, batches and the CUDA context


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


def _arena_gb(eng):
    t = eng.tables.numel() * eng.tables.element_size()
    a = eng.acc_ew.numel() * 4 if eng.acc_ew is not None else 0
    return t / 1e9, a / 1e9


def run_cfg2(dtype, opt, steps, warmup, ring):
    from dlrm_b200.data import DeviceBatch, make_batch
    from dlrm_b200.engine import Engine

    W = bench.workload("cfg2")
    D, rows, ln_bot, ln_top = bench.model_dims(W)
    B, lr = W["B"], 0.01
    dev = "cuda:0"
    eng = Engine(D, rows, ln_bot, ln_top, loss="bce", sigmoid_top=len(ln_top) - 2, device=dev, max_batch=B, gemm="tc",
                 emb_dtype=dtype)
    eng.init_params(100)
    eng.ensure_optimizer_state(opt)
    hbs = [make_batch(np.random.default_rng(1000 + i), rows, B, ln_bot[0], W["lmax"]) for i in range(ring)]
    stages = []
    for hb in hbs:
        st = DeviceBatch(hb.layout, dev)
        st.load(hb, non_blocking=False)
        stages.append(st)

    def step(i):
        st = stages[i % ring]
        return eng.train_step(st.X, st.sparse, st.target, lr, opt)

    for i in range(warmup):
        step(i)
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for r in range(steps):
        loss = step(warmup + r)
    ev1.record()
    torch.cuda.synchronize()
    ms = ev0.elapsed_time(ev1) / steps
    # the update alone: link (inside the training gather), backward without the fused update, then the update timed
    upd = []
    for r in range(min(steps, 20)):
        st = stages[r % ring]
        eng.forward(st.X, st.sparse, link=True, skip_head=True)
        eng.backward(st.X, st.sparse, st.target)
        eng.sync_update()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        eng.emb_update(st.sparse, optimizer=opt, lr=lr)
        b.record()
        torch.cuda.synchronize()
        upd.append(a.elapsed_time(b) * 1e3)
    tgb, agb = _arena_gb(eng)
    return {"ms_per_step": ms, "samples_per_s": B / (ms * 1e-3), "update_us_median": float(np.median(upd)),
            "tables_gb": tgb, "accumulators_gb": agb, "loss_last_step": float(loss.item()), "batch": B}


def run_cfg3(dtype, opt, steps, warmup, ring):
    from dlrm_b200 import dist as ddist, mlperf as M, placement as P

    os.environ.update(RANK="0", WORLD_SIZE="1", LOCAL_RANK="0", MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(bench._free_port()))
    os.environ.setdefault("NCCL_NVLS_ENABLE", "0")
    ddist.init_distributed("nccl")
    torch.cuda.set_device(0)
    dev = "cuda:0"
    W = bench.workload("cfg3")
    D = W["m_spa"]
    per_row = (D + 4) * 4 + D * 4                       # interleaved fp32 row + its element-wise accumulator row
    cap = max(M.TABLE_ROWS)
    while sum(min(r, cap) for r in M.TABLE_ROWS) * per_row > FIT_BYTES:
        cap = int(cap * 0.95)
    W["rows"] = [min(r, cap) for r in M.TABLE_ROWS]
    D, rows, ln_bot, ln_top = bench.model_dims(W)
    B, lr = W["B"], 0.01
    cost = bench.lookups_per_sample(W)
    pl = P.plan(rows, cost, 1, bytes_per_row=P.row_bytes(D, dtype))
    de = ddist.DistEngine(D, rows, ln_bot, ln_top, local_batch=B, device=dev, gemm="tc", exchange="p2p",
                          placement=pl, emb_dtype=dtype)
    eng = de.eng
    eng.init_params(100)
    eng.ensure_optimizer_state(opt)
    nsets = 2
    mh = ddist.MultiHotExchange(de, W["hot"], 13, nsets)
    devr = [mh.fill_host(mh.host_buffer(), 1234, i, rows).to(dev) for i in range(ring)]
    stages = [types.SimpleNamespace(sparse=mh.sparse[k], X=mh.X[k], target=mh.target[k]) for k in range(nsets)]

    def step(i):
        k = i % nsets
        mh.stage[k].copy_(devr[i % ring], non_blocking=True)
        mh.exchange(k)
        return eng.train_step(stages[k].X, stages[k].sparse, stages[k].target, lr, opt)

    for i in range(warmup):
        step(i)
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for r in range(steps):
        loss = step(warmup + r)
    ev1.record()
    torch.cuda.synchronize()
    ms = ev0.elapsed_time(ev1) / steps
    tgb, agb = _arena_gb(eng)
    return {"ms_per_step": ms, "samples_per_s": B / (ms * 1e-3), "row_cap": cap, "rows_total": int(sum(rows)),
            "tables_gb": tgb, "accumulators_gb": agb, "loss_last_step": float(loss.item()), "batch": B}


def one_run(name, steps, warmup, ring):
    wl, dtype, opt = RUNS[name]
    t0 = time.time()
    res = (run_cfg2 if wl == "cfg2" else run_cfg3)(dtype, opt, steps, warmup, ring)
    line = {"run": name, "workload": wl, "emb_dtype": dtype, "optimizer": opt, "steps": steps, "warmup": warmup,
            "cuda_graph": False, "wall_s": round(time.time() - t0, 1)}
    line.update(res)
    line.update(gpu_info(0))
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--ring", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=2, help="how many times a, b, c alternate")
    ap.add_argument("--runs", default="a,b,c,d", help="which of a, b, c, d to run")
    ap.add_argument("--one", default=None, help=argparse.SUPPRESS)     # internal: run one configuration here
    args = ap.parse_args()
    if args.one:
        return one_run(args.one, args.steps, max(args.warmup, 3), args.ring)
    want = [r for r in args.runs.split(",") if r]
    order = [r for _ in range(args.repeats) for r in ("a", "b", "c") if r in want] + (["d"] if "d" in want else [])
    failed = 0
    for name in order:
        cmd = [sys.executable, os.path.abspath(__file__), "--one", name, "--steps", str(args.steps),
               "--warmup", str(args.warmup), "--ring", str(args.ring)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
        if r.returncode != 0 or not lines:
            failed += 1
            print(json.dumps({"run": name, "error": (r.stderr or r.stdout)[-1500:]}), flush=True)
        else:
            print(lines[-1], flush=True)
    sys.exit(1 if failed else 0)


if __name__ == "__main__":
    main()
