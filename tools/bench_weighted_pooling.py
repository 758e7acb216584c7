#!/usr/bin/env python
"""The cost of weighted pooling in the fused embedding update, on one H100.

    python tools/bench_weighted_pooling.py [--steps K] [--warmup W] [--repeats 2] [--runs none-sgd,learned-sgd,...]

Workload: the cfg3 model (MLPerf table sizes capped at 20 M rows, dim 128, the multi-hot bags of dlrm_b200/mlperf.py,
MLPs 13-512-256-128 / 1024-1024-512-256-1), batch 8192, fp32 tables, one Engine (no sharding).  Configurations:
pooling none / fixed (v = 1, gathered with the weights, update unweighted) / learned (v stepped by the update) x
optimizer sgd / rwsadagrad.  Each configuration runs in its own process (the 65 GB of tables are freed before the
next), alternated a, b, a, b.  One JSON line per run: the median device time of the embedding update alone (CUDA
events around the update launches after a training forward and backward), ms/step of a captured training step
(CUDA-graph replays, device learning rate), and the GPU's name and power limit.
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

ROW_CAP = 20_000_000
CONFIGS = [p + "-" + o for o in ("sgd", "rwsadagrad") for p in ("none", "fixed", "learned")]


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


def one_run(cfg, steps, warmup, ring):
    from dlrm_b200 import mlperf as M
    from dlrm_b200.engine import Engine, GraphedTrainStep, sparse_from_reference

    pooling, opt = cfg.split("-")
    dev, B, lr, D = "cuda:0", 8192, 0.01, M.DIM
    rows = [min(r, ROW_CAP) for r in M.TABLE_ROWS]
    eng = Engine(D, rows, M.LN_BOT, M.ln_top(len(rows), D), loss="bce", sigmoid_top=len(M.TOP_TAIL) - 1, device=dev,
                 max_batch=B, gemm="tc", learned_row_weights=pooling == "learned")
    eng.init_params(100)
    if pooling == "fixed":
        eng.row_weights = torch.ones(eng.total_rows, dtype=torch.float32, device=dev)
    eng.ensure_optimizer_state(opt)
    stages = []
    for i in range(ring):
        idx = M.multi_hot_batch(1234, i, rows, M.MULTI_HOT, 0, B, dtype=np.int64)
        off = [np.arange(B, dtype=np.int64) * int(L) for L in M.MULTI_HOT]
        X, T = M.dense_and_targets(1234, i, 0, B)
        stages.append(types.SimpleNamespace(
            sparse=sparse_from_reference([torch.from_numpy(o) for o in off],
                                         [torch.from_numpy(a.reshape(-1)) for a in idx], dev),
            X=torch.from_numpy(X).to(dev), target=torch.from_numpy(T).to(dev)))
    # the update alone, on the gradients of a training forward + backward
    upd = []
    for r in range(warmup + steps):
        st = stages[r % ring]
        eng.forward(st.X, st.sparse, link=True, skip_head=True)
        eng.backward(st.X, st.sparse, st.target)
        eng.sync_update()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        eng.emb_update(st.sparse, optimizer=opt, lr=lr)
        b.record()
        torch.cuda.synchronize()
        if r >= warmup:
            upd.append(a.elapsed_time(b) * 1e3)
    # a captured training step, replayed
    g = GraphedTrainStep(eng, stages[0], lr, opt, warmup=3, device_lr=True)
    for _ in range(warmup):
        g.replay(lr)
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(steps):
        loss = g.replay(lr)
    ev1.record()
    torch.cuda.synchronize()
    ms = ev0.elapsed_time(ev1) / steps
    return {"update_us_median": float(np.median(upd)), "update_us_min": float(np.min(upd)), "ms_per_step": ms,
            "loss_last_step": float(loss.item()), "batch": B, "row_cap": ROW_CAP, "rows_total": int(sum(rows))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ring", type=int, default=4)
    ap.add_argument("--repeats", type=int, default=2, help="how many times the configurations alternate")
    ap.add_argument("--runs", default=",".join(CONFIGS), help="configurations, of " + ", ".join(CONFIGS))
    ap.add_argument("--one", default=None, help=argparse.SUPPRESS)     # internal: run one configuration here
    args = ap.parse_args()
    if args.one:
        t0 = time.time()
        line = {"run": args.one, "steps": args.steps, "warmup": args.warmup}
        line.update(one_run(args.one, args.steps, args.warmup, args.ring))
        line.update(gpu_info(0))
        line["wall_s"] = round(time.time() - t0, 1)
        print(json.dumps(line), flush=True)
        return
    want = [r for r in args.runs.split(",") if r]
    bad = [r for r in want if r not in CONFIGS]
    if bad:
        sys.exit("unknown configuration(s): %s (expected some of %s)" % (", ".join(bad), ", ".join(CONFIGS)))
    failed = 0
    for _ in range(args.repeats):
        for name in want:
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
