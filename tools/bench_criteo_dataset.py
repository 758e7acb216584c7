#!/usr/bin/env python
"""The preprocessed-Criteo input path on one GPU: a Kaggle-sized split resident in device memory.

    python tools/bench_criteo_dataset.py [--parts 1,2] [--samples 45840617] [--steps 3000] [--out DIR]

Prints one JSON line per measurement, each with the GPU name, power limit and SM clock read in the same run.
  1. A synthetic shuffled split of --samples samples (the processed Kaggle set holds 45,840,617) with Kaggle's 26
     table sizes: the resident bytes and the upload time of CriteoDataset.to_device(), then per batch at B = 128, 2048
     and 16384
       - gather: DeviceBatches[j] (dlrm_b200_gather_records on the resident split); host time (perf_counter around
         the call, which only enqueues) and device time (CUDA events around it from an idle device, median), and
         the kernel alone (torch.profiler's device-side duration of gather_records_kernel, mean over 200 launches);
       - host: the reference's path, CriteoDataset[i] per sample + collate + the four host-to-device copies;
         host time with the copies synchronised (median).
  2. bench/dlrm_s_criteo_kaggle.sh's PyTorch command (--use-gpu) plus --num-batches=--steps on a synthetic processed
     file of 7 x 200,000 samples with Kaggle's table sizes: the printed ms/it.
Synthetic files go to a temporary directory (or --out) and are removed afterwards.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from dlrm_b200 import criteo  # noqa: E402

# distinct values per categorical feature of the processed Kaggle set (its _fea_count.npz)
KAGGLE_COUNTS = [1460, 583, 10131227, 2202608, 305, 24, 12517, 633, 3, 93145, 5683, 8351593, 3194, 27, 14992,
                 5461306, 10, 5652, 2173, 4, 7046547, 18, 15, 286181, 105, 142572]
KAGGLE_SH = ["--arch-sparse-feature-size=16", "--arch-mlp-bot=13-512-256-64-16", "--arch-mlp-top=512-256-1",
             "--data-generation=dataset", "--data-set=kaggle", "--loss-function=bce", "--round-targets=True",
             "--learning-rate=0.1", "--mini-batch-size=128", "--print-freq=1024", "--print-time",
             "--test-mini-batch-size=16384", "--test-num-workers=16"]


def gpu_info():
    info = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": None, "sm_clock_max_mhz": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=20).stdout
        pw, clk = out.strip().splitlines()[0].split(",")
        info["power_limit_w"], info["sm_clock_max_mhz"] = float(pw), float(clk)
    except Exception:
        pass
    return info


def synthetic_arrays(n, seed):
    rng = np.random.default_rng(seed)
    X_int = np.empty((n, 13), np.int32)
    X_cat = np.empty((n, 26), np.int32)
    y = np.empty(n, np.int32)
    for lo in range(0, n, 1 << 22):
        m = min(1 << 22, n - lo)
        X_int[lo:lo + m] = np.where(rng.random((m, 13), np.float32) < 0.3, 0, rng.integers(0, 1 << 12, (m, 13)))
        X_cat[lo:lo + m] = (rng.random((m, 26), np.float32) * np.asarray(KAGGLE_COUNTS, np.float32)).astype(np.int32)
        y[lo:lo + m] = rng.random(m) < 0.25
    return X_int, X_cat, y


def resident_split(n, seed=0):
    """A CriteoDataset over in-memory arrays (the processed file would be 7.3 GB): a shuffled order of all n."""
    ds = object.__new__(criteo.CriteoDataset)
    ds.X_int, ds.X_cat, ds.y = synthetic_arrays(n, seed)
    ds.counts, ds.m_den, ds.n_emb = np.asarray(KAGGLE_COUNTS), 13, 26
    ds.max_ind_range, ds.memory_map, ds.split, ds._shared, ds.dev = -1, False, "train", None, None
    ds.order = np.random.default_rng(seed + 1).permutation(n).astype(np.int64)
    return ds


def part_input(n, reps=200):
    ds = resident_split(n)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ds.to_device("cuda:0")
    torch.cuda.synchronize()
    line = {"part": "upload", "samples": n, "resident_bytes": ds.resident_bytes(), "upload_s": time.perf_counter() - t0}
    line.update(gpu_info())
    print(json.dumps(line), flush=True)
    for B in (128, 2048, 16384):
        batches = criteo.DeviceBatches(ds, B, "cuda:0")
        nb = len(batches) - 1                                    # full batches only, spread over the split
        js = np.random.default_rng(B).integers(0, nb, reps + 10)
        host, dev = [], []
        for r, j in enumerate(js):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            t0 = time.perf_counter()
            batches[int(j)]
            t1 = time.perf_counter()
            e1.record()
            torch.cuda.synchronize()
            if r >= 10:
                host.append(t1 - t0)
                dev.append(e0.elapsed_time(e1))
        db = batches.batches[B][0]
        ids = ds.dev[3][:B]
        for _ in range(10):
            criteo.gather_records(ds, ids, db)
        # the kernel alone: launches from Python come slower than the kernel runs, so events around a loop of
        # them measure the launch rate; the profiler's device-side kernel durations do not
        from torch.profiler import ProfilerActivity, profile

        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for r in range(reps):
                criteo.gather_records(ds, ds.dev[3][int(js[r]) * B:int(js[r]) * B + B], db)
            torch.cuda.synchronize()
        k = [e for e in prof.key_averages() if "gather_records_kernel" in e.key]
        kernel_us = (getattr(k[0], "device_time_total", None) or k[0].cuda_time_total) / k[0].count if k else None
        href = []
        for r, j in enumerate(js[:min(reps, 40) + 3]):
            t0 = time.perf_counter()
            X, lS_o, lS_i, T = criteo.CriteoDataset.collate(ds[int(j) * B:int(j) * B + B])
            for t in (X, lS_o, lS_i, T):
                t.to("cuda:0")
            torch.cuda.synchronize()
            if r >= 3:
                href.append(time.perf_counter() - t0)
        line = {"part": "batch", "B": B, "gather_host_ms": 1e3 * float(np.median(host)),
                "gather_device_ms": float(np.median(dev)), "gather_kernel_us": kernel_us,
                "gather_bytes_read": B * (40 * 4 + 8), "gather_bytes_written": B * (13 * 4 + 4 + 26 * 8) + 26 * (B + 1) * 8,
                "host_collate_h2d_ms": 1e3 * float(np.median(href))}
        line.update(gpu_info())
        print(json.dumps(line), flush=True)


def part_run(tmp, steps):
    days, per_day = 7, 200_000
    X_int, X_cat, y = synthetic_arrays(days * per_day, 7)
    np.savez(os.path.join(tmp, "kaggle_processed.npz"), X_int=X_int, X_cat=X_cat, y=y,
             counts=np.asarray(KAGGLE_COUNTS, np.int32))
    np.savez(os.path.join(tmp, "train_day_count.npz"), total_per_file=np.full(days, per_day))
    cmd = [sys.executable, os.path.join(ROOT, "dlrm_s_pytorch.py")] + KAGGLE_SH + [
        "--raw-data-file=" + os.path.join(tmp, "train.txt"),
        "--processed-data-file=" + os.path.join(tmp, "kaggle_processed.npz"), "--use-gpu",
        "--num-batches=%d" % steps, "--print-freq=%d" % (steps // 3)]
    t0 = time.perf_counter()
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=tmp)
    lines = r.stdout.splitlines()
    ms = [float(v.split(" ms/it")[0].split(", ")[-1]) for v in lines if v.startswith("Finished training")]
    line = {"part": "kaggle_sh", "returncode": r.returncode, "steps": steps, "ms_per_it": ms,
            "wall_s": time.perf_counter() - t0, "lines": [v for v in lines if v.startswith("Finished")]}
    if r.returncode != 0:
        line["tail"] = (r.stdout + r.stderr).splitlines()[-30:]
    line.update(gpu_info())
    print(json.dumps(line), flush=True)
    return r.returncode


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", default="1,2")
    ap.add_argument("--samples", type=int, default=45_840_617)
    ap.add_argument("--steps", type=int, default=3000)
    ap.add_argument("--out", default=None, help="directory for the synthetic files (default: a temporary one)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("ERROR: needs a CUDA device")
    parts = set(args.parts.split(","))
    rc = 0
    with tempfile.TemporaryDirectory(dir=args.out) as tmp:
        if "1" in parts:
            part_input(args.samples)
        if "2" in parts:
            rc = part_run(tmp, args.steps)
    sys.exit(rc)


if __name__ == "__main__":
    main()
