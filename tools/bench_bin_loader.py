#!/usr/bin/env python
"""The MLPerf binary-record path on one GPU: input path, metrics finalize and the run_and_time.sh command.

    python tools/bench_bin_loader.py [--parts 1,2,3] [--train-batches 300] [--test-batches 3] [--out DIR]

Prints one JSON line per measurement, each with the GPU name and power limit read in the same run.
  1. Per-batch input path at B = 2048 and 16384: the host fill() into the packed pinned batch plus its one H2D copy,
     against CriteoBinDataset.load() (pinned raw copy, H2D of the records, decode kernel).  Host time (perf_counter
     around the host work), device time (CUDA events around the copies and the decode), bytes crossing the bus, and
     the decode kernel alone (events around repeated launches on records already on the device).
  2. Metrics finalize at 89,137,319 synthetic scores with ties (the size of the reference's Terabyte test split):
     device time of ScoreKeys.finalize(), the peak of its temporary device memory, and sklearn's time for the reference's six calls on the same arrays when
     sklearn imports (else "not measured").
  3. bench/run_and_time.sh's flags plus --emb-dtype=fp16 --num-batches=N on a synthetic Terabyte-shaped file (the
     40 M-capped table sizes of dlrm_b200/mlperf.py, uniform ids): the printed ms/it and the wall time of one test
     pass (from the 'Testing at' line to the metric line).
Synthetic files are written to a temporary directory (or --out) and removed afterwards.
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

from dlrm_b200 import binrecords as BR  # noqa: E402
from dlrm_b200.data import DeviceBatch, HostBatch, PackedLayout  # noqa: E402

RUN_AND_TIME = ["--arch-sparse-feature-size=128", "--arch-mlp-bot=13-512-256-128", "--arch-mlp-top=1024-1024-512-256-1",
                "--max-ind-range=40000000", "--data-generation=dataset", "--data-set=terabyte", "--loss-function=bce",
                "--round-targets=True", "--learning-rate=1.0", "--mini-batch-size=2048", "--print-freq=2048",
                "--print-time", "--test-freq=102400", "--test-mini-batch-size=16384", "--test-num-workers=16",
                "--memory-map", "--mlperf-logging", "--mlperf-auc-threshold=0.8025", "--mlperf-bin-loader",
                "--mlperf-bin-shuffle"]


def gpu_info():
    info = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        info["power_limit_w"] = float(out.splitlines()[0])
    except Exception:
        pass
    return info


def write_records(path, n, counts, seed):
    rng = np.random.default_rng(seed)
    with open(path, "wb") as f:
        for lo in range(0, n, 1 << 18):
            m = min(1 << 18, n - lo)
            rec = np.empty((m, 40), dtype=np.int32)
            rec[:, 0] = rng.random(m) < 0.25
            rec[:, 1:14] = np.where(rng.random((m, 13)) < 0.3, 0, rng.integers(0, 1 << 16, (m, 13)))
            rec[:, 14:] = (rng.random((m, 26)) * np.asarray(counts)).astype(np.int64)
            f.write(rec.tobytes())


def part_input(tmp, reps=50):
    from dlrm_b200.mlperf import TABLE_ROWS

    for B in (2048, 16384):
        nb = 8
        p = os.path.join(tmp, "in_%d.bin" % B)
        write_records(p, B * nb, TABLE_ROWS, B)
        ds = BR.CriteoBinDataset(p, None, batch_size=B, max_ind_range=40_000_000)
        L = PackedLayout(B, 26, 13, B * 26)
        hb, db = HostBatch(L), DeviceBatch(L, "cuda:0")
        res = {}
        for name in ("host_fill_packed_h2d", "raw_h2d_device_decode"):
            host_s, ev = 0.0, []
            for r in range(reps + 5):
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0 = time.perf_counter()
                if name == "host_fill_packed_h2d":
                    ds.fill(r % nb, hb)
                    t1 = time.perf_counter()
                    e0.record()
                    nbytes = db.load(hb)
                else:
                    e0.record()
                    ds.load(r % nb, db)
                    t1 = time.perf_counter()
                    nbytes = B * 160
                e1.record()
                torch.cuda.synchronize()
                if r >= 5:
                    host_s += t1 - t0
                    ev.append(e0.elapsed_time(e1))
            res[name] = {"host_ms": 1e3 * host_s / reps, "device_ms": float(np.median(ev)), "h2d_bytes": nbytes}
        # the decode kernel alone, on the records load() left on the device (index writes are table-major)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        raw = ds._raw[:B]
        for _ in range(5):
            BR.decode_records(raw, ds.max_ind_range, db)
        e0.record()
        for _ in range(reps):
            BR.decode_records(raw, ds.max_ind_range, db)
        e1.record()
        torch.cuda.synchronize()
        res["decode_kernel_us"] = 1e3 * e0.elapsed_time(e1) / reps
        line = {"part": "input_path", "B": B, **res}
        line.update(gpu_info())
        print(json.dumps(line), flush=True)


def part_metrics(n=89_137_319):
    from dlrm_b200 import metrics as M

    g = torch.Generator(device="cuda:0").manual_seed(1)
    s = torch.randint(0, 1 << 16, (n,), device="cuda:0", generator=g).float() / 65535     # 65536 distinct scores
    y = (torch.rand(n, device="cuda:0", generator=g) < 0.1 + 0.3 * s).float()
    acc = M.ScoreKeys(n, "cuda:0")
    acc.add(s, y)
    acc.finalize()                                            # warm-up (allocator, sort workspace)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    acc.finalize()
    finalize_temp_bytes = torch.cuda.max_memory_allocated() - base     # temporaries beyond the keys and the scores
    times = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = acc.finalize()                                  # ends in host reads: synchronised
        times.append(time.perf_counter() - t0)
    line = {"part": "metrics_finalize", "n": n, "device_finalize_s": float(np.median(times)), "auc": res["roc_auc"],
            "keys_bytes": acc.keys.numel() * 4, "finalize_temp_bytes": finalize_temp_bytes}
    try:
        import sklearn.metrics as skm
    except ImportError:
        line["sklearn_s"] = "not measured"
    else:
        sn, yn = s.cpu().numpy(), y.cpu().numpy()
        t0 = time.perf_counter()
        pred = np.round(sn)
        for f in (skm.recall_score, skm.precision_score, skm.f1_score, skm.accuracy_score):
            f(yn, pred)
        skm.average_precision_score(yn, sn)
        auc = skm.roc_auc_score(yn, sn)
        line["sklearn_s"] = time.perf_counter() - t0
        line["sklearn_auc_minus_device"] = auc - res["roc_auc"]
    line.update(gpu_info())
    print(json.dumps(line), flush=True)


def part_run(tmp, train_batches, test_batches):
    from dlrm_b200.mlperf import TABLE_ROWS

    write_records(os.path.join(tmp, "tb_train.bin"), 2048 * train_batches, TABLE_ROWS, 1)
    write_records(os.path.join(tmp, "tb_test.bin"), 16384 * test_batches, TABLE_ROWS, 2)
    np.savez(os.path.join(tmp, "day_fea_count.npz"), counts=np.asarray(TABLE_ROWS))
    cmd = [sys.executable, os.path.join(ROOT, "dlrm_s_pytorch.py")] + RUN_AND_TIME + [
        "--raw-data-file=" + os.path.join(tmp, "day"), "--processed-data-file=" + os.path.join(tmp, "tb.npz"),
        "--use-gpu", "--emb-dtype=fp16", "--num-batches=%d" % train_batches, "--print-freq=%d" % (train_batches // 2),
        "--test-freq=%d" % train_batches]
    t_start = time.perf_counter()
    proc = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, cwd=tmp)
    lines, t_test, test_s = [], None, None
    for ln in proc.stdout:
        lines.append(ln.rstrip())
        if ln.startswith("Testing at"):
            t_test = time.perf_counter()
        elif ln.startswith("recall ") and t_test is not None:
            test_s = time.perf_counter() - t_test
    rc = proc.wait()
    ms = [float(v.split(" ms/it")[0].split(", ")[-1]) for v in lines if v.startswith("Finished training")]
    line = {"part": "run_and_time_fp16", "returncode": rc, "train_batches": train_batches,
            "test_samples": 16384 * test_batches, "ms_per_it": ms, "test_pass_s": test_s,
            "wall_s": time.perf_counter() - t_start,
            "lines": [v for v in lines if v.startswith(("Finished", "Testing", "recall", "MLPerf"))]}
    if rc != 0:
        line["tail"] = lines[-30:]
    line.update(gpu_info())
    print(json.dumps(line), flush=True)
    return rc


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", default="1,2,3")
    ap.add_argument("--train-batches", type=int, default=300)
    ap.add_argument("--test-batches", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for the synthetic files (default: a temporary one)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("ERROR: needs a CUDA device")
    parts = set(args.parts.split(","))
    rc = 0
    with tempfile.TemporaryDirectory(dir=args.out) as tmp:
        if "1" in parts:
            part_input(tmp)
        if "2" in parts:
            part_metrics()
        if "3" in parts:
            rc = part_run(tmp, args.train_batches, args.test_batches)
    sys.exit(rc)


if __name__ == "__main__":
    main()
