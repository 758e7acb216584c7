#!/usr/bin/env python
"""The per-day Criteo path (--memory-map) on one GPU: inflate, ingest, stream, and the Terabyte command.

    python tools/bench_criteo_days.py [--parts 1,2,3] [--samples 3000000] [--steps 1500] [--data DIR]

One synthetic float64 day of --samples samples is written as the reference writes a reordered day
(savez_compressed of X_int [n, 13], X_cat [n, 26], y [n]; Terabyte table sizes, the 40 M-capped counts of
dlrm_b200/mlperf.py, uniform ids, sparse small counts), and linked under all 24 Terabyte day names.  Its
compressibility, and with it the inflate rate, is that of this synthetic data, not of the real set.  --data keeps the
files in DIR between runs (they are made once); by default a temporary directory is used and removed.
Prints one JSON line per measurement, each with the GPU name, power limit and SM clock read in the same run.
  1. host: inflate rate of each member alone and of the worker thread (three members at once), in samples/s; the
     reference's path per batch at B = 2048 and 16384 (its np.load of a whole day, then per-sample items and the
     collate, here criteo.CriteoDataset.collate, with the four host-to-device copies).
  2. device: the ingest kernel per chunk of CHUNK_ROWS float64 samples (torch.profiler's device time of
     ingest_records_kernel, mean of 50), its bytes per second against 3.35 TB/s; DayBatches ms per batch at
     B = 2048 and 16384 with nothing else running (the stream's own rate), its device bytes and pinned host bytes.
  3. bench/dlrm_s_criteo_terabyte.sh's PyTorch command (--use-gpu) plus --memory-map and --num-batches=--steps,
     against the same command on a resident split (no --memory-map; a processed file of 24 x 200,000 samples of the
     same day): the printed ms/it (training step only) and the wall time per iteration of the whole training loop
     (from the first to the last 'Finished training' line).
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

from dlrm_b200 import criteo, criteo_days as CD, _lib  # noqa: E402
from dlrm_b200.mlperf import TABLE_ROWS  # noqa: E402

TERABYTE_SH = ["--arch-sparse-feature-size=64", "--arch-mlp-bot=13-512-256-64", "--arch-mlp-top=512-512-256-1",
               "--max-ind-range=10000000", "--data-generation=dataset", "--data-set=terabyte", "--loss-function=bce",
               "--round-targets=True", "--learning-rate=0.1", "--mini-batch-size=2048", "--print-freq=1024",
               "--print-time", "--test-mini-batch-size=16384", "--test-num-workers=16"]
HBM_BYTES_PER_S = 3.35e12


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


def emit(line):
    line.update(gpu_info())
    print(json.dumps(line), flush=True)


def make_day(n, seed=0):
    rng = np.random.default_rng(seed)
    X_int = np.where(rng.random((n, 13), np.float32) < 0.3, 0, rng.geometric(0.02, (n, 13)) - 1).astype(np.float64)
    X_cat = np.floor(rng.random((n, 26)) * np.asarray(TABLE_ROWS, np.float64))
    y = (rng.random(n) < 0.25).astype(np.float64)
    return X_int, X_cat, y


def prepare(d, n):
    """`d/day_{0..23}_reordered.npz` (one file, linked), the day and feature counts, and a resident processed file."""
    raw = os.path.join(d, "day")
    files, count_file, fea_file = CD.day_files("terabyte", raw)
    if not os.path.exists(files[-1]):
        X_int, X_cat, y = make_day(n)
        t0 = time.perf_counter()
        np.savez_compressed(files[0], X_int=X_int, X_cat=X_cat, y=y)
        emit({"part": "generate", "samples": n, "compress_s": time.perf_counter() - t0,
              "file_bytes": os.path.getsize(files[0]), "inflated_bytes": X_int.nbytes + X_cat.nbytes + y.nbytes})
        for f in files[1:]:
            os.link(files[0], f)
        np.savez(count_file, total_per_file=np.full(24, n))
        np.savez(fea_file, counts=np.asarray(TABLE_ROWS))
        m = 200_000
        np.savez(os.path.join(d, "terabyte_processed.npz"), X_int=np.tile(X_int[:m].astype(np.int32), (24, 1)),
                 X_cat=np.tile(X_cat[:m].astype(np.int32), (24, 1)), y=np.tile(y[:m].astype(np.int32), 24),
                 counts=np.asarray(TABLE_ROWS))
        np.savez(os.path.join(d, "resident_day_count.npz"), total_per_file=np.full(24, m))
    return raw, files


def part_host(files, n):
    for name, cols in CD.MEMBERS:
        r = CD.MemberReader(files[0], name, cols)
        buf = np.empty(CD.CHUNK_ROWS * cols * 8, np.uint8)
        t0 = time.perf_counter()
        for lo in range(0, n, CD.CHUNK_ROWS):
            r.readinto(buf, min(CD.CHUNK_ROWS, n - lo))
        dt = time.perf_counter() - t0
        r.close()
        emit({"part": "inflate_member", "member": name, "samples_per_s": n / dt, "inflated_mb_per_s": n * cols * 8 / dt / 1e6})
    bufs = [np.empty(CD.slot_bytes(CD.CHUNK_ROWS), np.uint8) for _ in range(CD.SLOTS)]
    t0 = time.perf_counter()
    pr = CD._Producer(files[:1], [n], [(0, 0, n)], 0, CD.CHUNK_ROWS, bufs)
    while True:
        c = pr.ready.get()
        if c is None or isinstance(c, BaseException):
            break
        pr.free.put(c.slot)
    dt = time.perf_counter() - t0
    pr.close()
    emit({"part": "inflate_worker", "samples_per_s": n / dt, "error": repr(c) if c is not None else None})
    # the reference's path: np.load of a whole day, then per-sample items and the collate
    t0 = time.perf_counter()
    with np.load(files[0]) as z:
        X_int, X_cat, y = z["X_int"], z["X_cat"], z["y"]
    load_s = time.perf_counter() - t0
    mir = 10_000_000
    for B in (2048, 16384):
        times = []
        for r in range(6):
            lo = r * B
            t0 = time.perf_counter()
            items = [(X_int[i], X_cat[i] % mir, y[i]) for i in range(lo, lo + B)]
            for t in criteo.CriteoDataset.collate(items):
                t.to("cuda:0")
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
        emit({"part": "reference_path", "B": B, "day_np_load_s": load_s, "items_collate_h2d_ms": 1e3 * float(np.median(times[1:])),
              "day_load_ms_per_batch": 1e3 * load_s * B / n})
    del X_int, X_cat, y


def part_device(raw, n):
    from torch.profiler import ProfilerActivity, profile

    C = CD.CHUNK_ROWS
    X_int, X_cat, y = (torch.from_numpy(a[:C]).to("cuda:0") for a in make_day(C, 1))
    ring = (torch.empty(2 * C, 13, dtype=torch.int32, device="cuda:0"),
            torch.empty(2 * C, 26, dtype=torch.int32, device="cuda:0"), torch.empty(2 * C, dtype=torch.int32, device="cuda:0"))
    bad = torch.full((1,), -1, dtype=torch.int64, device="cuda:0")

    def launch(dst):
        _lib.check(_lib.lib().dlrm_b200_ingest_records(X_int.data_ptr(), 0, X_cat.data_ptr(), 0, y.data_ptr(), 0, C,
                                                       13, 26, ring[0].data_ptr(), ring[1].data_ptr(),
                                                       ring[2].data_ptr(), 2 * C, dst, bad.data_ptr(), None))
    for i in range(10):
        launch(i * 977 % (2 * C))
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(50):
            launch(i * 977 % (2 * C))
        torch.cuda.synchronize()
    k = [e for e in prof.key_averages() if "ingest_records_kernel" in e.key]
    us = (getattr(k[0], "device_time_total", None) or k[0].cuda_time_total) / k[0].count
    nbytes = C * 40 * (8 + 4)
    emit({"part": "ingest_kernel", "chunk_samples": C, "kernel_us": us, "bytes": nbytes,
          "bytes_per_s": nbytes / (us * 1e-6), "share_of_3.35TB_s": nbytes / (us * 1e-6) / HBM_BYTES_PER_S,
          "bad_word": int(bad.item())})
    for B in (2048, 16384):
        s = CD.DayBatches("terabyte", raw, "train", B, 10_000_000, "cuda:0")
        nb = min(len(s), (2 * n) // B)                # two days: one day switch in the window
        s[0]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for j in range(1, nb):
            s[j]
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        emit({"part": "stream", "B": B, "batches": nb - 1, "ms_per_batch": 1e3 * dt / (nb - 1),
              "samples_per_s": (nb - 1) * B / dt, "device_bytes": s.device_bytes(), "pinned_host_bytes": s.host_bytes()})
        s.close()


def part_cli(d, raw, steps):
    out = {}
    for mode in ("memory_map", "resident"):
        flags = ["--memory-map", "--raw-data-file=" + raw] if mode == "memory_map" else [
            "--raw-data-file=" + os.path.join(d, "resident"),
            "--processed-data-file=" + os.path.join(d, "terabyte_processed.npz")]
        cmd = [sys.executable, os.path.join(ROOT, "dlrm_s_pytorch.py")] + TERABYTE_SH + flags + [
            "--use-gpu", "--num-batches=%d" % steps, "--print-freq=%d" % (steps // 5)]
        r = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, cwd=d)
        stamps, lines = [], []
        for ln in r.stdout:
            if ln.startswith("Finished training"):
                stamps.append(time.perf_counter())
                lines.append(ln.strip())
        r.wait()
        ms = [float(v.split(" ms/it")[0].split(", ")[-1]) for v in lines]
        wall = 1e3 * (stamps[-1] - stamps[0]) / (steps - steps // 5) if len(stamps) > 1 else None
        out[mode] = wall
        emit({"part": "terabyte_sh", "mode": mode, "returncode": r.returncode, "steps": steps,
              "printed_step_ms_per_it": ms, "wall_ms_per_it": wall, "lines": lines})
    if all(out.values()):
        emit({"part": "terabyte_sh_ratio", "memory_map_over_resident_wall": out["memory_map"] / out["resident"]})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", default="1,2,3")
    ap.add_argument("--samples", type=int, default=3_000_000)
    ap.add_argument("--steps", type=int, default=1500)
    ap.add_argument("--data", default=None, help="directory that keeps the synthetic files between runs")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("ERROR: needs a CUDA device")
    parts = set(args.parts.split(","))
    with tempfile.TemporaryDirectory() as tmp:
        d = args.data or tmp
        os.makedirs(d, exist_ok=True)
        raw, files = prepare(d, args.samples)
        if "1" in parts:
            part_host(files, args.samples)
        if "2" in parts:
            part_device(raw, args.samples)
        if "3" in parts:
            part_cli(d, raw, args.steps)


if __name__ == "__main__":
    main()
