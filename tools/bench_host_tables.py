"""Host embedding tables on one GPU: the staging kernels alone, and the MLPerf training step with tables on the host.

  python tools/bench_host_tables.py [--out DIR] [--steps 200] [--iters 50]

1. Staging kernels: stage-in and write-back of n distinct random rows of a pinned fp32 table of >= 8 GB (528-byte
   interleaved rows), CUDA events over many launches; beside them a cudaMemcpy of a contiguous pinned buffer of the
   same bytes, the link's practical rate.
2. Train step of bench/run_and_time.sh's model (MLPerf MLPs, D = 128, one-hot, batch 2048, rwsadagrad, fp32 tables):
   (a) every table on the device vs (b) tables 0, 9, 19, 20, 21 on the host, both at a 10 M row cap, timed a, b, a, b;
   (c) the 40 M cap with those five tables on the host.
Every size that would not fit into MemAvailable (less a 16 GB margin) is refused before anything is pinned, and the
output says what ran instead.  Prints one JSON object; the card's name, power limit and max SM clock come first."""
import argparse
import ctypes as C
import gc
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from dlrm_b200 import _lib  # noqa: E402
from dlrm_b200.engine import Engine  # noqa: E402
from dlrm_b200.mlperf import TABLE_ROWS  # noqa: E402

DEV = "cuda:0"
ROW = 132 * 4          # interleaved fp32 row at D = 128
MARGIN = 16 << 30
BIG = [0, 9, 19, 20, 21]


def mem_available():
    for ln in open("/proc/meminfo"):
        if ln.startswith("MemAvailable:"):
            return int(ln.split()[1]) * 1024
    return 0


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q


def events_ms(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def staging(rows, sizes, iters):
    lib = _lib.lib()
    table = torch.zeros(rows, 132)
    t0 = time.time()
    assert lib.dlrm_b200_host_register(table.data_ptr(), table.numel() * 4) == 0, lib.dlrm_b200_last_error()
    pin_s = time.time() - t0
    out = dict(table_rows=rows, table_bytes=rows * ROW, register_s=round(pin_s, 2), sizes=[])
    try:
        smap = torch.zeros(rows, dtype=torch.int32, device=DEV)
        for n in sizes:
            idx = torch.randperm(rows, device=DEV)[:n].contiguous()
            off = torch.tensor([0, n], dtype=torch.int64, device=DEV)
            sw = torch.zeros(n, 132, device=DEV)
            sidx = torch.zeros(n, dtype=torch.int64, device=DEV)
            lst = torch.zeros(n, dtype=torch.int32, device=DEV)
            key = torch.zeros(n, dtype=torch.int64, device=DEV)
            cnt = torch.zeros(1, dtype=torch.int32, device=DEV)
            d = (_lib.HostTable * 1)()
            d[0].weight, d[0].indices, d[0].offsets, d[0].nnz = table.data_ptr(), idx.data_ptr(), off.data_ptr(), n
            d[0].rows, d[0].map = rows, smap.data_ptr()
            st = _lib.HostStage(weight=sw.data_ptr(), slot_idx=sidx.data_ptr(), list=lst.data_ptr(), key=key.data_ptr(),
                                count=cnt.data_ptr(), capacity=n, ld=132, head_col=129)
            s = torch.cuda.current_stream().cuda_stream
            si = lambda: _lib.check(lib.dlrm_b200_host_stage_in(d, 1, C.byref(st), 128, 1, 8, 1, s), "stage_in")
            wb = lambda: _lib.check(lib.dlrm_b200_host_write_back(d, 1, C.byref(st), 128, s), "write_back")
            si(), wb()
            torch.cuda.synchronize()
            a, b, c, e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            t_in = t_wb = 0.0
            for _ in range(iters):
                a.record(); si(); b.record(); wb(); c.record()
                torch.cuda.synchronize()
                t_in += a.elapsed_time(b)
                t_wb += b.elapsed_time(c)
            t_in, t_wb = t_in / iters, t_wb / iters
            assert int(cnt.item()) == n and int(smap.abs().sum().item()) == 0
            hb = torch.empty(n * 132, dtype=torch.float32).pin_memory()
            db = torch.empty(n * 132, dtype=torch.float32, device=DEV)
            h2d = events_ms(lambda: db.copy_(hb, non_blocking=True), iters)
            d2h = events_ms(lambda: hb.copy_(db, non_blocking=True), iters)
            nb = n * ROW
            out["sizes"].append(dict(rows=n, bytes=nb,
                                     stage_in_us=round(t_in * 1e3, 1), stage_in_Mrows_s=round(n / t_in / 1e3, 2),
                                     stage_in_GB_s=round(nb / t_in / 1e6, 2),
                                     write_back_us=round(t_wb * 1e3, 1), write_back_Mrows_s=round(n / t_wb / 1e3, 2),
                                     write_back_GB_s=round(nb / t_wb / 1e6, 2),
                                     memcpy_h2d_GB_s=round(nb / h2d / 1e6, 2), memcpy_d2h_GB_s=round(nb / d2h / 1e6, 2)))
            del hb, db
    finally:
        torch.cuda.synchronize()
        lib.dlrm_b200_host_unregister(table.data_ptr())
    return out


def model(cap, host):
    rows = [min(r, cap) for r in TABLE_ROWS]
    t0 = time.time()
    e = Engine(128, rows, [13, 512, 256, 128], [479, 1024, 1024, 512, 256, 1], sigmoid_top=4, device=DEV,
               max_batch=2048, gemm="tc", host_tables=host)
    e.init_params(seed=0)
    torch.cuda.synchronize()
    return e, rows, round(time.time() - t0, 1)


def batches(rows, n, seed):
    from dlrm_b200.data import make_batch, to_device_packed

    rng = np.random.default_rng(seed)
    return [to_device_packed(make_batch(rng, rows, 2048, lmax=1, fixed=True), DEV) for _ in range(n)]


def step_ms(e, bs, steps):
    for b in bs[:3]:
        e.train_step(b.X, b.sparse, b.target, 0.01, "rwsadagrad")
    torch.cuda.synchronize()
    a, z = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(steps):
        b = bs[i % len(bs)]
        e.train_step(b.X, b.sparse, b.target, 0.01, "rwsadagrad")
    z.record()
    torch.cuda.synchronize()
    return a.elapsed_time(z) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    res = dict(card=card(), mem_available=mem_available())
    # 1. staging kernels: a >= 8 GB table when it fits
    rows = 16_000_000
    while rows * ROW + MARGIN > mem_available() and rows > 2_000_000:
        rows //= 2
    res["staging_note"] = "ran a %d-row table (%.1f GB)" % (rows, rows * ROW / 1e9)
    res["staging"] = [staging(rows, [10240, 53248, 1 << 20], args.iters) for _ in range(2)]
    # 2. train step at the 10 M cap: a / b alternated
    need_b = sum(min(TABLE_ROWS[k], 10_000_000) for k in BIG) * ROW
    if need_b + MARGIN > mem_available():
        res["train_10M"] = "not run: %d pinned bytes do not fit MemAvailable %d" % (need_b, mem_available())
    else:
        ea, rows10, ta = model(10_000_000, [])
        eb, _, tb = model(10_000_000, BIG)
        bs = batches(rows10, 8, 1)
        times = {"a_device": [], "b_host": []}
        for _ in range(2):
            times["a_device"].append(round(step_ms(ea, bs, args.steps), 3))
            times["b_host"].append(round(step_ms(eb, bs, args.steps), 3))
        res["train_10M"] = dict(ms_per_step=times, pinned_bytes=eb.pinned_bytes, build_init_s=[ta, tb])
        del ea, eb, bs
        gc.collect()                 # the engines' pinned arenas go back before (c) reads MemAvailable
        torch.cuda.empty_cache()
    # 3. the 40 M cap with the five 40 M tables on the host
    need_c = sum(TABLE_ROWS[k] for k in BIG) * ROW
    if need_c + MARGIN > mem_available():
        res["train_40M"] = "not run: %d pinned bytes (+16 GB margin) do not fit MemAvailable %d" % (
            need_c, mem_available())
    else:
        ec, rows40, tc = model(40_000_000, BIG)
        bs = batches(rows40, 8, 2)
        res["train_40M"] = dict(ms_per_step=[round(step_ms(ec, bs, args.steps), 3) for _ in range(2)],
                                pinned_bytes=ec.pinned_bytes, build_init_s=tc)
    txt = json.dumps(res)
    print(txt)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_host_tables.json"), "w") as fh:
            fh.write(txt + "\n")


if __name__ == "__main__":
    main()
